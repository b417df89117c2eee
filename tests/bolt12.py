"""BOLT12 test helpers: bech32 without checksum, TLV streams, the fixture, and the reference's BOLT12 check as an oracle.

The reference side is oracle/bolt12_harness.c (built by oracle/bolt12.mk into oracle/_ref/libcln_bolt12.so):
cln_bolt12_check runs CLN's own fromwire_tlv, merkle_tlv, sighash_from_merkle and check_schnorr_sig.  Tests reach it
through tests/oracle_replay.py like every other reference call, so they replay its recorded answers where the reference is
not built.
"""
import ctypes
import os

import numpy as np

from tests import oracle_replay

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "bolt12_vectors.npz")
LIB = os.path.join(ROOT, "oracle", "_ref", "libcln_bolt12.so")
# (messagename, fieldname) pairs the fixture signs under: the tags of invoice and invoice_request signatures
NAMES = [(b"invoice", b"signature"), (b"invoice_request", b"signature")]

# cln_bolt12_check(stream, len, messagename, fieldname, xonly32, sig64, merkle32_out, sighash32_out); names are passed
# as Python bytes, so reading 64 bytes takes the whole (shorter) string
oracle_replay.SPEC.setdefault(
    "cln_bolt12_check", (lambda v: {0: v[1], 2: 64, 3: 64, 4: 32, 5: 64}, lambda v: {6: 32, 7: 32}, ()))

_CHARSET = "qpzry9x8gf2tvdw0s3jn54khce6mua7l"


def bech32_decode_nochk(s):
    """BOLT12 string (lno/lnr/lni, '+' continuations allowed) -> (hrp, raw TLV bytes), or None.  No checksum."""
    s = "".join(s.split()).replace("+", "").lower()
    if "1" not in s:
        return None
    hrp, data = s.rsplit("1", 1)
    acc = bits = 0
    out = bytearray()
    for c in data:
        v = _CHARSET.find(c)
        if v < 0:
            return None
        acc = (acc << 5) | v
        bits += 5
        if bits >= 8:
            bits -= 8
            out.append((acc >> bits) & 0xFF)
    return hrp, bytes(out)


def bigsize(v):
    if v < 0xFD:
        return bytes([v])
    if v <= 0xFFFF:
        return b"\xfd" + v.to_bytes(2, "big")
    if v <= 0xFFFFFFFF:
        return b"\xfe" + v.to_bytes(4, "big")
    return b"\xff" + v.to_bytes(8, "big")


def record(t, value):
    return bigsize(t) + bigsize(len(value)) + bytes(value)


def parse_fields(stream):
    """(type, value offset, value) of every record of a well-formed stream (no validity checks beyond the walk)."""
    out, pos = [], 0

    def get(p):
        b = stream[p]
        n = {0xFD: 2, 0xFE: 4, 0xFF: 8}.get(b, 0)
        return (b, 1) if n == 0 else (int.from_bytes(stream[p + 1:p + 1 + n], "big"), 1 + n)

    while pos < len(stream):
        t, a = get(pos)
        ln, b = get(pos + a)
        vo = pos + a + b
        out.append((t, vo, stream[vo:vo + ln]))
        pos = vo + ln
    return out


def load_fixture():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


def streams(fx):
    blob = fx["blob"].tobytes()
    return [blob[o:o + n] for o, n in zip(fx["off"].tolist(), fx["len"].tolist())]


def oracle():
    """The reference's cln_bolt12_check, recorded on the module's `cln` tape (tests/oracle_replay.py)."""
    o = oracle_replay.Oracle("cln")
    o.lib = ctypes.CDLL(LIB) if (oracle_replay.RECORD_DIR or os.path.exists(LIB)) else None
    return o


def ref_check(o, stream, names, xonly, sig):
    """-> (status, merkle32, sighash32) from the reference"""
    m, h = np.zeros(32, np.uint8), np.zeros(32, np.uint8)
    p8 = ctypes.POINTER(ctypes.c_uint8)
    r = o.cln_bolt12_check(bytes(stream), ctypes.c_size_t(len(stream)), names[0], names[1], bytes(xonly), bytes(sig),
                           m.ctypes.data_as(p8), h.ctypes.data_as(p8))
    return int(r), m.tobytes(), h.tobytes()
