"""BOLT11 test helpers: the signing hash, the fixture, and how Core Lightning's answers map to the engine's statuses.

The reference side is oracle/bolt11_harness.c (built by oracle/bolt11.mk into oracle/_ref/libcln_bolt11.so): its
cln_bolt11_check runs CLN's own bolt11_decode and bolt11_decode_nosig, cln_ecdsa_recover libsecp256k1's
secp256k1_ecdsa_recover.  tests/golden/make_bolt11.py stores their answers in the fixture; tests reach the library through
tests/oracle_replay.py, so they replay the recorded answers where the reference is not built.
"""
import ctypes
import hashlib
import os

import numpy as np

from tests import oracle_replay

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "bolt11_vectors.npz")
LIB = os.path.join(ROOT, "oracle", "_ref", "libcln_bolt11.so")
CHARSET = "qpzry9x8gf2tvdw0s3jn54khce6mua7l"
UNCHECKED = 9  # expected_status of an invoice CLN refuses for a field value the engine does not check

# cln_bolt11_check(buf, len, node33_out, hash32_out, fail256_out, nosig_fail256_out)
oracle_replay.SPEC.setdefault(
    "cln_bolt11_check", (lambda v: {0: v[1]}, lambda v: {2: 33, 3: 32, 4: 256, 5: 256}, ()))
oracle_replay.SPEC.setdefault("cln_ecdsa_recover", (lambda v: {0: 64, 2: 32}, lambda v: {3: 33}, ()))

# bolt11_decode's messages for the signature step's refusals (status 0)
SIG_REFUSALS = ("invalid recovery ID", "signature invalid", "signature recovery failed", "invalid signature")
# its messages for an unsound structure (status -1): bech32, timestamp, tag walk, signature length, the `n` key
STRUCTURAL = ("Bad bech32 string", "Can't get 35-bit timestamp", "Can't get tag", "Can't get length",
              "can't read signature", "invalid public key")


def signing_hash(hrp, words):
    """hash_u5 (common/hash_u5.c): SHA-256 of the lowercased hrp and the words packed to bytes, zero-padded"""
    v, nbits = 0, 0
    for w in words:
        v, nbits = (v << 5) | w, nbits + 5
    pad = (-nbits) % 8
    data = (v << pad).to_bytes((nbits + pad) // 8, "big") if nbits else b""
    return hashlib.sha256(hrp.lower().encode() + data).digest()


def expected_status(ret, fail, label_names):
    """Status the engine must give each fixture item, from CLN's answer (bit 0 of ret: bolt11_decode accepted), or
    UNCHECKED.  "non-zero trailing bits" names no field: it is the `n` check only for the items built for it."""
    out = np.full(len(ret), UNCHECKED, np.int32)
    for i, (r, f, lab) in enumerate(zip(ret, fail, label_names)):
        if r & 1:
            out[i] = 1
        elif f.startswith(SIG_REFUSALS):
            out[i] = 0
        elif f.startswith(STRUCTURAL) or (len(f) > 3 and f[1:] == ": truncated"):
            out[i] = -1
        elif f == "non-zero trailing bits" and lab == "n_trailing":
            out[i] = -1
    return out


def load_fixture():
    with np.load(FIXTURE) as z:
        fx = {k: z[k] for k in z.files}
    fx["label_name"] = fx["labels"][fx["label"]]
    fx["expected"] = expected_status(fx["ret"], fx["fail"], fx["label_name"])
    return fx


def invoices(fx):
    blob = fx["blob"].tobytes()
    return [blob[o:o + n] for o, n in zip(fx["off"].tolist(), fx["len"].tolist())]


def oracle():
    """The reference's BOLT11 decoder, recorded on the module's `cln` tape (tests/oracle_replay.py)."""
    o = oracle_replay.Oracle("cln")
    o.lib = ctypes.CDLL(LIB) if (oracle_replay.RECORD_DIR or os.path.exists(LIB)) else None
    return o


def ref_check(o, s):
    """-> (ret, node33, hash32, fail, nosig_fail) from the reference for the invoice bytes s (read up to a NUL)"""
    node, h = np.zeros(33, np.uint8), np.zeros(32, np.uint8)
    f, nf = ctypes.create_string_buffer(256), ctypes.create_string_buffer(256)
    p8 = ctypes.POINTER(ctypes.c_uint8)
    r = o.cln_bolt11_check(bytes(s), ctypes.c_size_t(len(s)), node.ctypes.data_as(p8), h.ctypes.data_as(p8), f, nf)
    return int(r), node.tobytes(), h.tobytes(), f.value.decode("utf-8", "replace"), nf.value.decode("utf-8", "replace")


def ref_recover(o, sig, recid, msg):
    out = np.zeros(33, np.uint8)
    r = o.cln_ecdsa_recover(bytes(sig), ctypes.c_int(int(recid)), bytes(msg), out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)))
    return int(r), out.tobytes()
