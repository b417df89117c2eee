"""Generate tests/golden/bolt12_vectors.npz: BOLT12 TLV streams with keys, signatures and the reference's answers.

Needs a Core Lightning source tree ($CLN_SRC, else /root/reference) and oracle/_ref/libcln_bolt12.so (oracle/bolt12.mk).
Inputs are data only:
  * the lno/lni/lnr strings in the reference's tests, and a seeded sample of its fuzz corpora
    tests/fuzz/corpora/fuzz-bolt12-{invoice,invrequest,offer}-decode, bech32-decoded without checksum (well-formed and
    malformed streams alike);
  * for every well-formed stream, a BIP-340 signature (tests/ecc.py, seeded key) over the reference's sighash, and
    variants: a flipped byte in a signed field, a changed byte in a signature-range field, a wrong key, a flipped
    signature byte, the other messagename;
  * constructed edge cases of the TLV parse and of the tree's shape.
Every item's status (1 / 0 / -1), Merkle root and sighash come from the reference (oracle/bolt12_harness.c).

Arrays: blob, off, len (stream i = blob[off:off+len]); names (index into tests.bolt12.NAMES); xonly (n, 32); sig (n, 64);
status (int8); merkle, sighash (n, 32); label (uint8, LABELS below).
Run:  python -m tests.golden.make_bolt12
"""
import ctypes
import hashlib
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import bolt12, ecc  # noqa: E402

REF = os.environ.get("CLN_SRC", "/root/reference")
LABELS = ["signed", "flip_signed_field", "flip_signature_field", "wrong_key", "flip_sig", "other_name", "unsigned",
          "edge"]
L = {k: i for i, k in enumerate(LABELS)}
FUZZ_PER_CORPUS = 500


def _sk(i):
    return hashlib.sha256(b"tests/golden/make_bolt12 key %d" % i).digest()


class Gen:
    def __init__(self):
        self.lib = ctypes.CDLL(bolt12.LIB)
        self.items = []  # (stream, name index, xonly, sig, label)
        self.nkeys = 0

    def key(self):
        self.nkeys += 1
        sk = _sk(self.nkeys)
        return sk, ecc.pubkey_create(sk)[1][:32]

    def ref(self, stream, ni, x, s):
        m, h = np.zeros(32, np.uint8), np.zeros(32, np.uint8)
        p8 = ctypes.POINTER(ctypes.c_uint8)
        r = self.lib.cln_bolt12_check(bytes(stream), ctypes.c_size_t(len(stream)), bolt12.NAMES[ni][0], bolt12.NAMES[ni][1],
                                      bytes(x), bytes(s), m.ctypes.data_as(p8), h.ctypes.data_as(p8))
        return r, h.tobytes()

    def add(self, stream, ni, x, s, label):
        self.items.append((bytes(stream), ni, bytes(x), bytes(s), L[label]))

    def signed(self, stream, ni, label="signed", variants=True):
        """sign the reference's sighash; returns False if the reference refuses the stream"""
        sk, x = self.key()
        r, h = self.ref(stream, ni, x, bytes(64))
        if r < 0:
            self.add(stream, ni, x, hashlib.sha512(stream).digest(), "unsigned")
            return False
        sig, x2 = ecc.schnorr_sign(sk, h)
        assert x2 == x
        self.add(stream, ni, x, sig, label)
        if not variants:
            return True
        fields = bolt12.parse_fields(stream)
        signed_f = [f for f in fields if not (240 <= f[0] <= 1000) and f[2]]
        sigrange_f = [f for f in fields if 240 <= f[0] <= 1000 and f[2]]
        if signed_f:
            t, vo, v = signed_f[len(stream) % len(signed_f)]
            s2 = bytearray(stream)
            s2[vo + len(v) // 2] ^= 0x20
            self.add(s2, ni, x, sig, "flip_signed_field")
        if sigrange_f:
            t, vo, v = sigrange_f[0]
            s2 = bytearray(stream)
            s2[vo] ^= 0x01
            self.add(s2, ni, x, sig, "flip_signature_field")
        self.add(stream, ni, self.key()[1], sig, "wrong_key")
        s2 = bytearray(sig)
        s2[len(stream) % 64] ^= 0x04
        self.add(stream, ni, x, s2, "flip_sig")
        self.add(stream, 1 - ni, x, sig, "other_name")
        return True


def real_strings():
    out = set()
    pat = re.compile(r"ln[oir]1[qpzry9x8gf2tvdw0s3jn54khce6mua7l]{30,}")
    for d in ("tests", "common/test", "plugins/test", "devtools"):
        base = os.path.join(REF, d)
        for f in sorted(os.listdir(base)) if os.path.isdir(base) else []:
            if f.endswith((".py", ".c", ".json")):
                with open(os.path.join(base, f), errors="replace") as fh:
                    out.update(pat.findall(fh.read()))
    return sorted(out)


def fuzz_strings(rng):
    out = []
    for c in ("invoice", "invrequest", "offer"):
        d = os.path.join(REF, "tests", "fuzz", "corpora", f"fuzz-bolt12-{c}-decode")
        files = sorted(os.listdir(d))
        for f in rng.choice(files, size=min(FUZZ_PER_CORPUS, len(files)), replace=False):
            with open(os.path.join(d, f), "rb") as fh:
                out.append(fh.read().decode("latin-1"))
    return out


def edge_streams():
    r, bs = bolt12.record, bolt12.bigsize
    e = []
    # BigSize forms (common/bigsize.c): each non-minimal encoding, in the type and in the length, and the minimal ones
    for nm in (b"\xfd\x00\xfc", b"\xfd\x00\x00", b"\xfe\x00\x00\xff\xff", b"\xfe\x00\x00\x00\x01",
               b"\xff\x00\x00\x00\x00\xff\xff\xff\xff", b"\xff\x00\x00\x00\x00\x00\x00\x00\x01"):
        e.append(nm + b"\x01x")                       # non-minimal type
        e.append(b"\x01" + nm + b"x")                 # non-minimal length (and usually past the end)
    e.append(b"\xfd\x00\xfd\x01x")                      # minimal 0xfd form
    e.append(b"\xfe\x00\x01\x00\x00\x01x")              # minimal 0xfe form
    e.append(b"\xff\x00\x00\x00\x01\x00\x00\x00\x00\x01x")  # minimal 0xff form
    e.append(b"\x02\xfd\x00\xfd" + bytes(253))           # minimal 0xfd length
    # truncated type / truncated length / type without a length / length past the end
    e += [b"\xfd\x01", b"\xfe\x00\x01", b"\xff\x00\x00\x00\x01\x00", b"\x01\xfd\x00", b"\x01\xfe\x00\x01", b"\x01",
          r(0, b"ok") + b"\x03", b"\x01\x05abc", r(1, b"a") + b"\x02\x02b"]
    e.append(r(1, b"a") + r(1, b"b"))                   # duplicate type
    e.append(r(2, b"a") + r(1, b"b"))                   # descending types
    e.append(r(0, b"a") + r(0, b"a"))
    e.append(b"")                                         # empty stream
    e.append(r(0, b""))                                   # single field
    e.append(r(7, b"single"))
    e.append(r(240, bytes(64)) + r(1000, b""))            # signature fields only: all-zero root
    e.append(r(250, bytes(64)))
    e.append(r(500, b"first") + r(1001, b"a") + r(2000, b"b"))  # a signature-range field first: still the nonce source
    e.append(r(239, b"a") + r(240, b"b") + r(1000, b"c") + r(1001, b"d"))
    e.append(r(2**32, b"a") + r(2**64 - 2, b"b") + r(2**64 - 1, b"c"))  # 9-byte types up to 2^64 - 1
    e.append(r(0, bytes(range(100))) + r(2, b"x") + r(4, b"y"))  # first record longer than one SHA block
    e.append(r(1, bytes(55 - 2)) + r(3, bytes(56 - 2)) + r(5, bytes(64 - 3)))  # records at the padding boundaries
    for k in (2, 3, 5, 7, 31, 32, 33, 63, 64, 65, 100, 257):  # tree shapes, lane striding past 32 fields
        e.append(b"".join(r(2 * t + 1, bytes([t & 0xFF]) * (t % 5)) for t in range(k)))
    e.append(b"".join(r(t, b"") for t in range(5200)))    # more than 5,000 zero-length fields
    e.append(r(0, b"v") + r(9, bytes([0x5A]) * 70000))     # a value longer than 64 KiB
    e.append(bs(1) + bs(2**16 + 5) + bytes(10))            # a huge length past the end
    return e


def main():
    rng = np.random.default_rng(20260401)
    g = Gen()
    strings = [(s, True) for s in real_strings()] + [(s, False) for s in fuzz_strings(rng)]
    ok = bad = 0
    for s, _real in strings:
        d = bolt12.bech32_decode_nochk(s)
        if d is None:
            continue
        hrp, stream = d
        ni = 1 if hrp == "lnr" else 0
        if g.signed(stream, ni):
            ok += 1
        else:
            bad += 1
    for st in edge_streams():
        if g.signed(st, 0, label="edge", variants=False):
            g.add(st, 0, g.items[-1][2], bytes(64), "edge")  # the same stream with an all-zero signature
    # lay the streams out once each; variants that keep the bytes share the span
    where, blob = {}, bytearray()
    off, ln = [], []
    for st, *_ in g.items:
        if st not in where:
            where[st] = len(blob)
            blob += st
        off.append(where[st])
        ln.append(len(st))
    n = len(g.items)
    status = np.zeros(n, np.int8)
    merkle = np.zeros((n, 32), np.uint8)
    sighash = np.zeros((n, 32), np.uint8)
    p8 = ctypes.POINTER(ctypes.c_uint8)
    for i, (st, ni, x, s, _lab) in enumerate(g.items):
        status[i] = g.lib.cln_bolt12_check(st, ctypes.c_size_t(len(st)), bolt12.NAMES[ni][0], bolt12.NAMES[ni][1], x, s,
                                           merkle[i].ctypes.data_as(p8), sighash[i].ctypes.data_as(p8))
    np.savez_compressed(
        os.path.join(ROOT, "tests", "golden", "bolt12_vectors.npz"),
        blob=np.frombuffer(bytes(blob), np.uint8), off=np.array(off, np.uint64), len=np.array(ln, np.uint32),
        names=np.array([it[1] for it in g.items], np.uint8),
        xonly=np.frombuffer(b"".join(it[2] for it in g.items), np.uint8).reshape(n, 32),
        sig=np.frombuffer(b"".join(it[3] for it in g.items), np.uint8).reshape(n, 64),
        status=status, merkle=merkle, sighash=sighash, label=np.array([it[4] for it in g.items], np.uint8))
    print(f"{n} items from {ok} well-formed and {bad} refused decoded strings; status 1/0/-1: "
          f"{(status == 1).sum()}/{(status == 0).sum()}/{(status == -1).sum()}; blob {len(blob)} bytes")


if __name__ == "__main__":
    main()
