"""Generate tests/golden/bolt11_vectors.npz: BOLT11 invoices with Core Lightning's own answers.

Needs a Core Lightning source tree ($CLN_SRC, else /root/reference) and oracle/_ref/libcln_bolt11.so (oracle/bolt11.mk).

The corpus (seeded, so a re-run gives the same file):
  spec          the BOLT #11 example invoices (the strings of the reference's common/test/run-bolt11.c)
  signed        invoices signed here, without `n` (the key is recovered), of several sizes and amounts
  signed_n      the same with an `n` field;  upper: signed invoices in upper case
  recid_flip    the recovery id's parity bit flipped (another key is recovered; with `n` it is not read)
  recid23       recovery id 2 / 3 made valid: R.x in [n, p) chosen first, r = R.x - n
  recid_high    recovery ids 4..255;  r_s_range: r / s at n, above n and zero, with and without `n`
  high_s        s replaced by n - s (recovery accepts it, verification against `n` does not)
  off_curve     r with r^3 + 7 not a square;  recid2_overflow: recovery id 2 with r + n >= p
  n_wrong_len   a 52-word `n` (an unknown field: the key is recovered);  n_dup: a second `n` after a valid one, or a
                valid one after a wrong-length one;  n_bad_key: a 53-word `n` that is not a key;  n_trailing: its
                trailing bit set
  long          route hints, above 2,000 characters
  bech32m       the BECH32M constant;  nul: a NUL inside the span;  charset: bad characters, mixed case, no '1', short
  flip          one 5-bit word of one invoice changed in every region (hrp, timestamp, tag, length, data, signature),
                checksum recomputed, and one raw character flipped in every position (checksum not recomputed)
  trunc         every truncation of one invoice: raw prefixes, and word prefixes with the checksum recomputed
Each item records bolt11_decode's result (bit 0) and bolt11_decode_nosig's (bit 1), the receiver_id, the signing hash and
both failure messages.  recover_*: (signature, recovery id, message) triples with secp256k1_ecdsa_recover's answer,
including Q = infinity (s R = e G) and the refusals before any point arithmetic.
"""
import ctypes
import hashlib
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import bolt11, ecc  # noqa: E402

P, N = ecc.P, ecc.N
CHARSET = bolt11.CHARSET
REF = os.environ.get("CLN_SRC", "/root/reference")


def b32(x):
    return x.to_bytes(32, "big")


def polymod(values):
    gen = (0x3b6a57b2, 0x26508e6d, 0x1ea119fa, 0x3d4233dd, 0x2a1462b3)
    chk = 1
    for v in values:
        b = chk >> 25
        chk = ((chk & 0x1ffffff) << 5) ^ v
        for i in range(5):
            chk ^= gen[i] if (b >> i) & 1 else 0
    return chk


def encode(hrp, words, const=1):
    hv = [ord(c) >> 5 for c in hrp] + [0] + [ord(c) & 31 for c in hrp]
    pm = polymod(hv + list(words) + [0] * 6) ^ const
    chk = [(pm >> 5 * (5 - i)) & 31 for i in range(6)]
    return hrp + "1" + "".join(CHARSET[w] for w in list(words) + chk)


def to_words(data, nbits=None):
    nbits = 8 * len(data) if nbits is None else nbits
    v = int.from_bytes(data, "big") if data else 0
    nw = (nbits + 4) // 5
    v <<= 5 * nw - 8 * len(data)
    return [(v >> 5 * (nw - 1 - i)) & 31 for i in range(nw)]


def field(tag, words):
    n = len(words)
    return [CHARSET.index(tag), n >> 5, n & 31] + list(words)


def sign_recoverable(sk, h):
    d, z = int.from_bytes(sk, "big"), int.from_bytes(h, "big")
    ctr = 0
    while True:
        k = int.from_bytes(hashlib.sha256(b"make_bolt11 nonce" + sk + h + bytes([ctr])).digest(), "big") % N
        ctr += 1
        if not k:
            continue
        x, y = ecc.base_mult(k)
        r = x % N
        s = pow(k, -1, N) * (z + r * d) % N
        if not r or not s:
            continue
        recid = (y & 1) | (2 if x >= N else 0)
        if s > N // 2:
            s, recid = N - s, recid ^ 1
        return b32(r) + b32(s), recid


def sqrt_p(a):
    y = pow(a, (P + 1) // 4, P)
    return y if y * y % P == a % P else None


class Gen:
    def __init__(self, rng):
        self.rng = rng
        self.items = []  # (bytes, label)
        self.nk = 0

    def key(self):
        self.nk += 1
        sk = hashlib.sha256(b"make_bolt11 key %d" % self.nk).digest()
        return sk, ecc.pubkey_create(sk)[0]

    def rb(self, n):
        return bytes(self.rng.integers(0, 256, n, dtype=np.uint8))

    def fields(self, with_n=None, desc=b"coffee", hints=0, extra=()):
        f = field("p", to_words(self.rb(32))) + field("s", to_words(self.rb(32))) + field("d", to_words(desc))
        for _ in range(hints):  # r fields of 10 hops (51 bytes each)
            f += field("r", to_words(b"".join(self.key()[1] + self.rb(18) for _ in range(10))))
        if with_n is not None:
            f += field("n", to_words(with_n, 264))
        for e in extra:
            f += e
        return f

    def body(self, fields, ts=1496314658):
        return [(ts >> 5 * (6 - i)) & 31 for i in range(7)] + list(fields)

    def signed(self, hrp, words, sk, mutate=None):
        """-> (invoice str, signed words, sig64, recid)"""
        h = bolt11.signing_hash(hrp, words)
        sig, recid = sign_recoverable(sk, h)
        if mutate:
            sig, recid = mutate(sig, recid)
        return encode(hrp, words + to_words(sig + bytes([recid]))), words, sig, recid

    def add(self, s, label):
        self.items.append((s.encode() if isinstance(s, str) else bytes(s), label))


def build(rng):
    g = Gen(rng)
    src = open(os.path.join(REF, "common", "test", "run-bolt11.c")).read()
    for s in sorted(set(re.findall(r'"(ln[a-z0-9]*1[a-z0-9]+)"', src))):
        g.add(s, "spec")
    hrps = ["lnbc", "lnbc2500u", "lntb20m", "lnbcrt1", "lnbc10n", "lntbs1m"]
    base = None
    for i in range(120):
        sk, pub = g.key()
        hrp = hrps[i % len(hrps)]
        desc = g.rb(int(rng.integers(0, 300))) if i % 3 else b"1 cup coffee"
        with_n = i % 2 == 1
        hints_here = i % 4 == 0
        w = g.body(g.fields(pub if with_n else None, desc=desc, hints=hints_here))
        s, words, sig, recid = g.signed(hrp, w, sk)
        g.add(s, "signed_n" if with_n else "signed")
        if base is None and not with_n and not hints_here:
            base = (hrp, w, sk, s)
        if i % 5 == 0:
            g.add(s.upper(), "upper")
        flip = lambda sg, rc: (sg, rc ^ 1)  # noqa: E731
        g.add(g.signed(hrp, w, sk, flip)[0], "recid_flip")
        g.add(g.signed(hrp, w, sk, lambda sg, rc: (sg[:32] + b32(N - int.from_bytes(sg[32:], "big")), rc ^ 1))[0], "high_s")
    # recovery id 2 / 3: R.x in [n, p)
    for t in range(1, 4000):
        x = N + t
        if x >= P:
            break
        if sqrt_p(x ** 3 + 7) is None:
            continue
        for parity in (0, 1):
            sk, pub = g.key()
            hrp, w = "lnbc", g.body(g.fields(None))
            sg = b32(x - N) + b32(int.from_bytes(g.rb(32), "big") % N or 1)
            g.add(encode(hrp, w + to_words(sg + bytes([2 | parity]))), "recid23")
        if sum(1 for _, lab in g.items if lab == "recid23") >= 24:
            break
    hrp, w, sk, s0 = base
    _, _, sig0, recid0 = g.signed(hrp, w, sk)
    sk_n, pub_n = g.key()
    wn = g.body(g.fields(pub_n))
    _, _, sign, recidn = g.signed(hrp, wn, sk_n)

    def raw(words, sig, recid, label, const=1):
        g.add(encode(hrp, words + to_words(sig + bytes([recid])), const), label)

    for rc in range(4, 256):
        raw(w, sig0, rc, "recid_high")
        if rc % 16 == 4:
            raw(wn, sign, rc, "recid_high")
    r0, s0i = sig0[:32], sig0[32:]
    for words, sg in ((w, sig0), (wn, sign)):
        for rv in (N, N + 1, 2 ** 256 - 1, 0):
            raw(words, b32(rv) + sg[32:], 0, "r_s_range")
            raw(words, sg[:32] + b32(rv), 0, "r_s_range")
    for t in range(1, 200):
        if sqrt_p(t ** 3 + 7) is None:
            raw(w, b32(t) + s0i, 0, "off_curve")
            if sum(1 for _, lab in g.items if lab == "off_curve") >= 4:
                break
    for rv in (P - N, P - N + 1, N - 1):
        raw(w, b32(rv) + s0i, 2, "recid2_overflow")
    # `n` variants
    _, pub_other = g.key()
    w52 = g.body(g.fields(None, extra=[field("n", to_words(pub_n[:32]))]))  # 52 words
    g.add(g.signed(hrp, w52, sk)[0], "n_wrong_len")
    wdup = g.body(g.fields(pub_n, extra=[field("n", to_words(pub_other, 264))]))
    g.add(g.signed(hrp, wdup, sk_n)[0], "n_dup")
    wdup2 = g.body(g.fields(None, extra=[field("n", to_words(pub_other[:32])), field("n", to_words(pub_n, 264))]))
    g.add(g.signed(hrp, wdup2, sk_n)[0], "n_dup")
    bad_keys = [b"\x04" + pub_n[1:], b"\x02" + b32(P), b"\x02" + b32(5)]  # sqrt(5^3 + 7) does not exist
    for bk in bad_keys:
        g.add(g.signed(hrp, g.body(g.fields(bk)), sk_n)[0], "n_bad_key")
    wt = g.body(g.fields(None, extra=[field("n", to_words(pub_n, 264)[:-1] + [to_words(pub_n, 264)[-1] | 1])]))
    g.add(g.signed(hrp, wt, sk_n)[0], "n_trailing")
    # long invoices: route hints
    for hints in (4, 6, 8):
        sk2, pub2 = g.key()
        w2 = g.body(g.fields(pub2 if hints == 6 else None, hints=hints))
        g.add(g.signed("lnbc1m", w2, sk2)[0], "long")
    # BECH32M, NUL, charset
    raw(w, sig0, recid0, "bech32m", const=0x2bc830a3)
    s_ok = encode(hrp, w + to_words(sig0 + bytes([recid0])))
    g.add(s_ok.encode() + b"\x00garbage", "nul")
    g.add(s_ok.encode()[:40] + b"\x00" + s_ok.encode()[41:], "nul")
    for bad in (s_ok[:7], s_ok.replace("1", "b", 1)[:5], s_ok[:20] + "b" + s_ok[21:], s_ok[:10] + s_ok[10:].upper(),
                "lnbc1" + "q" * 5, "\x7f" + s_ok[1:], s_ok.replace("lnbc", "ln bc"), "1" + "q" * 10):
        g.add(bad, "charset")
    g.add(s_ok.encode()[:30] + b"\xc3" + s_ok.encode()[31:], "charset")
    # flips in every region (checksum recomputed), and raw character flips (checksum not recomputed)
    sigw = to_words(sig0 + bytes([recid0]))
    allw = w + sigw
    for k in range(len(allw)):
        for bit in (1, 16):
            ww = list(allw)
            ww[k] ^= bit
            g.add(encode(hrp, ww), "flip")
    for k in range(len(hrp)):
        g.add(encode(hrp[:k] + chr(ord(hrp[k]) ^ 1) + hrp[k + 1:], allw), "flip")
    for k in range(len(s_ok)):
        c = s_ok[k]
        c2 = CHARSET[CHARSET.index(c) ^ 1] if c in CHARSET else chr(ord(c) ^ 1)
        g.add(s_ok[:k] + c2 + s_ok[k + 1:], "flip")
    for k in range(len(s_ok)):
        g.add(s_ok[:k], "trunc")
    for k in range(len(allw)):
        g.add(encode(hrp, allw[:k]), "trunc")
    return g


def recover_vectors(rng):
    """(sig64, recid, msg32) triples for secp256k1_ecdsa_recover directly"""
    out = []
    for i in range(200):
        sk = hashlib.sha256(b"make_bolt11 rec %d" % i).digest()
        msg = hashlib.sha256(b"make_bolt11 msg %d" % i).digest()
        sig, recid = sign_recoverable(sk, msg)
        out.append((sig, recid if i % 7 else recid ^ 1, msg))
    for i in range(8):  # Q = infinity: R = k G and e = s k, so s R = e G
        k = 12345 + 1000 * i
        x, y = ecc.base_mult(k)
        s = (777 + i) % N
        e = s * k % N
        out.append((b32(x % N) + b32(s), (y & 1) | (2 if x >= N else 0), b32(e)))
    m = hashlib.sha256(b"m").digest()
    for r, s, rc in ((0, 5, 0), (5, 0, 0), (N, 5, 0), (5, N, 0), (P - N, 5, 2), (P - N - 1, 5, 3), (1, 1, 0), (2, 3, 1)):
        out.append((b32(r) + b32(s), rc, m))
    return out


def main():
    rng = np.random.default_rng(20261018)
    g = build(rng)
    lib = ctypes.CDLL(bolt11.LIB)
    blob, off, ln = bytearray(), [], []
    n = len(g.items)
    ret = np.zeros(n, np.int8)
    node = np.zeros((n, 33), np.uint8)
    h = np.zeros((n, 32), np.uint8)
    fail, nfail = [], []
    for i, (s, _) in enumerate(g.items):
        off.append(len(blob))
        ln.append(len(s))
        blob += s
        f, nf = ctypes.create_string_buffer(256), ctypes.create_string_buffer(256)
        ret[i] = lib.cln_bolt11_check(s, ctypes.c_size_t(len(s)), node[i].ctypes.data, h[i].ctypes.data, f, nf)
        fail.append(f.value.decode("utf-8", "replace"))
        nfail.append(nf.value.decode("utf-8", "replace"))
    rv = recover_vectors(rng)
    rsig = np.frombuffer(b"".join(v[0] for v in rv), np.uint8).reshape(-1, 64)
    rrec = np.array([v[1] for v in rv], np.int32)
    rmsg = np.frombuffer(b"".join(v[2] for v in rv), np.uint8).reshape(-1, 32)
    rok = np.zeros(len(rv), np.int8)
    rkey = np.zeros((len(rv), 33), np.uint8)
    for i, (sg, rc, m) in enumerate(rv):
        rok[i] = lib.cln_ecdsa_recover(sg, rc, m, rkey[i].ctypes.data)
    labels = sorted({lab for _, lab in g.items})
    np.savez_compressed(
        bolt11.FIXTURE, blob=np.frombuffer(bytes(blob), np.uint8), off=np.array(off, np.uint64), len=np.array(ln, np.uint32),
        ret=ret, node=node, hash=h, fail=np.array(fail), nosig_fail=np.array(nfail), labels=np.array(labels),
        label=np.array([labels.index(lab) for _, lab in g.items], np.uint8),
        recover_sig=rsig, recover_recid=rrec, recover_msg=rmsg, recover_ok=rok, recover_key=rkey)
    st = bolt11.expected_status(ret, np.array(fail), np.array(labels)[[labels.index(lab) for _, lab in g.items]])
    print(f"{n} invoices, blob {len(blob)} bytes; expected status 1/0/-1/unchecked: {(st == 1).sum()}/{(st == 0).sum()}/"
          f"{(st == -1).sum()}/{(st == bolt11.UNCHECKED).sum()}; {len(rv)} recovery vectors, {rok.sum()} recover")


if __name__ == "__main__":
    main()
