"""Adversarial-but-VALID signatures with prescribed (u1, u2), built with plain Python integers.

An attacker who knows the private key controls both scalars of the verification equation
R = u1*G + u2*Q (choose R, solve for s and the message hash).  These inputs steer the fixed-window
ladder and the comb through their exceptional branches (accumulator == +-table point, infinity,
zero digits, top-window carries, GLV lattice vectors ...), where a verifier that mishandles a case
would wrongly reject a signature the reference accepts."""
import numpy as np

P = 2**256 - 2**32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72


def inv(x, m=P):
    return pow(x, -1, m)  # x != 0 mod m: the same value as x^(m-2), eight times faster


def add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    if a[0] == b[0]:
        if (a[1] + b[1]) % P == 0:
            return None
        l = 3 * a[0] * a[0] * inv(2 * a[1]) % P
    else:
        l = (b[1] - a[1]) * inv(b[0] - a[0]) % P
    x = (l * l - a[0] - b[0]) % P
    return (x, (l * (a[0] - x) - a[1]) % P)


def mul(k, pt):
    k %= N
    r = None
    while k:
        if k & 1:
            r = add(r, pt)
        pt = add(pt, pt)
        k >>= 1
    return r


G = (GX, GY)


def craft(d, u1, u2, exact=False, r_if_infinity=None):
    """Return (msg32, pub33, pubxy, sig64) of a signature that verifies with scalars (+-u1, +-u2), or None.

    exact: the verifier must see exactly (u1, u2): None instead of negating both when s would be high.
    r_if_infinity: when u1*G + u2*Q is infinity, sign with this r instead (an invalid signature whose verification
    still runs with exactly these scalars)."""
    u1 %= N
    u2 %= N
    if u2 == 0 or d % N == 0:
        return None
    Q = mul(d, G)
    R = mul((u1 + u2 * d) % N, G)
    if R is None and r_if_infinity is None:
        return None
    r = R[0] % N if R is not None else r_if_infinity % N
    if r == 0:
        return None
    s = r * inv(u2, N) % N
    if s > N // 2:  # negating both scalars keeps x(R) and flips s
        if exact:
            return None
        s = N - s
        u1 = (N - u1) % N
    m = u1 * s % N
    b = lambda v: np.frombuffer(v.to_bytes(32, "big"), dtype=np.uint8)
    pub33 = np.concatenate([np.array([2 + (Q[1] & 1)], np.uint8), b(Q[0])])
    return b(m).copy(), pub33, np.concatenate([b(Q[0]), b(Q[1])]), np.concatenate([b(r), b(s)])


def special_scalars():
    a1 = 0x3086D221A7D46BCDE86C90E49284EB15
    b1 = 0xE4437ED6010E88286F547FA90ABFE4C3
    a2 = 0x114CA50F7A8E2F3F657C1108D9D44CFD8
    vals = [0, 1, 2, 3, 4, 7, 8, 15, 16, 17, 31, 32, 33, N - 1, N - 2, N - 3, (N - 1) // 2, (N + 1) // 2,
            LAMBDA, LAMBDA + 1, LAMBDA - 1, N - LAMBDA, 2 * LAMBDA % N, a1, b1, a2, N - a1, N - b1,
            (a1 + b1 * LAMBDA) % N, 2**128, 2**128 - 1, 2**128 + 1, 2**127, 2**129, 2**255, 2**255 - 1,
            0x8000, 0x8001, 0x7FFF, 0xFFFF, 0x10000, 0x80000000, 0xFFFF << 240, 0x8000 << 240, (0x8000 << 224) - 1,
            int("8000" * 16, 16) % N, int("7FFF" * 16, 16), int("8001" * 16, 16) % N, int("F" * 64, 16) % N,
            int("1" * 64, 16), int("8" * 64, 16) % N]
    return vals


def cases(limit=None):
    """(msg32[n,32], pub33[n,33], pubxy[n,64], sig[n,64]) arrays of crafted signatures."""
    sc = special_scalars()
    out = []
    ds = [1, 2, 3, 5, N - 1, N - 2, (N + 1) // 2, LAMBDA, 0xDEADBEEFCAFEBABE0123456789ABCDEF]
    for di, d in enumerate(ds):
        for i, u2 in enumerate(sc):
            for j, u1 in enumerate(sc):
                if (i + 2 * j + di) % (3 if di < 4 else 11):  # thin the cross product deterministically
                    continue
                c = craft(d, u1, u2)
                if c is not None:
                    out.append(c)
    # collisions inside the ladder: u2 small multiples with Q = G so that u1*G and u2*Q cancel or coincide
    for u in range(1, 40):
        for d in (1, 2, N - 1):
            for u1 in (u, N - u, (u * d) % N, (N - u * d) % N, (2 * u * d) % N):
                c = craft(d, u1, u)
                if c is not None:
                    out.append(c)
    if limit:
        out = out[:limit]
    cols = list(zip(*out))
    return tuple(np.stack(c) for c in cols)


BETA = 0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE  # lambda*(x, y) = (beta*x, y)


def _schnorr_sign_nonce(d0, k0, msg32):
    """BIP-340 signature of msg32 under secret d0 with the nonce k0 chosen by the caller (both negated as BIP-340 requires
    when their point has odd y) -> (sig64, xonly32).  k0 = d0 gives R = P."""
    from tests import ecc
    x, y = ecc.base_mult(d0)
    d = d0 if y % 2 == 0 else N - d0
    rx, ry = (x, y) if k0 == d0 else ecc.base_mult(k0)
    k = k0 if ry % 2 == 0 else N - k0
    px = x.to_bytes(32, "big")
    e = int.from_bytes(ecc.tagged_hash("BIP0340/challenge", rx.to_bytes(32, "big") + px + bytes(msg32)), "big") % N
    return rx.to_bytes(32, "big") + ((k + e * d) % N).to_bytes(32, "big"), px


def bip340_collision_groups(size=1024):
    """Four all-valid groups of `size` BIP-340 signatures whose points meet inside the buckets of batch verification
    (batch.cuh: every R_i, lambda*R_i, P_i, lambda*P_i enters a bucket; equal points there need a doubling, opposite ones
    give infinity):
      copies  one signature repeated
      onekey  one key, a fresh message and nonce per signature
      r_eq_p  nonce = key, so R = P
      r_eq_lp nonce = lambda*key, so R = lambda*P = (beta*x, y): even y, since P has it
    Returns [(name, msg (size, 32), xonly (size, 32), sig (size, 64))], deterministic."""
    import hashlib
    h = lambda *a: int.from_bytes(hashlib.sha256(b"/".join(str(v).encode() for v in a)).digest(), "big") % N or 1
    m32 = lambda *a: hashlib.sha256(b"msg/" + b"/".join(str(v).encode() for v in a)).digest()
    out = []

    def pack(name, rows):
        msg = np.array([np.frombuffer(m, np.uint8) for m, _, _ in rows])
        key = np.array([np.frombuffer(k, np.uint8) for _, k, _ in rows])
        sig = np.array([np.frombuffer(s, np.uint8) for _, _, s in rows])
        out.append((name, msg, key, sig))
    s, px = _schnorr_sign_nonce(h("copies"), h("copies", "k"), m32("copies"))
    pack("copies", [(m32("copies"), px, s)] * size)
    rows = []
    for i in range(size):
        s, px = _schnorr_sign_nonce(h("onekey"), h("onekey", i), m32("onekey", i))
        rows.append((m32("onekey", i), px, s))
    pack("onekey", rows)
    rows = []
    for i in range(size):
        d = h("r_eq_p", i)
        s, px = _schnorr_sign_nonce(d, d, m32("r_eq_p", i))
        assert s[:32] == px
        rows.append((m32("r_eq_p", i), px, s))
    pack("r_eq_p", rows)
    rows = []
    for i in range(size):
        d = h("r_eq_lp", i)
        s, px = _schnorr_sign_nonce(d, LAMBDA * d % N, m32("r_eq_lp", i))
        assert int.from_bytes(s[:32], "big") == BETA * int.from_bytes(px, "big") % P
        rows.append((m32("r_eq_lp", i), px, s))
    pack("r_eq_lp", rows)
    return out


# ---- soundness of BIP-340 batch verification: invalid signatures that cancel in a group equation -------------------------
# A group of the batch (batch.cuh) passes iff  sum a_i*R_i + sum (a_i*e_i)*P_i - (sum a_i*s_i)*G == infinity.  A BIP-340
# signature has exactly one valid s for its (r, P, m), so moving s_i by d_i makes it invalid and adds -a_i*d_i*G to its
# group's sum: a group whose only damage is such shifts passes iff sum a_i*d_i == 0 (mod n).  The random coefficients a_i
# are what keeps invalid signatures from cancelling; the helpers below build signatures that cancel when a_i are weaker
# than they should be (all equal, predictable, or derived from the wrong index).

BATCH_GROUP = 1024  # SV_SB_GROUP: signatures per group equation


def batch_coefficient(seed32, i):
    """a_i of signature i (its index in the WHOLE batch) as sb_prepare (batch.cuh) derives it: W0..W7 = SHA-256(seed32 ||
    LE64(i)) as big-endian 32-bit words, alpha = (W1 << 32 | W0) | 1, beta = W3 << 32 | W2, a_i = alpha + beta*lambda mod n."""
    import hashlib
    import struct
    w = struct.unpack(">8I", hashlib.sha256(bytes(seed32) + int(i).to_bytes(8, "little")).digest())
    return (((w[1] << 32 | w[0]) | 1) + (w[3] << 32 | w[2]) * LAMBDA) % N


def _shift_s(sig, i, d):
    s = int.from_bytes(bytes(sig[i, 32:]), "big")
    sig[i, 32:] = np.frombuffer(((s + d) % N).to_bytes(32, "big"), np.uint8)


def forge_pair(sig, i, j, seed32, d=1):
    """Copy of the (n, 64) signatures with s_i += d*a_j and s_j -= d*a_i (mod n), a = batch_coefficient(seed32, .): two
    invalid signatures whose shifts cancel, -a_i*d*a_j + a_j*d*a_i = 0, in a batch verified with seed32 when i and j share
    a group."""
    out = sig.copy()
    _shift_s(out, i, d * batch_coefficient(seed32, j))
    _shift_s(out, j, -d * batch_coefficient(seed32, i))
    return out


def cancel_pair(sig, i, j, d=1):
    """Copy of the (n, 64) signatures with s_i += d and s_j -= d (mod n): invalid signatures that cancel whenever a_i = a_j."""
    out = sig.copy()
    _shift_s(out, i, d)
    _shift_s(out, j, -d)
    return out


def s_shifts(sig0, sig1):
    """{i: (s1_i - s0_i) mod n} over the rows where two (n, 64) signature arrays differ in s only."""
    rows = np.nonzero((sig0 != sig1).any(axis=1))[0]
    out = {}
    for i in rows:
        assert np.array_equal(sig0[i, :32], sig1[i, :32]), "r differs: not an s shift"
        out[int(i)] = (int.from_bytes(bytes(sig1[i, 32:]), "big") - int.from_bytes(bytes(sig0[i, 32:]), "big")) % N
    return out


def predict_groups(n, seed32, shifts):
    """Per-group verdicts of a batch of n signatures, valid but for the s shifts {i: d_i}, verified with seed32: group g
    passes iff sum over its members of a_i*d_i == 0 (mod n)."""
    acc = [0] * ((n + BATCH_GROUP - 1) // BATCH_GROUP)
    for i, d in shifts.items():
        acc[i // BATCH_GROUP] += batch_coefficient(seed32, i) * d
    return [int(a % N == 0) for a in acc]


def swap_nonce_pair(msg, xonly, sig, i, j):
    """Copies of (msg (n, 32), xonly (n, 32), sig (n, 64)) with items i and j replaced by two signatures under fresh keys,
    each made with the OTHER one's nonce point: item i is (r_j, k_i + H(r_j || P_i || m_i)*d_i), likewise item j.  Item i
    is off by R_i - R_j and item j by R_j - R_i, so together they add (a_i - a_j)*(R_i - R_j) to their group's sum:
    nothing when a_i = a_j.  Deterministic in (i, j)."""
    import hashlib
    from tests import ecc
    h = lambda *a: int.from_bytes(hashlib.sha256(b"swap/" + b"/".join(str(v).encode() for v in a)).digest(), "big") % N or 1
    side = []
    for t in (i, j):
        d0, k0 = h(i, j, t, "key"), h(i, j, t, "nonce")
        x, y = ecc.base_mult(d0)
        rx, ry = ecc.base_mult(k0)
        m = hashlib.sha256(b"swap/msg/%d/%d/%d" % (i, j, t)).digest()
        side.append((d0 if y % 2 == 0 else N - d0, k0 if ry % 2 == 0 else N - k0, x.to_bytes(32, "big"), rx.to_bytes(32, "big"), m))
    msg, xonly, sig = msg.copy(), xonly.copy(), sig.copy()
    for t, (d, k, px, _, m), other in ((i, side[0], side[1]), (j, side[1], side[0])):
        r = other[3]
        e = int.from_bytes(ecc.tagged_hash("BIP0340/challenge", r + px + m), "big") % N
        msg[t] = np.frombuffer(m, np.uint8)
        xonly[t] = np.frombuffer(px, np.uint8)
        sig[t] = np.frombuffer(r + ((k + e * d) % N).to_bytes(32, "big"), np.uint8)
    return msg, xonly, sig


def by_key():
    """The committed fixture grouped by signing key: [(pub33, pubxy, indices)], one entry per key."""
    msg, pub33, pubxy, sig = load()
    keys, first, inv = np.unique(pub33, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    return [(pub33[f], pubxy[f], np.nonzero(inv == g)[0]) for g, f in enumerate(first)]


FIXTURE = __import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "golden", "adversarial.npz")


def load():
    """The committed fixture (generated by `python -m tests.adversarial`; pure-Python EC maths takes minutes)."""
    z = np.load(FIXTURE)
    return z["msg"], z["pub33"], z["pubxy"], z["sig"]


if __name__ == "__main__":
    m, p33, pxy, s = cases()
    keep = np.arange(m.shape[0]) % 3 == 0  # thin to ~1600 cases
    np.savez_compressed(FIXTURE, msg=m[keep], pub33=p33[keep], pubxy=pxy[keep], sig=s[keep])
    print("wrote", FIXTURE, int(keep.sum()), "cases")
