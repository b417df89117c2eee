"""The engine's fixed-base comb table, built with plain Python integers.

The table (verify.cuh SV_GT_*, built once per context by k_gtable_bases / k_gtable_fill) holds d * 2^(16 i) * G for 16 rows:
rows 0..14 hold d = 1..32768, row 15 holds d = 1..65536, entry e = row * 32768 + d - 1, 557,056 affine points in all.
Every verification adds u1*G (BIP-340: s*G) from it, one entry per non-zero signed 16-bit digit of u1 (sc_prepare_u1).

build() returns the whole table as (ENTRIES, 16) uint32: x then y, each as 8 little-endian 32-bit limbs, the layout of the
device's ge_mem and of SV_ST_ECMULT_GEN's output.  Each row is a chain of affine additions of its base; the 16 rows step
together so that one modular inversion serves all of them (Montgomery's trick), and row 15's upper half (d > 32768) runs as
a 17th chain from 32768 * B_15."""
import numpy as np

P = 2**256 - 2**32 - 977
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
G = (0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798,
     0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8)
ROW = 32768                     # SV_GT_ROW: entries of rows 0..14
TOP = 65536                     # entries of row 15
ROWS = 16
ENTRIES = 15 * ROW + TOP        # SV_GT_ENTRIES = 557,056
CARRY_SCALAR = 2**256 - 2**224  # windows 14 and 15 both 0xFFFF: digits (-1 at row 14, 65536 at row 15)


def entry(row, d):
    """index of d * 2^(16 row) * G"""
    assert 0 <= row < ROWS and 1 <= d <= (TOP if row == 15 else ROW), (row, d)
    return row * ROW + d - 1


def row_d(e):
    """(row, d) of entry e"""
    row = min(e // ROW, 15)
    return row, e - row * ROW + 1


def row_size(row):
    return TOP if row == 15 else ROW


def scalar_for(e):
    """the scalar whose comb digits read entry e: d * 2^(16 row), one non-zero digit.  Row 15's d = 65536 is not a window
    value: only the carry out of window 14 = 0xFFFF (digit -1) into window 15 = 0xFFFF reaches it, so its scalar
    2^256 - 2^224 also reads entry(14, 1), negated."""
    row, d = row_d(e)
    if row == 15 and d == TOP:
        return CARRY_SCALAR
    return d << (16 * row)


def digits_for(e):
    """the comb digits scalar_for(e) must recode to, as {row: digit}"""
    row, d = row_d(e)
    if row == 15 and d == TOP:
        return {14: -1, 15: TOP}
    return {row: d}


def _double(a):
    lam = 3 * a[0] * a[0] * pow(2 * a[1], -1, P) % P
    x = (lam * lam - 2 * a[0]) % P
    return x, (lam * (a[0] - x) - a[1]) % P


def bases():
    """B_i = 2^(16 i) * G, i = 0..15, by doubling"""
    out, b = [], G
    for _ in range(ROWS):
        out.append(b)
        for _ in range(16):
            b = _double(b)
    return out


def _chain_mul(k, a):
    """k * a for small k > 0 (double and add, affine)"""
    r = None
    for bit in bin(k)[2:]:
        if r is not None:
            r = _double(r)
        if bit == "1":
            r = a if r is None else _add(r, a)
    return r


def _add(a, b):
    lam = (b[1] - a[1]) * pow(b[0] - a[0], -1, P) % P
    x = (lam * lam - a[0] - b[0]) % P
    return x, (lam * (a[0] - x) - a[1]) % P


def build():
    """the whole table, (ENTRIES, 16) uint32 limbs: x then y, little-endian"""
    bs = bases()
    # chains: (first entry index, base, start point); chain c's k-th point (k = 0, 1, ...) is start + k * base
    chains = [(entry(r, 1), bs[r], bs[r]) for r in range(ROWS)]
    chains.append((entry(15, ROW + 1), bs[15], _chain_mul(ROW + 1, bs[15])))
    xs = [0] * ENTRIES
    ys = [0] * ENTRIES
    cur = [c[2] for c in chains]
    for (e0, _, _), pt in zip(chains, cur):
        xs[e0], ys[e0] = pt
    for k in range(1, ROW):
        # denominators of cur + base (k = 1 on the first 16 chains: cur == base, a doubling)
        dens = []
        for c, (e0, b, _) in enumerate(chains):
            a = cur[c]
            dens.append(2 * a[1] % P if a == b else (b[0] - a[0]) % P)
        pre = [0] * len(dens)
        acc = 1
        for i, v in enumerate(dens):
            acc = acc * v % P
            pre[i] = acc
        inv = pow(acc, -1, P)
        for i in range(len(dens) - 1, -1, -1):
            di = inv * pre[i - 1] % P if i else inv
            inv = inv * dens[i] % P
            e0, b, _ = chains[i]
            a = cur[i]
            if a == b:
                lam = 3 * a[0] * a[0] * di % P
            else:
                lam = (b[1] - a[1]) * di % P
            x = (lam * lam - a[0] - b[0]) % P
            y = (lam * (a[0] - x) - a[1]) % P
            cur[i] = (x, y)
            xs[e0 + k], ys[e0 + k] = x, y
    buf = b"".join(x.to_bytes(32, "little") + y.to_bytes(32, "little") for x, y in zip(xs, ys))
    return np.frombuffer(buf, dtype=np.uint32).reshape(ENTRIES, 16)


def point(table, e):
    """entry e of a limb table as an affine (x, y) pair of ints"""
    b = table[e].tobytes()
    return int.from_bytes(b[:32], "little"), int.from_bytes(b[32:], "little")


def scalar_limbs(scalars):
    """ints (< 2^256) -> (n, 8) uint32 little-endian limbs"""
    buf = b"".join(v.to_bytes(32, "little") for v in scalars)
    return np.frombuffer(buf, dtype=np.uint32).reshape(-1, 8).copy()
