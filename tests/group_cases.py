"""Group-law self-test cases: the point operations and multiplication schedules of the engine, one at a time, against
plain Python integers.

Run on the GPU through the C ABI by tests/test_gpu_group.py (sv_selftest_group_host -> k_selftest_group) and, at reduced
sizes, on the host build of the same headers by tests/test_group_emul.py.  The reference is affine arithmetic on
y^2 = x^3 + b: the formulas of ge.cuh never use b, so points are drawn from secp256k1 and from curves y^2 = x^3 + 7c^3
for random c (the isomorphic curve of the flows without the square root, or its twist when c is a non-residue).
Jacobian inputs are converted by exact division; outputs are compared modulo p, whatever weak form the engine left.

Cases (every record of an op runs the production function unchanged, see selftest_group_item in selftest.cuh):
  * random Z, Z = 1, Z = p - 1, and coordinates in the weak range [p, 2^256);
  * a == b, a == -b, either operand at infinity, a doubling of infinity;
  * gej_add_ge's rzr: H in the generic case, 2Y when it doubles, 0 when the sum is infinity, and always Z3 = Z1 * rzr;
  * gej_add_gej with r aliasing a and r aliasing b;
  * ge_set_xo on residues and non-residues, x = 0, both parities;
  * the odd-multiples table, both ladders, the comb (added onto a point and from infinity), the whole ecmult_ladder and
    the linear form of the flows without the square root.
The hit count of every branch is written to $SV_SELFTEST_COVERAGE_DIR/group_coverage.json when that is set."""
import random

import numpy as np

from tests import ecc
from tests import group_schedule as S

P, N = ecc.P, ecc.N
BETA = S.BETA
LAMBDA = S.LAMBDA
IN_WORDS, OUT_WORDS = 64, 200
OPS = dict(GEJ_DOUBLE=0, GEJ_ADD_GE=1, GEJ_ADD_GEJ=2, GE_SET_XO=3, QTABLE_BUILD=4, ECMULT_LADDER_Q=5, ECMULT_HALF_LADDER=6,
           ECMULT_COMB_ADD=7, SMALL_COMB=8, ECMULT_LADDER=9, NS_LINEAR_FORM=10)
COVERAGE = {}
INF = None


def hit(key, k=1):
    COVERAGE[key] = COVERAGE.get(key, 0) + k


# ---- plain affine arithmetic on y^2 = x^3 + b (b never enters) ---------------------------------------------------------
def neg(a):
    return None if a is None else (a[0], (-a[1]) % P)


def add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    if a[0] == b[0]:
        if (a[1] + b[1]) % P == 0:
            return None
        lam = 3 * a[0] * a[0] * pow(2 * a[1], -1, P) % P
    else:
        lam = (b[1] - a[1]) * pow(b[0] - a[0], -1, P) % P
    x = (lam * lam - a[0] - b[0]) % P
    return x, (lam * (a[0] - x) - a[1]) % P


def endo(a):
    return None if a is None else (BETA * a[0] % P, a[1])


def mul(k, a):
    """k * a for any integer k (negative allowed), through Jacobian coordinates"""
    if a is None or k == 0:
        return None
    if k < 0:
        k, a = -k, neg(a)
    J = (0, 1, 0)
    for bit in bin(k)[2:]:
        J = ecc._jdouble(*J)
        if bit == "1":
            J = ecc._jadd_affine(*J, *a)
    return ecc._affine(*J)


def aff(X, Y, Z):
    zi = pow(Z % P, -1, P)
    return X * zi * zi % P, Y * zi * zi * zi % P


def jac(a, Z):
    return a[0] * Z * Z % P, a[1] * Z * Z * Z % P, Z % P


def random_point(rnd, b=7, small_x=False):
    while True:
        x = rnd.randrange(1 << 30) if small_x else rnd.randrange(P)
        c = (x * x * x + b) % P
        y = pow(c, (P + 1) // 4, P)
        if y * y % P == c:
            return x, (y if rnd.random() < 0.5 else P - y)


def random_curve(rnd):
    """b of secp256k1 or of y^2 = x^3 + 7c^3 for a random c"""
    if rnd.random() < 0.5:
        return 7
    c = rnd.randrange(1, P)
    return 7 * c * c * c % P


def weak(v, rnd):
    """v or, when it fits, the same residue in the weak range [p, 2^256)"""
    return v + P if v + P < 2**256 and rnd.random() < 0.5 else v


def random_z(rnd):
    r = rnd.random()
    if r < 0.1:
        return 1
    if r < 0.2:
        return P - 1
    if r < 0.3:
        return rnd.randrange(1, 1 << 32)  # leaves room for the weak form
    return rnd.randrange(1, P)


# ---- records -----------------------------------------------------------------------------------------------------------
def put(rec, off, v, words=8):
    for k in range(words):
        rec[off + k] = (v >> (32 * k)) & 0xFFFFFFFF


def get(out, off, words=8):
    v = 0
    for k in range(words):
        v |= int(out[off + k]) << (32 * k)
    return v


def put_jac(rec, off, pt, Z, rnd):
    """pt (affine or None) at Jacobian Z; infinity carries arbitrary coordinates"""
    if pt is None:
        put(rec, off, rnd.getrandbits(256))
        put(rec, off + 8, rnd.getrandbits(256))
        put(rec, off + 16, rnd.getrandbits(256))
        rec[off + 24] = 1
        return
    X, Y, Zm = jac(pt, Z)
    put(rec, off, weak(X, rnd))
    put(rec, off + 8, weak(Y, rnd))
    put(rec, off + 16, weak(Zm, rnd))
    rec[off + 24] = 0


def get_jac(out, off=0):
    if out[off + 24]:
        return None
    X, Y, Z = get(out, off), get(out, off + 8), get(out, off + 16)
    assert Z % P, "finite result with Z == 0"
    return aff(X, Y, Z)


def new_records(n):
    return np.zeros((n, IN_WORDS), dtype=np.uint32)


def put_work(rec, k1, k2, u1=0):
    """k1, k2 signed (|k| < 2^131) in the sign/magnitude words of the work record; u1 < n"""
    for off, k in ((32, k1), (40, k2)):
        put(rec, off, abs(k) | ((1 << 159) if k < 0 else 0), 5)
    put(rec, 48, u1)


# ---- the point operations ----------------------------------------------------------------------------------------------
def point_pairs(rnd, n):
    """(a, b, label) with a, b on a common curve: random pairs, then a == b, a == -b, infinities, all in equal shares"""
    out = []
    for i in range(n):
        b_ = random_curve(rnd)
        small = rnd.random() < 0.15
        p1 = random_point(rnd, b_, small)
        kind = i % 8
        if kind == 0 or kind == 1 or kind == 2:
            p2, lab = random_point(rnd, b_, rnd.random() < 0.15), "generic"
        elif kind == 3:
            p2, lab = p1, "equal"
        elif kind == 4:
            p2, lab = neg(p1), "opposite"
        elif kind == 5:
            p1, p2, lab = None, random_point(rnd, b_), "a_inf"
        elif kind == 6:
            p2, lab = None, "b_inf"
        else:
            p1, p2, lab = None, None, "both_inf"
        out.append((p1, p2, lab))
    return out


def case_gej_double(engine, n=100_000, seed=31):
    rnd = random.Random(seed)
    recs = new_records(n)
    pts = []
    for i in range(n):
        b_ = random_curve(rnd)
        p = None if i % 10 == 0 else random_point(rnd, b_, rnd.random() < 0.15)
        put_jac(recs[i], 0, p, random_z(rnd), rnd)
        pts.append(p)
    out = engine.selftest_group(OPS["GEJ_DOUBLE"], recs)
    for i, p in enumerate(pts):
        want = add(p, p)
        assert get_jac(out[i]) == want, ("gej_double", i, p)
        hit("gej_double." + ("infinity" if p is None else "finite"))


def case_gej_add_ge(engine, n=100_000, seed=32):
    rnd = random.Random(seed)
    pairs = [pp for pp in point_pairs(rnd, 2 * n) if pp[1] is not None][:n]
    recs = new_records(len(pairs))
    zs = []
    for i, (p1, p2, _) in enumerate(pairs):
        z = random_z(rnd)
        zs.append(z)
        put_jac(recs[i], 0, p1, z, rnd)
        put(recs[i], 32, weak(p2[0], rnd))
        put(recs[i], 40, weak(p2[1], rnd))
        recs[i, 60] = i & 1  # every other record: r aliases a
    out = engine.selftest_group(OPS["GEJ_ADD_GE"], recs)
    for i, (p1, p2, lab) in enumerate(pairs):
        want = add(p1, p2)
        got = get_jac(out[i])
        assert got == want, ("gej_add_ge", lab, i)
        rzr = get(out[i], 32) % P
        if p1 is not None:
            X1, Y1, Z1 = jac(p1, zs[i])
            if p1[0] != p2[0]:
                branch = "generic"
                assert rzr == (p2[0] * Z1 * Z1 - X1) % P, ("rzr != H", i)
            elif want is not None:
                branch = "double"
                assert rzr == 2 * Y1 % P, ("rzr != 2Y", i)
            else:
                branch = "infinity"
                assert rzr == 0, ("rzr != 0", i)
            if want is not None:
                assert get(out[i], 16) % P == Z1 * rzr % P, ("Z3 != Z1 * rzr", branch, i)
        else:
            branch = "a_inf"
        hit("gej_add_ge." + branch)
        hit("gej_add_ge.alias_a." + branch, i & 1)


def case_gej_add_gej(engine, n=100_000, seed=33):
    rnd = random.Random(seed)
    pairs = point_pairs(rnd, n)
    recs = new_records(n)
    for i, (p1, p2, _) in enumerate(pairs):
        put_jac(recs[i], 0, p1, random_z(rnd), rnd)
        put_jac(recs[i], 32, p2, random_z(rnd), rnd)
        recs[i, 60] = i % 3  # r separate, r aliases a, r aliases b
    out = engine.selftest_group(OPS["GEJ_ADD_GEJ"], recs)
    for i, (p1, p2, lab) in enumerate(pairs):
        assert get_jac(out[i]) == add(p1, p2), ("gej_add_gej", lab, ("separate", "alias a", "alias b")[i % 3], i)
        branch = {"equal": "double", "opposite": "infinity"}.get(lab, lab)
        hit("gej_add_gej." + branch)
        hit("gej_add_gej." + ("separate", "alias_a", "alias_b")[i % 3] + "." + branch)


def case_ge_set_xo(engine, n=100_000, seed=34):
    rnd = random.Random(seed)
    xs = [0, 1, 2, 3, 7, P - 1, P - 7] + [rnd.randrange(P) for _ in range(n - 7)]
    recs = new_records(len(xs))
    for i, x in enumerate(xs):
        put(recs[i], 0, x)
        recs[i, 8] = i & 1
    out = engine.selftest_group(OPS["GE_SET_XO"], recs)
    for i, x in enumerate(xs):
        c = (x * x * x + 7) % P
        res = pow(c, (P - 1) // 2, P) == 1 or c == 0
        assert int(out[i, 16]) == res, ("ge_set_xo residue flag", hex(x))
        assert get(out[i], 0) % P == x
        if res:
            y = get(out[i], 8) % P
            assert y * y % P == c and y % 2 == (i & 1), ("ge_set_xo root / parity", hex(x))
        hit("ge_set_xo." + ("residue" if res else "non_residue") + (".odd" if i & 1 else ".even"))


def case_qtable_build(engine, n=3000, seed=35):
    rnd = random.Random(seed)
    qs = [random_point(rnd, random_curve(rnd), rnd.random() < 0.1) for _ in range(n)]
    recs = new_records(n)
    for i, q in enumerate(qs):
        put(recs[i], 0, q[0])
        put(recs[i], 8, q[1])
    out = engine.selftest_group(OPS["QTABLE_BUILD"], recs)
    for i, q in enumerate(qs):
        zc = get(out[i], 192) % P
        m = q
        q2 = add(q, q)
        for e in range(8):
            X, Y, H = get(out[i], 24 * e), get(out[i], 24 * e + 8), get(out[i], 24 * e + 16)
            assert aff(X, Y, zc) == m, ("qtable entry", e, i)
            assert H % P == BETA * X % P, ("qtable beta*x slot", e, i)
            m = add(m, q2)
    hit("qtable_build.tables", n)


# ---- schedules ---------------------------------------------------------------------------------------------------------
def ladder_inputs(rnd, n, crafted=()):
    """(Q, k1, k2): random u2 through the engine's recoding, random odd halves, and the crafted ladder cases"""
    out = list(crafted)
    while len(out) < n:
        b_ = 7 if rnd.random() < 0.7 else random_curve(rnd)
        q = random_point(rnd, b_)
        if rnd.random() < 0.5:
            k1, k2 = S.prepare_u2(rnd.randrange(1, N))
        else:
            k1, k2 = [rnd.getrandbits(rnd.choice((5, 64, 128, 131))) | 1 for _ in range(2)]
            k1, k2 = k1 * rnd.choice((1, -1)), k2 * rnd.choice((1, -1))
        out.append((q, k1, k2))
    return out[:max(n, len(crafted))]


def case_ladders(engine, n=2000, seed=36, crafted=()):
    """ecmult_ladder_q, both half ladders and ecmult_ladder against k1*Q + k2*(beta x, y) (+ u1*G)"""
    rnd = random.Random(seed)
    cases = ladder_inputs(rnd, n, crafted)
    recs = new_records(len(cases))
    u1s = []
    for i, (q, k1, k2) in enumerate(cases):
        put(recs[i], 0, q[0])
        put(recs[i], 8, q[1])
        u1 = rnd.choice((0, 1, N - 1, rnd.randrange(N), rnd.randrange(N)))
        u1s.append(u1)
        put_work(recs[i], k1, k2, u1)
    out_q = engine.selftest_group(OPS["ECMULT_LADDER_Q"], recs)
    out_l = engine.selftest_group(OPS["ECMULT_LADDER"], recs)
    halves = []
    for lam in (0, 1):
        r2 = recs.copy()
        r2[:, 60] = lam
        if lam:
            r2[:, 32:37] = recs[:, 40:45]
        halves.append(engine.selftest_group(OPS["ECMULT_HALF_LADDER"], r2))
    for i, (q, k1, k2) in enumerate(cases):
        a, b = mul(k1, q), mul(k2, endo(q))
        want = add(a, b)
        assert get_jac(out_q[i]) == want, ("ecmult_ladder_q", i)
        if (q[1] * q[1] - q[0] ** 3 - 7) % P == 0:  # the comb adds u1*G: only meaningful on secp256k1 itself
            assert get_jac(out_l[i]) == add(want, ecc.base_mult(u1s[i])), ("ecmult_ladder", i)
        for lam, part in ((0, a), (1, b)):
            o = halves[lam][i]
            zc = get(o, 32) % P
            got = None if o[24] else aff(get(o, 0), get(o, 8), get(o, 16) * zc)
            assert got == part, ("ecmult_half_ladder", lam, i)
    hit("ladders.cases", len(cases))
    hit("ladders.crafted", len(crafted))


def case_combs(engine, n=3000, seed=37, crafted=()):
    """ecmult_comb_add onto a point (random, infinity, or one that meets a comb row) and small_comb from infinity"""
    rnd = random.Random(seed)
    cases = list(crafted)
    while len(cases) < n:
        u1 = rnd.choice((0, 1, N - 1, 2**16, 2**255, rnd.randrange(N), rnd.randrange(N), rnd.randrange(N)))
        r = rnd.random()
        start = None if r < 0.2 else rnd.randrange(1, N)
        cases.append((start, u1))
    recs = new_records(len(cases))
    for i, (start, u1) in enumerate(cases):
        put_jac(recs[i], 0, None if start is None else ecc.base_mult(start), random_z(rnd), rnd)
        put(recs[i], 48, u1)
    out_a = engine.selftest_group(OPS["ECMULT_COMB_ADD"], recs)
    out_s = engine.selftest_group(OPS["SMALL_COMB"], recs)
    for i, (start, u1) in enumerate(cases):
        s = 0 if start is None else start
        want = ecc.base_mult((s + u1) % N) if (s + u1) % N else None
        assert get_jac(out_a[i]) == want, ("ecmult_comb_add", i, start, u1)
        assert get_jac(out_s[i]) == (ecc.base_mult(u1) if u1 % N else None), ("small_comb", i, u1)
    hit("combs.cases", len(cases))
    hit("combs.crafted", len(crafted))


def case_ns_linear_form(engine, n=5000, seed=38):
    """D == y*B exactly when r = x(S + T); y(S + T) == N / (D*CG); the exceptional flag iff x(S) == x(T)"""
    rnd = random.Random(seed)
    recs = new_records(n)
    cases = []
    for i in range(n):
        p1 = random_point(rnd, 7)
        k = i % 6
        p2 = p1 if k == 0 else neg(p1) if k == 1 else random_point(rnd, 7)
        y = random.Random(i).randrange(1, P) if k != 5 else 1
        z1, z2 = random_z(rnd), random_z(rnd)
        X1, Y1, Z1 = jac(p1, z1)
        Zs = Z1 * pow(y, -1, P) % P
        s = add(p1, p2)
        good = k in (2, 3, 5)
        r = s[0] if (s is not None and good) else rnd.randrange(P)
        put(recs[i], 0, X1)
        put(recs[i], 8, Y1)
        put(recs[i], 16, Zs)
        put(recs[i], 24, y * y % P)
        X2, Y2, Z2 = jac(p2, z2)
        put(recs[i], 32, X2)
        put(recs[i], 40, Y2)
        put(recs[i], 48, Z2)
        put(recs[i], 56, r)
        cases.append((p1, p2, y, s, r, good))
    out = engine.selftest_group(OPS["NS_LINEAR_FORM"], recs)
    for i, (p1, p2, y, s, r, good) in enumerate(cases):
        D, B, Nn, CG = (get(out[i], 8 * j) % P for j in range(4))
        exact = int(out[i, 32])
        assert exact == (p1[0] == p2[0]), ("ns_linear_form exceptional flag", i)
        if exact:
            hit("ns_linear_form.equal_x")
            continue
        assert B != 0
        assert (D == y * B % P) == (r == s[0]), ("ns_linear_form D == y*B iff r == x(S+T)", i)
        if good:
            assert Nn == s[1] * D * CG % P, ("ns_linear_form y(S+T) == N/(D*CG)", i)
        hit("ns_linear_form." + ("match" if good else "mismatch"))
