"""ECDSA signatures forged for 64-byte keys off secp256k1, which only the key check can refuse.

A 64-byte key x||y is accepted by secp256k1_ec_pubkey_parse(04||x||y) only when y^2 = x^3 + 7.  The engine decodes it
without an early exit (verify.cuh key_decode): an off-curve key carries a false flag and its coordinates through the
table build and the ladder, and the flag alone keeps the verdict at 0.  None of ge.cuh's formulas use the curve constant,
so for a point Q on y^2 = x^3 + b' the ladder computes u2*Q correctly on THAT curve.  Such a curve can have small
subgroups, and there the result of the ladder can be steered:

  * the six curves y^2 = x^3 + b over F_p (p = 1 mod 6) fall into six isomorphism classes; with t = p + 1 - n and
    4p = t^2 + 3v^2 their orders are p + 1 - T for T in {t, -t, (t+3v)/2, (t-3v)/2, -(t+3v)/2, -(t-3v)/2}.  Each class's
    representative is found below by checking a random point against the six candidate orders (class_orders);
  * Q = a random point times the cofactor order/h has order h, a prime h = 1 mod 3 dividing that order.  The endomorphism
    (x, y) -> (beta*x, y) the ladder uses for its lambda half acts on <Q> as multiplication by mu, a cube root of unity
    mod h (not lambda: lambda is its eigenvalue mod n on secp256k1);
  * with message 0 (the 32 zero bytes, or the encoding of n, which reduces to 0) u1 = 0, so the engine's R is the
    ladder's u2*Q alone: with (k1, k2) the GLV split of u2 forced odd (sc_prepare_u2), R = (k1 + mu*k2)*Q =: j*Q.
    Any u2 thus names its own j.  Take r = x(j*Q) when that is below n, and s = r/u2: then u2 = r/s, and the signature
    (r, s) is accepted by a build that forgets the key flag.  Keep it when s <= n/2 (the engine refuses high S).

The forcing to odd halves adds a vector (a, b) with a + b*lambda = 0 mod n, but a + b*mu is not 0 mod h: a prediction from
the plain GLV split is right only when both halves are odd already.  predict() follows the device's recoding; ladder_point()
repeats its 4-bit windows over the table {1, 3, ..., 15}*Q point by point.

Classes and their subgroups (orders factored by trial division below 2^17, checked in subgroups()):
  b' = 2: 3319, 22639;  b' = 4: 199, 18979;  b' = 6: 10903 (5290657 lies beyond the search);  b' = 3: 109903.
  b' = 1 has no usable subgroup: below 2^17 its order has only the factors 2^2 and 3, and a point of order <= 4 makes
  the table of odd multiples {1, ..., 15}*Q run into infinity (like the order-3 lift of x = 0 the suite tests elsewhere).
  b' = 7 is secp256k1 itself (order n).

The fixture tests/golden/invalid_curve.npz holds the cases (python -m tests.golden.make_invalid_curve)."""
import ctypes
import math
import os
import random
import shutil
import subprocess

import numpy as np

from tests import group_schedule as S
from tests.util import P as ptr

P, N = S.P, S.N
BETA = S.BETA
T = P + 1 - N
V = math.isqrt((4 * P - T * T) // 3)
assert 3 * V * V == 4 * P - T * T
TRACES = (T, -T, (T + 3 * V) // 2, (T - 3 * V) // 2, -(T + 3 * V) // 2, -(T - 3 * V) // 2)
ORDERS = tuple(P + 1 - t for t in TRACES)
# (b', h): every prime h = 1 mod 3, 15 < h < 2^17, dividing the order of y^2 = x^3 + b', b' a class representative
SUBGROUPS = ((2, 3319), (2, 22639), (4, 199), (4, 18979), (6, 10903), (3, 109903))
FACTOR_BOUND = 2**17
SIGS_PER_KEY = 4  # distinct signatures per forged key, each with both messages
MESSAGES = (bytes(32), N.to_bytes(32, "big"))  # both reduce to 0 mod n
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "invalid_curve.npz")


# ---- affine arithmetic on any y^2 = x^3 + b (the formulas do not involve b); None is the point at infinity ----------
def add(A, B):
    if A is None:
        return B
    if B is None:
        return A
    (x1, y1), (x2, y2) = A, B
    if x1 == x2:
        if (y1 + y2) % P == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, P) % P
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, P) % P
    x3 = (lam * lam - x1 - x2) % P
    return x3, (lam * (x1 - x3) - y1) % P


def neg(A):
    return None if A is None else (A[0], -A[1] % P)


def mul(k, A):
    if k < 0:
        return mul(-k, neg(A))
    R = None
    while k:
        if k & 1:
            R = add(R, A)
        A = add(A, A)
        k >>= 1
    return R


def phi(A):
    """the endomorphism of the lambda half: (x, y) -> (beta*x, y)"""
    return None if A is None else (BETA * A[0] % P, A[1])


def on_curve(A, b):
    return (A[1] * A[1] - A[0] ** 3 - b) % P == 0


def random_point(b, rng):
    while True:
        x = rng.randrange(P)
        c = (x ** 3 + b) % P
        if pow(c, (P - 1) // 2, P) == 1:
            y = pow(c, (P + 1) // 4, P)
            return x, (y if rng.random() < 0.5 else P - y)


# ---- the six classes -------------------------------------------------------------------------------------------------
def class_orders(bmax=12):
    """{b: order of y^2 = x^3 + b} for the smallest b of each of the six classes, each order found as the one candidate
    that a random point of the curve is killed by"""
    rng = random.Random("invalid-curve/classes")
    out = {}
    for b in range(1, bmax + 1):
        R = random_point(b, rng)
        hits = [o for o in ORDERS if mul(o, R) is None]
        assert len(hits) == 1, (b, len(hits))
        if hits[0] not in out.values():
            out[b] = hits[0]
    assert sorted(out.values()) == sorted(ORDERS), "not all six classes met"
    return out


def small_primes(order, bound=FACTOR_BOUND):
    out, m, d = [], order, 2
    while d < bound:
        if m % d == 0:
            out.append(d)
            while m % d == 0:
                m //= d
        d += 1
    return out


def subgroups():
    """[(b', h, order)] of SUBGROUPS, each h checked to be exactly the usable primes of its class below the bound"""
    orders = class_orders()
    assert orders[7] == N and sorted(orders) == [1, 2, 3, 4, 6, 7], orders
    usable = {b: [q for q in small_primes(o) if q > 15 and q % 3 == 1] for b, o in orders.items() if b != 7}
    assert usable[1] == [] and small_primes(orders[1]) == [2, 3], "class b' = 1 has a usable subgroup after all"
    assert sorted((b, h) for b, hs in usable.items() for h in hs) == sorted(SUBGROUPS), usable
    return [(b, h, orders[b]) for b, h in SUBGROUPS]


def point_of_order(b, h, order, rng):
    """a point of exact order h on y^2 = x^3 + b, off secp256k1"""
    while True:
        Q = mul(order // h, random_point(b, rng))
        if Q is not None:
            break
    assert mul(h, Q) is None and on_curve(Q, b) and not on_curve(Q, 7)
    return Q


def eigenvalue(Q, h):
    """mu with phi(Q) == mu*Q: one of the two primitive cube roots of unity mod h"""
    w = next(pow(c, (h - 1) // 3, h) for c in range(2, h) if pow(c, (h - 1) // 3, h) != 1)
    mu = next(m for m in (w, w * w % h) if mul(m, Q) == phi(Q))
    assert (mu * mu + mu + 1) % h == 0
    return mu


# ---- what the device computes --------------------------------------------------------------------------------------
def predict(u2, mu, h):
    """j with u2*Q == j*Q on the device: the windows of the forced-odd halves (sc_prepare_u2, window4 / qtable_fetch)
    summed as ecmult_ladder_q adds them, with phi acting as mu on <Q>"""
    k1, k2 = S.prepare_u2(u2)
    t1, w1 = S.ladder_digits(k1)
    t2, w2 = S.ladder_digits(k2)
    acc = (t1 + mu * t2) % h
    for a, b in zip(w1, w2):
        acc = (16 * acc + a + mu * b) % h
    return acc


def ladder_point(u2, Q):
    """u2*Q as ecmult_ladder_q computes it, point by point: odd-multiples table {1, 3, ..., 15}*Q, the top digits of both
    halves, then per window four doublings and one table point per half (phi applied to the second)"""
    k1, k2 = S.prepare_u2(u2)
    tab = [Q]
    for _ in range(7):
        tab.append(add(tab[-1], add(Q, Q)))
    fetch = lambda d, lam: (phi if lam else (lambda A: A))(tab[abs(d) // 2] if d > 0 else neg(tab[abs(d) // 2]))
    t1, w1 = S.ladder_digits(k1)
    t2, w2 = S.ladder_digits(k2)
    R = add(fetch(t1, False), fetch(t2, True))
    for a, b in zip(w1, w2):
        for _ in range(4):
            R = add(R, R)
        R = add(add(R, fetch(a, False)), fetch(b, True))
    return R


def forge(Q, mu, h, count, rng):
    """count signatures (r, s, j, u2) valid for Q on its own curve at message 0, with distinct s"""
    out = []
    while len(out) < count:
        u2 = rng.randrange(1, N)
        j = predict(u2, mu, h)
        if j == 0:
            continue
        r = mul(j, Q)[0]
        if r >= N:
            continue
        s = r * pow(u2, -1, N) % N
        if s > N // 2 or any(s == o[1] for o in out):
            continue
        out.append((r, s, j, u2))
    return out


def build_cases():
    """the construction, as the fixture's arrays (everything but the verdicts)"""
    b_, h_, j_, g_ = [], [], [], []
    key, sig, msg = [], [], []
    for g, (b, h, order) in enumerate(subgroups()):
        rng = random.Random(f"invalid-curve/{b}/{h}")
        Q = point_of_order(b, h, order, rng)
        mu = eigenvalue(Q, h)
        for r, s, j, _ in forge(Q, mu, h, SIGS_PER_KEY, rng):
            for m in MESSAGES:
                b_.append(b), h_.append(h), j_.append(j), g_.append(g)
                key.append(Q[0].to_bytes(32, "big") + Q[1].to_bytes(32, "big"))
                sig.append(r.to_bytes(32, "big") + s.to_bytes(32, "big"))
                msg.append(m)
    arr = lambda v, w: np.frombuffer(b"".join(v), np.uint8).reshape(-1, w).copy()
    return dict(b=np.array(b_, np.int64), h=np.array(h_, np.int64), j=np.array(j_, np.int64),
                group=np.array(g_, np.int64), key=arr(key, 64), sig=arr(sig, 64), msg=arr(msg, 32))


def load():
    with np.load(FIXTURE) as z:
        return {k: z[k] for k in z.files}


# ---- the key gates, and host builds without one ---------------------------------------------------------------------
# name -> (file under lightning_b200/csrc, the gate's text, the text without it, the host-build entry points that run it)
ROUTES = ("emul_verify_batch", "emul_verify_small_batch", "emul_verify_small_pair_batch", "emul_verify_samekey")
MUTANTS = {
    "key_decode": ("verify.cuh", "        return ge_is_on_curve(Q) && ok;\n", "        return ok;\n", ROUTES),
    "verify_curve_side": ("verify.cuh", "    ok = kd && ok;\n", "    (void)kd;\n", ("emul_verify_batch",)),
    "verify_curve_side_shared": ("verify.cuh", "(flags & SV_WF_VALID) != 0 && sk->ok != 0;\n", "(flags & SV_WF_VALID) != 0;\n",
                                 ("emul_verify_samekey",)),
    "small_finish": ("verify.cuh", "\n    bool ok = (flags & SV_WF_VALID) != 0 && it->key_ok != 0;\n",
                     "\n    bool ok = (flags & SV_WF_VALID) != 0;\n", ("emul_verify_small_batch", "emul_verify_small_pair_batch")),
}


def build_mutant(name, workdir, csrc=None):
    """the host build (tests/host_emul/emul.cpp, the g++ line of lightning_b200.build.build_host_emul) of a copy of the
    kernel source (lightning_b200/csrc, or csrc) with gate `name` removed; returns the library's path.  The gate's text
    must occur exactly once."""
    from lightning_b200 import build
    fname, gate, without, _ = MUTANTS[name]
    root = os.path.join(workdir, name)
    shutil.rmtree(root, ignore_errors=True)
    shutil.copytree(csrc or build.CSRC, os.path.join(root, "lightning_b200", "csrc"), ignore=shutil.ignore_patterns("*.o", "*.so"))
    shutil.copytree(os.path.join(build.ROOT, "tests", "host_emul"), os.path.join(root, "tests", "host_emul"),
                    ignore=shutil.ignore_patterns("*.so", "*.o"))
    shutil.copytree(os.path.join(build.ROOT, "include"), os.path.join(root, "include"))
    path = os.path.join(root, "lightning_b200", "csrc", fname)
    text = open(path).read()
    assert text.count(gate) == 1, f"{name}: the gate {gate.strip()!r} occurs {text.count(gate)} times in {fname}"
    open(path, "w").write(text.replace(gate, without))
    lib = os.path.join(root, "libemul.so")
    r = subprocess.run(build.HOST_EMUL_CXX + ["-o", lib, os.path.join(root, "tests", "host_emul", "emul.cpp")],
                       capture_output=True, text=True)
    assert r.returncode == 0, f"g++ ({name} mutant) failed:\n{r.stdout}{r.stderr}"
    return lib


def run_route(lib, route, fx):
    """verdicts of host-build entry point `route` (kind 1) on every case of the fixture; the shared-key entry point runs
    each forged key's cases as one batch"""
    n = fx["msg"].shape[0]
    out = np.zeros(n, np.uint8)
    if route != "emul_verify_samekey":
        getattr(lib, route)(1, ptr(fx["msg"]), ptr(fx["key"]), ptr(fx["sig"]), ctypes.c_size_t(n), ptr(out))
        return out
    for g in np.unique(fx["group"]):
        sel = np.nonzero(fx["group"] == g)[0]
        m, s = np.ascontiguousarray(fx["msg"][sel]), np.ascontiguousarray(fx["sig"][sel])
        k = np.ascontiguousarray(fx["key"][sel[0]])
        assert (fx["key"][sel] == k).all()
        o = np.zeros(sel.size, np.uint8)
        lib.emul_verify_samekey(1, ptr(k), ptr(m), ptr(s), ctypes.c_size_t(sel.size), ptr(o))
        out[sel] = o
    return out
