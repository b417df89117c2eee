"""Which group additions a verification performs, in order, and which branch of the group law each one takes.

Every addition of the engine's multiplication schedules adds two multiples of G: with Q = d*G the accumulator and the
addend are known scalars mod n, so the branch of gej_add_ge / gej_add_gej (ge.cuh) follows from modular arithmetic alone:
  accumulator at infinity -> a_inf;  addend at infinity (gej_add_gej only) -> b_inf;
  accumulator == addend   -> double; accumulator == -addend -> infinity;  otherwise generic.
The scalars come from the engine's own recodings: the GLV split forced odd (sc_prepare_u2, restated by prepare_u2 below and
checked against SV_ST_PREPARE_U2), the signed odd 4-bit windows read by window4 / qtable_fetch, and the comb digits of
sc_prepare_u1.  The host build logs the branch of every addition (SV_GE_TRACE), and tests/test_group_emul.py checks that
this model predicts that log addition by addition.

Schedules (verify.cuh):
  main       throughput kernel: odd-multiples table (7 additions), joint ladder over both GLV halves (1 + 2 x 32
             additions), then the comb added onto the ladder's result (one addition per non-zero digit of u1).  The
             shared-key path and the fee grind run the same ladder and comb with a prebuilt table.
  main_ns    the flows without the square root: same table and ladder on E', the comb summed from infinity, and the plain
             `main` schedule again when the linear form does not apply (SV_NS_EXACT: T or S at infinity, x(S) == x(T), or
             the r + n candidate of compressed-key ECDSA).  B == 0 never happens: B = 2 Y1 Y2 c Zs^3 Z2^3 and no point of
             odd prime order has y = 0.
  small      small-batch kernel: table, two half ladders, the comb summed from infinity, join 1 = R1 + R2 on the scaled
             curve, join 2 = (R1 + R2) + u1*G.
  small_ns   the same, then `main` when the linear form does not apply.

Exceptional step classes and why some cannot be reached (a step class is (step, branch); `reach` below lists the reachable
ones per schedule, and the fixture of tests/golden/group_exceptional.npz reaches each of them):
  table       never exceptional: the accumulator (2k-1)Q meets 2Q, and (2k-1) == +-2 mod n has no solution for k < 8.
  top         never exceptional: the top digits t1*Q + lambda*t2*Q with |t1|, |t2| < 16 would need t1 -+ lambda*t2 == 0
              mod n, a non-zero vector of length < 2^5 in the GLV lattice {(a, b): a + b*lambda == 0}, whose shortest
              vectors are longer than 2^126.
  window      ladder windows of the joint ladder: before the add of window i the accumulator is 16*(p1 + lambda*p2) (p =
              the digit prefixes), so an exceptional add needs a lattice vector whose entries are about |k| / 16^i.  Only
              windows 0 and 1 qualify, and there the condition pins u2 to one value per choice of the low digits
              (window_candidates).  Enumerating all of them: exactly one u2 (an odd multiple of 2*lambda) is consistent
              with its own recoding, and it doubles at half 1 of window 0.  No other window addition can double or
              cancel, so no later one can start from infinity.
  half        a single half ladder never is: its prefixes are integers below 2^131 < n, never 0 and never +-the
              odd digit after a multiplication by 16 (an even number).
  comb        the comb added onto the ladder: any row, double and infinity, by the choice of d (u2*d == the needed
              residue); a_inf after an infinity that is not at the last non-zero row.
  comb_sum    the comb summed from infinity: its first addition is always a_inf.  Later rows are never exceptional: the
              prefix sums S_j = sum_{i<j} gd_i 2^(16i) are integers with |S_j| < 2^(16j-1) * 1.0001 while a non-zero
              addend is at least 2^(16j) in magnitude, so S_j -+ a_j is a non-zero integer below n for j < 15, and for
              j = 15 it would force u1 = S_15 + a_15 to be 0 or >= n.
  join1       R1 + R2 == k1*Q + lambda*k2*Q: double iff k1 == lambda*k2 mod n, a short vector of the GLV lattice
              that the split of u2 == 2*k1 returns (found by search); infinity iff u2 == 0, which a valid encoding
              excludes; neither side is ever infinity (k odd, |k| < 2^131).
  join2       (u2*d)*G + u1*G: double iff u2*d == u1, infinity iff u2*d == -u1, b_inf iff u1 == 0 (message hash 0, or
              BIP-340 s == 0); a_inf would need join 1 at infinity.
  BIP-340: u2 = -e is a hash of (R.x, P, m) and u1 = s is free, so the conditions that involve only u2 (window, join1)
  cannot be steered; those that tie u1 to u2*d (comb, join2) can: choose d, r, m, compute e, then s.  Signatures built
  that way hit the branch and are invalid (r is fixed before R is known).
"""
from tests import limb_model as M

N = M.N
P = M.P
LAMBDA = 0x5363AD4CC05C30E0A5261C028812645A122E22EA20816678DF02967C1B23BD72
BETA = 0x7AE96A2B657C07106E64479EAC3434E99CF0497512F58995C1396C28719501EE
A1 = 0x3086D221A7D46BCDE86C90E49284EB15
B1 = -0xE4437ED6010E88286F547FA90ABFE4C3
A2 = 0x114CA50F7A8E2F3F657C1108D9D44CFD8

GENERIC, DOUBLE, INFINITY, A_INF, B_INF = 0, 1, 2, 3, 4
BRANCH = {GENERIC: "generic", DOUBLE: "double", INFINITY: "infinity", A_INF: "a_inf", B_INF: "b_inf"}
MIXED, FULL = 0, 8


def prepare_u2(u2):
    """sc_prepare_u2: GLV split, both halves forced odd by adding a lattice vector -> signed (k1, k2)"""
    r1, r2 = M.split_lambda(u2 % N)
    a = r1 - N if r1 > (N - 1) // 2 else r1
    b = r2 - N if r2 > (N - 1) // 2 else r2
    if a % 2 == 0 and b % 2 == 0:
        a, b = a + A1, b + B1
    elif b % 2 == 0:
        a, b = a + A2, b + A1
    elif a % 2 == 0:
        a, b = a + A1 + A2, b + B1 + A1
    return a, b


def prepare_u1(u1):
    """sc_prepare_u1: 16 signed 16-bit comb digits"""
    gd, carry = [], 0
    for i in range(16):
        win = ((u1 >> (16 * i)) & 0xFFFF) + carry
        if i < 15 and win > 0x8000:
            gd.append(win - 0x10000)
            carry = 1
        else:
            gd.append(win)
            carry = 0
    return gd


def ladder_digits(k):
    """window4 / qtable_fetch on the sign/magnitude of k: (top digit, [digit of window i for i = 31..0]), signed"""
    m, s = abs(k), (-1 if k < 0 else 1)
    top = 2 * ((m >> 129) & 7) + 1
    win = [2 * ((m >> (4 * i + 1)) & 15) - 15 for i in range(31, -1, -1)]
    assert top * 16**32 + sum(w * 16**i for w, i in zip(win, range(31, -1, -1))) == m, "recoding does not sum to |k|"
    return s * top, [s * w for w in win]


class Run:
    """the additions of one verification: steps = [(form, step, branch)]"""

    def __init__(self):
        self.steps = []

    def add(self, form, step, acc, addend):
        """acc, addend: scalars mod n (None = infinity); returns the sum and logs the branch"""
        if acc is None:
            br, out = A_INF, addend
        elif addend is None:
            br, out = B_INF, acc
        elif acc == addend:
            br, out = DOUBLE, 2 * acc % N
        elif (acc + addend) % N == 0:
            br, out = INFINITY, None
        else:
            br, out = GENERIC, (acc + addend) % N
        self.steps.append((form, step, br))
        return out

    def codes(self):
        return [form | br for form, _, br in self.steps]


def _mulq(k, d):
    return k * d % N or None


def table(run, d):
    acc = d % N
    two = 2 * d % N
    for _ in range(7):
        acc = run.add(MIXED, "table", acc, two)


def ladder(run, k1, k2, d):
    t1, w1 = ladder_digits(k1)
    t2, w2 = ladder_digits(k2)
    acc = _mulq(t1, d)
    acc = run.add(MIXED, "top", acc, _mulq(t2 * LAMBDA, d))
    for j in range(32):
        acc = None if acc is None else 16 * acc % N
        i = 31 - j
        acc = run.add(MIXED, f"window{i}.half0" if i < 2 else "window", acc, _mulq(w1[j], d))
        acc = run.add(MIXED, f"window{i}.half1" if i < 2 else "window", acc, _mulq(w2[j] * LAMBDA, d))
    return acc


def half_ladder(run, k, lam, d):
    t, w = ladder_digits(k)
    f = LAMBDA if lam else 1
    acc = _mulq(t * f, d)
    for j in range(32):
        acc = None if acc is None else 16 * acc % N
        acc = run.add(MIXED, "half", acc, _mulq(w[j] * f, d))
    return acc


def comb(run, acc, u1, step):
    for j, g in enumerate(prepare_u1(u1)):
        if g:
            acc = run.add(MIXED, step, acc, g * 2**(16 * j) % N)
    return acc


def schedule(name, u1, u2, d, r_plus_n=False, run=None):
    """the Run of schedule `name` for scalars u1, u2 (< n) and key Q = d*G; r_plus_n: compressed-key ECDSA with r < p - n"""
    run = run or Run()
    k1, k2 = prepare_u2(u2)
    if name in ("main", "samekey"):
        if name == "main":
            table(run, d)
        comb(run, ladder(run, k1, k2, d), u1, "comb")
        return run
    table(run, d)
    if name == "main_ns":
        S = ladder(run, k1, k2, d)
        T = comb(run, None, u1, "comb_sum")
    else:
        R1 = half_ladder(run, k1, False, d)
        R2 = half_ladder(run, k2, True, d)
        T = comb(run, None, u1, "comb_sum")
        S = run.add(FULL, "join1", R1, R2)
        if name == "small":
            run.add(FULL, "join2", S, T)
            return run
    exact = S is None or T is None or r_plus_n or S == T or (S + T) % N == 0
    run.exact = exact
    if exact:
        schedule("main", u1, u2, d, run=run)
    return run


SCHEDULES = ("main", "main_ns", "small", "small_ns")
# (step, branch) classes each schedule can reach (see the module docstring for the others)
LADDER_REACH = {("window0.half1", "double")}
REACH = {
    "main": LADDER_REACH | {("comb", "double"), ("comb", "infinity"), ("comb", "a_inf")},
    "main_ns": LADDER_REACH | {("comb_sum", "a_inf")},
    "small": {("comb_sum", "a_inf"), ("join1", "double"), ("join2", "double"), ("join2", "infinity"), ("join2", "b_inf")},
    "small_ns": {("comb_sum", "a_inf"), ("join1", "double")},
}
# the no-sqrt flows fall back to `main` on these triggers (the classes of `main` are then reached through them as well)
NS_TRIGGERS = ("T_inf", "H_zero_double", "H_zero_infinity", "r_plus_n")


def classes(run, schedule_name):
    """{(step, branch)} of the exceptional additions of a run, the fallback's steps under 'fallback.'"""
    out = set()
    fallback_start = None
    if getattr(run, "exact", False):
        # the first `table` step after the first ladder/comb begins the fallback
        seen_ladder = False
        for i, (_, step, _) in enumerate(run.steps):
            if step != "table":
                seen_ladder = True
            elif seen_ladder:
                fallback_start = i
                break
    for i, (_, step, br) in enumerate(run.steps):
        if br == GENERIC:
            continue
        pre = "fallback." if fallback_start is not None and i >= fallback_start else ""
        out.add((pre + step, BRANCH[br]))
    return out


def ns_trigger(u1, u2, d, r_plus_n=False):
    """why the flows without the square root hand a verification to the plain path, or None"""
    S = u2 * d % N
    if u1 % N == 0:
        return "T_inf"
    if S == u1 % N:
        return "H_zero_double"
    if (S + u1) % N == 0:
        return "H_zero_infinity"
    if r_plus_n:
        return "r_plus_n"
    return None


# ---- solving for (d, u1, u2) -------------------------------------------------------------------------------------------
def _low_digits(k, count):
    m, s = abs(k), (-1 if k < 0 else 1)
    return [s * (2 * ((m >> (4 * i + 1)) & 15) - 15) for i in range(count)]


def window_candidates(window):
    """Every u2 whose own recoding makes an addition of ladder window `window` (0 or 1) exceptional: [(u2, step, branch)].

    With L1, L2 the value of the digits of k1, k2 below window i and e1, e2 their digits at window i, the accumulator
    before half 0 of window i is 16^-i * (k1 - L1 - e1*16^i + lambda*(k2 - L2 - e2*16^i)), so that addition meets +-e1
    iff u2 == L1 + e1*16^i +- e1*16^i + lambda*(L2 + e2*16^i); before half 1 it meets +-lambda*e2 iff
    u2 == L1 + lambda*(L2 + e2*16^i +- e2*16^i) (the minus sign would need u2 == 0 at window 0).  Each candidate is kept iff the recoding of that u2 has exactly
    those digits.  Windows i >= 2 need a non-zero GLV-lattice vector with entries below 2^131 / 16^i + 16 < 2^124, shorter
    than any there is, so they have no candidates at all."""
    out = []
    odd = [s * v for v in range(1, 16, 2) for s in (1, -1)]
    lows = [[]]
    for _ in range(window + 1):
        lows = [l + [e] for l in lows for e in odd]
    sc = 16**window
    for d1 in lows:
        L1 = sum(e * 16**j for j, e in enumerate(d1))  # includes e1 at window i
        for d2 in lows:
            L2 = sum(e * 16**j for j, e in enumerate(d2))
            e1, e2 = d1[-1] * sc, d2[-1] * sc
            for step, br, u2 in ((f"window{window}.half0", "double", L1 + e1 + LAMBDA * L2),
                                 (f"window{window}.half0", "infinity", L1 - e1 + LAMBDA * L2),
                                 (f"window{window}.half1", "double", L1 - e1 + LAMBDA * (L2 + e2)),
                                 (f"window{window}.half1", "infinity", L1 - e1 + LAMBDA * (L2 - e2))):
                u2 %= N
                if not u2:
                    continue
                k1, k2 = prepare_u2(u2)
                if _low_digits(k1, window + 1) == d1 and _low_digits(k2, window + 1) == d2:
                    out.append((u2, step, br))
    return sorted(set(out))


def join1_candidates(limit=40):
    """u2 for which R1 == R2 in the small kernel's first join: k1 == lambda*k2 with (k1, k2) the forced-odd split of u2;
    enumerated over short vectors (x, y) of the GLV lattice, k1 = x, k2 = -y  (x + y*lambda == 0)"""
    out = []
    B2 = A1  # b2 of the lattice basis (a1, b1), (a2, b2)
    for i in range(-6, 7):
        for j in range(-6, 7):
            x, y = i * A1 + j * A2, i * B1 + j * B2
            if (x + y * LAMBDA) % N:
                continue
            k1, k2 = x, -y
            if k1 % 2 == 0 or k2 % 2 == 0 or abs(k1) >= 2**131 or abs(k2) >= 2**131:
                continue
            u2 = (k1 + k2 * LAMBDA) % N
            if u2 and prepare_u2(u2) == (k1, k2):
                out.append(u2)
    return sorted(set(out))[:limit]
