"""CPU: the group law and the multiplication schedules on the HOST build of the kernel headers (tests/host_emul).

  * the group self-test ops of tests/group_cases.py against Python integers, at reduced sizes (the device forms run at
    full size in tests/test_gpu_group.py);
  * the schedule model of tests/group_schedule.py against the branch log of the host build, addition by addition, for
    every schedule, over the constructed fixture, the adversarial fixture and random signatures;
  * the constructed fixture (tests/golden/group_exceptional.npz) through the host-build verifiers against the reference;
  * coverage: every step class the model calls reachable is hit in each schedule."""
import ctypes
import random
from collections import Counter, defaultdict

import numpy as np
import pytest

from tests import adversarial, bolt11
from tests import group_cases as C
from tests import group_fixture as F
from tests import group_schedule as S
from tests import selftest_cases as SC
from tests.util import P as ptr, ref_verify


class EmulGroup:
    def __init__(self, emul):
        self.emul = emul
        emul.emul_gtable_build()

    def selftest_group(self, op, rec):
        rec = np.ascontiguousarray(rec, dtype=np.uint32).reshape(-1, C.IN_WORDS)
        out = np.zeros((rec.shape[0], C.OUT_WORDS), dtype=np.uint32)
        self.emul.emul_selftest_group(int(op), rec.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(rec.shape[0]),
                                      out.ctypes.data_as(ctypes.c_void_p))
        return out

    def selftest(self, op, a, b=None):
        a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1, 8)
        b = np.zeros_like(a) if b is None else np.ascontiguousarray(b, dtype=np.uint32).reshape(-1, 8)
        out = np.zeros((a.shape[0], 16), dtype=np.uint32)
        self.emul.emul_selftest(int(op), a.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                                ctypes.c_size_t(a.shape[0]), out.ctypes.data_as(ctypes.c_void_p))
        return out


@pytest.fixture(scope="module")
def eng(emul):
    emul.emul_trace_end.restype = ctypes.c_size_t
    return EmulGroup(emul)


def crafted_ladders():
    rnd = random.Random(7)
    out = []
    for u2, _, _ in S.window_candidates(0):
        for _ in range(4):
            out.append((adversarial.mul(rnd.randrange(1, S.N), adversarial.G),) + S.prepare_u2(u2))
    return out


def crafted_combs():
    """(start scalar, u1) pairs whose comb additions double or cancel at a chosen row"""
    rnd = random.Random(8)
    out = []
    for _ in range(12):
        u1 = rnd.randrange(1, S.N)
        gd = S.prepare_u1(u1)
        for row in [j for j, g in enumerate(gd) if g][::5]:
            for sign in (1, -1):
                out.append((F._row_target(u1, row, sign) or None, u1))
    return out


def test_group_ops_against_python(eng):
    C.case_gej_double(eng, n=4000)
    C.case_gej_add_ge(eng, n=4000)
    C.case_gej_add_gej(eng, n=4000)
    C.case_ge_set_xo(eng, n=2000)
    C.case_qtable_build(eng, n=200)
    C.case_ladders(eng, n=60, crafted=crafted_ladders())
    C.case_combs(eng, n=150, crafted=crafted_combs())
    C.case_ns_linear_form(eng, n=600)
    for key in ("gej_add_ge.double", "gej_add_ge.infinity", "gej_add_ge.a_inf", "gej_add_gej.double",
                "gej_add_gej.infinity", "gej_add_gej.a_inf", "gej_add_gej.b_inf", "gej_add_gej.alias_a.double",
                "gej_add_gej.alias_b.infinity", "ge_set_xo.non_residue.odd", "ns_linear_form.equal_x"):
        assert C.COVERAGE.get(key), key


def test_prepare_u2_model_matches_engine(eng):
    rnd = random.Random(9)
    ks = [u for u, _, _ in S.window_candidates(0)] + S.join1_candidates() + [rnd.randrange(1, S.N) for _ in range(3000)]
    out = eng.selftest(SC.OPS["PREPARE_U2"], SC.limbs([0] * len(ks)), SC.limbs(ks))
    for row, k in zip(out, ks):
        words = [sum(int(row[h * 5 + i]) << (32 * i) for i in range(5)) for h in (0, 1)]
        got = tuple(-(w & ((1 << 159) - 1)) if w >> 159 else w for w in words)
        assert got == S.prepare_u2(k), hex(k)


# ---- schedule model against the branch log ------------------------------------------------------------------------------
KEYLEN = {0: 33, 1: 64, 2: 32}


def trace(emul, fn, kind, msg, key, sig):
    out = np.zeros(1, np.uint8)
    buf = np.zeros(4096, np.uint8)
    emul.emul_trace_begin()
    fn(kind, ptr(msg), ptr(key), ptr(sig), ctypes.c_size_t(1), ptr(out))
    n = emul.emul_trace_end(ptr(buf), ctypes.c_size_t(buf.size))
    assert n <= buf.size
    return [int(v) for v in buf[:n]], int(out[0])


def routes(emul):
    """schedule name -> (kinds, how the host build runs one item through it)"""
    def exact(on):
        emul.emul_set_ecdsa33_exact(on)
    return {
        "main": ((0, 1, 2), lambda k: exact(1) or emul.emul_verify_batch),
        "main_ns": ((0, 2), lambda k: exact(0) or emul.emul_verify_batch),
        "small": ((0, 1, 2), lambda k: exact(1) or emul.emul_verify_small_batch),
        "small_pair": ((0, 1, 2), lambda k: exact(1) or emul.emul_verify_small_pair_batch),
        "small_ns": ((0, 2), lambda k: exact(0) or emul.emul_verify_small_batch),
        "samekey": ((0, 1), lambda k: None),
    }


def items():
    """(kind, msg, key, sig, u1, u2, d, r_plus_n, source) of the constructed fixture, part of the adversarial fixture and
    a few random valid signatures"""
    fx = F.load()
    keys = F.ecdsa_keys(fx)
    for i in range(len(fx["ecdsa_label"])):
        u1, u2, d, rpn = F.ecdsa_scalars(fx["ecdsa_msg"][i], fx["ecdsa_sig"][i], fx["ecdsa_pubxy"][i], keys)
        for kind, key in ((0, fx["ecdsa_pub33"][i]), (1, fx["ecdsa_pubxy"][i])):
            yield kind, fx["ecdsa_msg"][i], key, fx["ecdsa_sig"][i], u1, u2, d, rpn and kind == 0, "constructed"
    for i in range(len(fx["bip340_label"])):
        u1, u2, d = F.bip340_scalars(fx["bip340_msg"][i], fx["bip340_xonly"][i], fx["bip340_sig"][i], F._int(fx["bip340_d"][i]))
        yield 2, fx["bip340_msg"][i], fx["bip340_xonly"][i], fx["bip340_sig"][i], u1, u2, d, False, "constructed"
    for kind, msg, key, sig, u1, u2, d, rpn in adversarial_items(every=9):
        yield kind, msg, key, sig, u1, u2, d, rpn, "adversarial"


def adversarial_items(every=1):
    """the committed adversarial fixture with its scalars; the key's d is found among the generator's key choices"""
    msg, pub33, pubxy, sig = adversarial.load()
    ds = [1, 2, 3, 5, S.N - 1, S.N - 2, (S.N + 1) // 2, adversarial.LAMBDA, 0xDEADBEEFCAFEBABE0123456789ABCDEF]
    from tests import ecc
    known = {ecc.base_mult(d): d for d in ds}
    for i in range(0, msg.shape[0], every):
        u1, u2, d, rpn = F.ecdsa_scalars(msg[i], sig[i], pubxy[i], known)
        yield 0, msg[i], pub33[i], sig[i], u1, u2, d, rpn
        yield 1, msg[i], pubxy[i], sig[i], u1, u2, d, False


def model_name(route):
    return {"small_pair": "small", "samekey": "main"}.get(route, route)


def recovery_items():
    """(invoice, u1, u2, d) of the BOLT11 invoices built to steer the key recovery (make_bolt11.py rec_*)"""
    fx = bolt11.load_fixture()
    invs = bolt11.invoices(fx)
    for i in np.nonzero(np.char.startswith(fx["label_name"], "rec_"))[0]:
        yield (invs[i],) + bolt11.rec_scalars(fx, i)


def trace_recovery(emul, inv):
    """branch log of one invoice through bolt11.cuh's host build (parse, hash, and the recovery's `main` schedule)"""
    h, node = np.zeros(32, np.uint8), np.zeros(33, np.uint8)
    have_n = ctypes.c_int()
    buf = np.zeros(4096, np.uint8)
    emul.emul_trace_begin()
    emul.emul_bolt11(inv, ctypes.c_uint32(len(inv)), ptr(h), ptr(node), ctypes.byref(have_n))
    n = emul.emul_trace_end(ptr(buf), ctypes.c_size_t(buf.size))
    assert n <= buf.size and have_n.value == 0
    return [int(v) for v in buf[:n]]


def test_schedule_model_matches_host_branch_log(eng, emul):
    """every item through every schedule the host build has, and the BOLT11 recoveries through theirs: the model's
    predicted branch sequence == the log"""
    rs = routes(emul)
    checked = Counter()
    try:
        for kind, msg, key, sig, u1, u2, d, rpn, _ in items():
            for route, (kinds, fn) in rs.items():
                if kind not in kinds:
                    continue
                if route == "samekey":
                    got, _ = trace(emul, lambda k, m, q, s, n, o: emul.emul_verify_samekey(k, q, m, s, n, o), kind, msg, key, sig)
                else:
                    got, _ = trace(emul, fn(kind), kind, msg, key, sig)
                want = S.schedule(model_name(route), u1, u2, d, rpn).codes()
                assert got == want, (route, kind, hex(u1), hex(u2), hex(d))
                checked[route] += 1
    finally:
        emul.emul_set_ecdsa33_exact(0)
    for inv, u1, u2, d in recovery_items():
        assert trace_recovery(emul, inv) == S.schedule("main", u1, u2, d).codes(), (inv, hex(u1), hex(u2), hex(d))
        checked["recovery"] += 1
    assert min(checked.values()) >= 40, checked


def test_constructed_fixture_host_verdicts_match_reference(emul, ref):
    fx = F.load()
    try:
        for kind, msg, key, sig in ((0, fx["ecdsa_msg"], fx["ecdsa_pub33"], fx["ecdsa_sig"]),
                                    (1, fx["ecdsa_msg"], fx["ecdsa_pubxy"], fx["ecdsa_sig"]),
                                    (2, fx["bip340_msg"], fx["bip340_xonly"], fx["bip340_sig"])):
            want = ref_verify(ref, kind, msg, key, sig)
            stored = fx["ref_verdict_%d" % kind]
            assert np.array_equal(want, stored), (kind, "fixture's stored reference verdicts are stale")
            # ECDSA: valid and invalid cases; BIP-340: r is fixed before R is known, so every case is invalid
            assert (want.any() and not want.all()) if kind != 2 else not want.any(), kind
            n = msg.shape[0]
            for exact in (0, 1):
                emul.emul_set_ecdsa33_exact(exact)
                for fn in (emul.emul_verify_batch, emul.emul_verify_small_batch, emul.emul_verify_small_pair_batch):
                    out = np.zeros(n, np.uint8)
                    fn(kind, ptr(msg), ptr(key), ptr(sig), ctypes.c_size_t(n), ptr(out))
                    assert np.array_equal(out, want), (kind, exact, fn.__name__, np.nonzero(out != want)[0])
            if kind != 2:
                out = np.zeros(1, np.uint8)
                for i in range(n):
                    emul.emul_verify_samekey(kind, ptr(key[i]), ptr(msg[i]), ptr(sig[i]), ctypes.c_size_t(1), ptr(out))
                    assert out[0] == want[i], (kind, i, "samekey")
    finally:
        emul.emul_set_ecdsa33_exact(0)


def coverage():
    """{schedule: Counter((step, branch))} over the constructed fixture, per signature kind family"""
    cov = defaultdict(Counter)
    for kind, _, _, _, u1, u2, d, rpn, source in items():
        if source != "constructed" or kind == 1:
            continue
        fam = "bip340" if kind == 2 else "ecdsa"
        for name in S.SCHEDULES:
            for c in S.classes(S.schedule(name, u1, u2, d, rpn), name):
                cov[f"{fam}.{name}"][c] += 1
    # BOLT11 key recovery: the `main` schedule of k_main<SV_KIND_SCHNORR>, with u2 as free as in ECDSA
    for _, u1, u2, d in recovery_items():
        for c in S.classes(S.schedule("main", u1, u2, d), "main"):
            cov["recovery.main"][c] += 1
    return cov


def test_every_reachable_step_class_is_hit():
    cov = coverage()
    for name, reach in S.REACH.items():
        missing = [c for c in reach if not cov[f"ecdsa.{name}"][c]]
        assert not missing, (name, missing)
    missing = [c for c in S.REACH["main"] if not cov["recovery.main"][c]]
    assert not missing, ("recovery.main", missing)
    # BIP-340: the classes that tie u1 to u2*d
    assert cov["bip340.main"][("comb", "double")] and cov["bip340.main"][("comb", "infinity")]
    for c in (("join2", "double"), ("join2", "infinity"), ("join2", "b_inf")):
        assert cov["bip340.small"][c], c
    # the no-sqrt flows hand every trigger to the plain path
    trig = Counter(S.ns_trigger(u1, u2, d, rpn) for kind, _, _, _, u1, u2, d, rpn, src in items() if src == "constructed")
    for t in S.NS_TRIGGERS:
        assert trig[t], t
