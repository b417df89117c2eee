"""CPU-only: soundness of BIP-340 batch verification by random linear combination (batch.cuh), host build of every stage.

A group of 1024 signatures passes on one equation, so its members are accepted without being checked one by one; what
keeps invalid signatures from cancelling inside that equation is the random coefficient a_i of each signature.  Here
batches of valid signatures get pairs of invalid ones that cancel under weak coefficients (all equal, or the ones a known
seed gives) and the per-group verdicts of emul_schnorr_batch are compared with the exact model of the coefficients in
tests/adversarial.py (batch_coefficient, predict_groups).  The same families run on the device in test_gpu_batch_rlc.py."""
import ctypes
import hashlib

import numpy as np
import pytest

from tests import adversarial as adv
from tests import ecc, util

P = util.P
N = adv.N
S = bytes(range(32))
ZERO = bytes(32)
S1 = bytes(range(1, 33))
N_ITEMS = 1024 + 76  # one full group and a ragged one


@pytest.fixture(scope="module")
def batch():
    """N_ITEMS valid BIP-340 signatures (tests/ecc.py), one key and message each: (msg, xonly, sig)."""
    rows = []
    for i in range(N_ITEMS):
        m = hashlib.sha256(b"rlc/msg/%d" % i).digest()
        sig, x = ecc.schnorr_sign(hashlib.sha256(b"rlc/key/%d" % i).digest(), m)
        rows.append((m, x, sig))
    return tuple(np.array([np.frombuffer(r[c], np.uint8) for r in rows]) for c in range(3))


def run(emul, m, k, s, seed):
    """emul_schnorr_batch -> (encoding verdicts, per-group verdicts as a list)"""
    n = m.shape[0]
    ok, gok = np.zeros(n, np.uint8), np.zeros((n + adv.BATCH_GROUP - 1) // adv.BATCH_GROUP, np.uint8)
    sd = np.frombuffer(seed, np.uint8).copy()
    m, k, s = (np.ascontiguousarray(a) for a in (m, k, s))
    emul.emul_schnorr_batch(P(m), P(k), P(s), ctypes.c_size_t(n), P(sd), P(ok), P(gok))
    return ok, [int(g) for g in gok]


def one_by_one(emul, m, k, s):
    out = np.zeros(m.shape[0], np.uint8)
    m, k, s = (np.ascontiguousarray(a) for a in (m, k, s))
    emul.emul_verify_batch(2, P(m), P(k), P(s), ctypes.c_size_t(m.shape[0]), P(out))
    return out


def _lift_x(x):
    y = pow((x ** 3 + 7) % adv.P, (adv.P + 1) // 4, adv.P)
    return x, (y if y % 2 == 0 else adv.P - y)


def unit_sum(m, k, s, idx):
    """sum over idx of R_i + e_i*P_i - s_i*G, every coefficient 1: None (infinity) iff the items cancel"""
    acc = None
    for i in idx:
        r, px = bytes(s[i, :32]), bytes(k[i])
        e = int.from_bytes(ecc.tagged_hash("BIP0340/challenge", r + px + bytes(m[i])), "big") % N
        acc = adv.add(acc, _lift_x(int.from_bytes(r, "big")))
        acc = adv.add(acc, adv.mul(e, _lift_x(int.from_bytes(px, "big"))))
        acc = adv.add(acc, adv.mul(-int.from_bytes(bytes(s[i, 32:]), "big"), adv.G))
    return acc


@pytest.mark.parametrize("construction", ["cancel_pair", "swap_nonce_pair"])
def test_pairs_cancelling_under_equal_coefficients_fail_their_groups(emul, batch, construction):
    """Two invalid signatures that cancel when every a_i is the same -- s_i + d with s_j - d (cancel_pair), or each signed
    with the other's nonce point (swap_nonce_pair) -- one pair in group 0 including item 0, one in the ragged group
    including item n - 1: each group fails under every seed.  With coefficient 1 each pair adds nothing (checked with
    Python integers), so a batch whose coefficients do not depend on the index would accept all four."""
    m, k, s = batch
    n = m.shape[0]
    pairs = ((0, 500), (1030, n - 1))
    m1, k1, s1 = m, k, s
    for i, j in pairs:
        if construction == "cancel_pair":
            s1 = adv.cancel_pair(s1, i, j, d=12345)
        else:
            m1, k1, s1 = adv.swap_nonce_pair(m1, k1, s1, i, j)
    for i, j in pairs:
        assert unit_sum(m1, k1, s1, (i, j)) is None
    touched = [i for p in pairs for i in p]
    assert not one_by_one(emul, m1[touched], k1[touched], s1[touched]).any()
    for seed in (S, ZERO):
        ok, gok = run(emul, m1, k1, s1, seed)
        assert ok.all() and gok == [0, 0], seed.hex()
        if construction == "cancel_pair":
            assert adv.predict_groups(n, seed, adv.s_shifts(s, s1)) == gok


@pytest.mark.parametrize("built_for", [S, ZERO], ids=["S", "zero"])
@pytest.mark.parametrize("i,j", [(3, 700), (1030, 1090)])
def test_forged_pair_passes_under_its_own_seed_only(emul, batch, built_for, i, j):
    """forge_pair(seed) makes two invalid signatures whose shifts cancel under that seed's coefficients (items i and j
    counted in the whole batch, so the pair in the ragged group pins the global index): the group passes when verified
    with that seed -- the model of the coefficients is exact -- and fails with any other seed."""
    m, k, s = batch
    n = m.shape[0]
    s1 = adv.forge_pair(s, i, j, built_for, d=7)
    assert not one_by_one(emul, m[[i, j]], k[[i, j]], s1[[i, j]]).any()
    g = i // adv.BATCH_GROUP
    for seed in (S, ZERO, S1):
        ok, gok = run(emul, m, k, s1, seed)
        want = adv.predict_groups(n, seed, adv.s_shifts(s, s1))
        assert want == ([1, 1] if seed == built_for else [int(x != g) for x in range(2)]), seed.hex()
        assert ok.all() and gok == want, seed.hex()


def test_forged_pair_across_the_group_boundary(emul, batch):
    """A pair forged for seed S at items 1023 and 1024 sits in two equations: each gets one uncancelled shift, both fail."""
    m, k, s = batch
    s1 = adv.forge_pair(s, 1023, 1024, S)
    ok, gok = run(emul, m, k, s1, S)
    assert ok.all() and gok == [0, 0] == adv.predict_groups(m.shape[0], S, adv.s_shifts(s, s1))


def test_encoding_failures_add_nothing_to_a_forged_group(emul, batch):
    """Encoding failures (r >= p, s >= n, x not on the curve) next to a pair forged for S in group 0: they are excluded with
    verdict 0 and add exactly nothing to the equation, so the forged pair still cancels and the group passes."""
    m, k, s = batch
    s1 = adv.forge_pair(s, 3, 700, S)
    k1 = k.copy()
    s1[10, :32] = 255  # r >= p
    s1[11, 32:] = 255  # s >= n
    k1[12] = 0
    k1[12, 31] = 5     # x = 5 is not on the curve
    idx = [3, 700, 10, 11, 12]
    assert not one_by_one(emul, m[idx], k1[idx], s1[idx]).any()
    ok, gok = run(emul, m, k1, s1, S)
    assert list(np.nonzero(ok == 0)[0]) == [10, 11, 12] and gok == [1, 1]


def test_pair_forged_for_the_wrong_seed_fails_only_its_group(emul, batch):
    """Pairs forged in both groups, the one in group 1 for the zero seed: verified with S, only group 1 fails."""
    m, k, s = batch
    s1 = adv.forge_pair(adv.forge_pair(s, 3, 700, S), 1030, 1090, ZERO)
    ok, gok = run(emul, m, k, s1, S)
    assert ok.all() and gok == [1, 0] == adv.predict_groups(m.shape[0], S, adv.s_shifts(s, s1))
