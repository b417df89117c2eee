"""GPU: soundness of BIP-340 batch verification by random linear combination (sv_verify_schnorr_batch_host, batch.cu).

The members of a group whose equation holds get verdict 1 without being verified one by one, so the random coefficients
a_i are the whole argument that an invalid signature cannot hide in a passing group.  The valid base batch comes from the
device generator; pairs of invalid signatures are planted in it that cancel under weak coefficients (all equal, or the
ones a known seed gives, tests/adversarial.py).  Expected verdicts come from the construction (a shifted or swapped
signature is invalid) and are cross-checked with one-by-one verification (engine.verify).  The host build runs the same
families against the exact model of the coefficients in test_host_batch_rlc.py."""
import numpy as np
import pytest
import torch

import lightning_b200 as L
from tests import adversarial as adv

pytestmark = pytest.mark.gpu
S = bytes(range(32))
ZERO = bytes(32)
S1 = bytes(range(1, 33))
SMALL = 1024 + 76  # one full group and a ragged one
BIG = 70_000       # 69 groups: items 65,536 and up need more than 16 bits of index


@pytest.fixture(scope="module")
def base(engine):
    """BIG valid BIP-340 signatures from the device generator, copied to the host: (msg, xonly, sig)."""
    msg = torch.empty((BIG, 32), dtype=torch.uint8, device="cuda")
    key = torch.empty((BIG, 32), dtype=torch.uint8, device="cuda")
    sig = torch.empty((BIG, 64), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.synth_device(L.KIND_SCHNORR, 3401, BIG, msg.data_ptr(), key.data_ptr(), sig.data_ptr())
    engine.sync()
    out = tuple(t.cpu().numpy() for t in (msg, key, sig))
    assert engine.verify(L.KIND_SCHNORR, *out).all()
    return out


def first(base, n):
    """copies of the first n items (tests edit them in place)"""
    return tuple(a[:n].copy() for a in base)


def one_by_one(engine, m, k, s, bad):
    """per-signature verdicts; the construction says exactly the items in `bad` are invalid"""
    want = engine.verify(L.KIND_SCHNORR, m, k, s)
    assert list(np.nonzero(want == 0)[0]) == sorted(bad)
    return want


def batch(engine, m, k, s, seed):
    v, gt, gf = engine.verify_schnorr_batch(m, k, s, seed32=seed)
    assert gt == (m.shape[0] + adv.BATCH_GROUP - 1) // adv.BATCH_GROUP
    return v, gf


@pytest.mark.parametrize("construction", ["cancel_pair", "swap_nonce_pair"])
def test_pairs_cancelling_under_equal_coefficients_fail_their_groups(engine, base, construction):
    """Two invalid signatures that cancel when every a_i is the same -- s_i + d with s_j - d (cancel_pair), or each signed
    with the other's nonce point (swap_nonce_pair) -- one pair in group 0 including item 0, one in the ragged group
    including item n - 1: both groups fail and fall back to one-by-one verification, with a given seed, the zero seed and
    the system's randomness."""
    m, k, s = first(base, SMALL)
    pairs = ((0, 500), (1030, SMALL - 1))
    for i, j in pairs:
        if construction == "cancel_pair":
            s = adv.cancel_pair(s, i, j, d=12345)
        else:
            m, k, s = adv.swap_nonce_pair(m, k, s, i, j)
    want = one_by_one(engine, m, k, s, [i for p in pairs for i in p])
    for seed in (S, ZERO, None):
        v, gf = batch(engine, m, k, s, seed)
        assert np.array_equal(v, want) and gf == 2, seed


FORGED = [(3, 700, SMALL), (1030, 1090, SMALL), (65_540, 66_000, BIG)]


@pytest.mark.parametrize("i,j,n", FORGED)
def test_pair_forged_for_a_known_seed_is_accepted_under_that_seed(engine, base, i, j, n):
    """White-box pin of the coefficients: forge_pair(S) makes two invalid signatures whose shifts cancel exactly under the
    coefficients seed S gives items i and j, so verified with S their group passes and BOTH INVALID SIGNATURES GET VERDICT
    1.  This is asserted on purpose: it is the only place where the suite sees the device's a_i (SHA-256 of the seed and
    the item's 64-bit index in the whole batch -- the ragged-group pair and the pair past item 65,535 pin the index), and
    it shows the rejections in the other tests here come from the coefficients, not from some other check.  It is also
    why a seed the signers can learn breaks the batch's soundness."""
    m, k, s = first(base, n)
    s = adv.forge_pair(s, i, j, S)
    one_by_one(engine, m, k, s, [i, j])
    v, gf = batch(engine, m, k, s, S)
    assert gf == 0 and v.all()


@pytest.mark.parametrize("i,j,n", FORGED)
def test_pair_forged_for_a_known_seed_is_rejected_under_other_seeds(engine, base, i, j, n):
    """The same forged batches verified with the zero seed, another fixed seed and twice with the system's randomness:
    exactly the forged pair's group fails, and every verdict is the one-by-one one."""
    m, k, s = first(base, n)
    s = adv.forge_pair(s, i, j, S)
    want = one_by_one(engine, m, k, s, [i, j])
    for seed in (ZERO, S1, None, None):
        v, gf = batch(engine, m, k, s, seed)
        assert np.array_equal(v, want) and gf == 1, seed


def test_pair_forged_for_the_zero_seed_is_rejected_without_a_seed(engine, base):
    """A pair forged for the all-zero seed passes when that seed is passed in, and fails when the seed is left to the
    engine (NULL: taken from getrandom()), so a missing seed does not become a fixed one."""
    m, k, s = first(base, SMALL)
    s = adv.forge_pair(s, 3, 700, ZERO)
    want = one_by_one(engine, m, k, s, [3, 700])
    v, gf = batch(engine, m, k, s, ZERO)
    assert gf == 0 and v.all()
    for _ in range(2):
        v, gf = batch(engine, m, k, s, None)
        assert np.array_equal(v, want) and gf == 1


def test_pair_forged_across_the_group_boundary(engine, base):
    """A pair forged for S at items 1023 and 1024 sits in two equations, one uncancelled shift each: both groups fail."""
    m, k, s = first(base, SMALL)
    s = adv.forge_pair(s, 1023, 1024, S)
    want = one_by_one(engine, m, k, s, [1023, 1024])
    v, gf = batch(engine, m, k, s, S)
    assert np.array_equal(v, want) and gf == 2


def test_encoding_failures_add_nothing_to_a_forged_group(engine, base):
    """Encoding failures (r >= p, s >= n, x not on the curve) in the group of a pair forged for S: they get verdict 0 and
    add exactly nothing to the equation, so the forged pair still cancels and the group passes."""
    m, k, s = first(base, SMALL)
    s = adv.forge_pair(s, 3, 700, S)
    s[10, :32] = 255  # r >= p
    s[11, 32:] = 255  # s >= n
    k[12] = 0
    k[12, 31] = 5     # x = 5 is not on the curve
    one_by_one(engine, m, k, s, [3, 10, 11, 12, 700])
    v, gf = batch(engine, m, k, s, S)
    assert gf == 0 and list(np.nonzero(v == 0)[0]) == [10, 11, 12]


def test_one_pair_forged_for_the_wrong_seed_among_three(engine, base):
    """Pairs forged in groups 0, 1 and 64, the one in group 1 for the zero seed, verified with S: only group 1 fails; its
    forged pair is caught and the other two pass."""
    m, k, s = first(base, BIG)
    s = adv.forge_pair(s, 3, 700, S)
    s = adv.forge_pair(s, 1030, 1090, ZERO)
    s = adv.forge_pair(s, 65_540, 66_000, S)
    want = one_by_one(engine, m, k, s, [3, 700, 1030, 1090, 65_540, 66_000])
    v, gf = batch(engine, m, k, s, S)
    want[[3, 700, 65_540, 66_000]] = 1
    assert gf == 1 and np.array_equal(v, want)
