"""BOLT12 signatures under several tags in one call (sv_verify_bolt12_tagged_host) against the fixture.

The fixture (tests/golden/bolt12_vectors.npz) records the reference's status, Merkle root and sighash of every item.  Here
the items of both of its tags go through one call, interleaved in fixture order, on the small-batch kernel and on the
throughput kernels; a large tiled batch also carries made-up tags, whose expected sighashes are computed with hashlib
from the reference's Merkle roots.
"""
import ctypes
import hashlib

import numpy as np
import pytest

from tests import bolt12

pytestmark = pytest.mark.gpu
SV_OK, SV_ERR_ARG = 0, -4


@pytest.fixture(scope="module")
def fx():
    return bolt12.load_fixture()


def _tagged(engine, fx, idx, tags, tag_of, sig=None):
    return engine.verify_bolt12_tagged(tags, tag_of, fx["blob"], fx["off"][idx], fx["len"][idx], fx["xonly"][idx],
                                       fx["sig"][idx] if sig is None else sig, want_sighash=True)


@pytest.mark.parametrize("small_max", [None, 0], ids=["small_batch_kernel", "throughput_kernels"])
@pytest.mark.parametrize("nosqrt", [1, 0], ids=["nosqrt", "plain"])
def test_fixture_one_call_all_tags(engine, fx, small_max, nosqrt):
    default = engine.small_max()
    try:
        if small_max is not None:
            engine.set_small_max(small_max)
        engine.set_nosqrt(nosqrt)
        idx = np.arange(len(fx["status"]))
        status, sh = _tagged(engine, fx, idx, bolt12.NAMES, fx["names"])
        np.testing.assert_array_equal(status, fx["status"].astype(np.int32))
        np.testing.assert_array_equal(sh, fx["sighash"])
    finally:
        engine.set_small_max(default)
        engine.set_nosqrt(1)


def test_same_as_one_call_per_tag(engine, fx):
    idx = np.arange(len(fx["status"]))
    status, sh = _tagged(engine, fx, idx, bolt12.NAMES, fx["names"])
    for ni, (mn, fn) in enumerate(bolt12.NAMES):
        sel = np.nonzero(fx["names"] == ni)[0]
        s1, h1 = engine.verify_bolt12_spans(mn, fn, fx["blob"], fx["off"][sel], fx["len"][sel], fx["xonly"][sel],
                                            fx["sig"][sel], want_sighash=True)
        np.testing.assert_array_equal(status[sel], s1)
        np.testing.assert_array_equal(sh[sel], h1)
    # one tag only, through the tagged entry point: the same as sv_verify_bolt12_host
    sel = np.nonzero(fx["names"] == 1)[0]
    s2, h2 = _tagged(engine, fx, sel, [bolt12.NAMES[1]], np.zeros(len(sel), np.uint32))
    np.testing.assert_array_equal(s2, status[sel])
    np.testing.assert_array_equal(h2, sh[sel])


def _tagged_hash(tag, root32):
    t = hashlib.sha256(tag).digest()
    return hashlib.sha256(t + t + root32).digest()


def test_large_tiled_batch_random_tags(engine, fx):
    """>= 200,000 streams under a table of 6 tags: the fixture's two and four made up (one of them longer than a SHA-256
    block, so its midstate takes several compressions).  Each stream gets its own fixture tag or a made-up one at random.
    Not the other fixture tag: the fixture holds streams signed under one name and recorded under the other, whose answer
    under the signing name it does not record."""
    tags = list(bolt12.NAMES) + [(b"offer", b"signature"), (b"invoice", b"payer_signature"), (b"x", b"y"),
                                 (b"invoice_request_" + b"m" * 150, b"f" * 70)]
    n0 = len(fx["status"])
    reps = -(-200_000 // n0)
    idx = np.tile(np.arange(n0), reps)
    n = len(idx)
    rng = np.random.default_rng(2026)
    own = rng.random(n) < 0.35
    tag_of = np.where(own, fx["names"][idx], rng.integers(len(bolt12.NAMES), len(tags), size=n)).astype(np.uint32)
    sig = fx["sig"][idx].copy()
    fst = fx["status"][idx].astype(np.int32)
    # no fixture signature was made under a made-up tag
    want = np.where(fst < 0, -1, np.where(own, fst, 0)).astype(np.int32)
    # corrupt only items whose answer is then certain: a flipped bit of a valid signature never verifies, -1 stays -1
    bad = (rng.random(n) < 0.1) & (want != 0)
    pos = rng.integers(0, 64, size=n)
    sig[np.nonzero(bad)[0], pos[bad]] ^= (1 << rng.integers(0, 8, size=int(bad.sum()))).astype(np.uint8)
    want[bad & (want == 1)] = 0
    # expected sighashes: the fixture's where the item carries its own tag, else the tagged hash of the reference's root
    full = [b"lightning" + mn + fn for mn, fn in tags]
    table = np.zeros((n0, len(tags), 32), np.uint8)
    for i in range(n0):
        if fx["status"][i] < 0:
            continue  # zeros: never hashed
        root = fx["merkle"][i].tobytes()
        for t, tag in enumerate(full):
            table[i, t] = np.frombuffer(_tagged_hash(tag, root), np.uint8)
        assert table[i, fx["names"][i]].tobytes() == fx["sighash"][i].tobytes(), i  # the fixture agrees with hashlib
    status, sh = _tagged(engine, fx, idx, tags, tag_of, sig=sig)
    assert n >= 200_000 and np.bincount(tag_of, minlength=len(tags)).min() > 20_000
    np.testing.assert_array_equal(status, want)
    np.testing.assert_array_equal(sh, table[idx, tag_of])


def test_arguments(engine):
    lib, ctx = engine.lib, engine._ctx
    blob = np.frombuffer(bolt12.record(1, b"abc") * 2, np.uint8)
    x, s = np.zeros((2, 32), np.uint8), np.zeros((2, 64), np.uint8)
    st = np.zeros(2, np.int32)
    off = np.array([0, 5], np.uint64)
    ln = np.array([5, 5], np.uint32)
    mn = (ctypes.c_char_p * 2)(b"invoice", b"invoice_request")
    fn = (ctypes.c_char_p * 2)(b"signature", b"signature")
    tag_of = np.array([1, 0], np.uint32)

    def call(ntags=2, m=mn, f=fn, t=tag_of, n=2, blob_p=blob.ctypes.data):
        return lib.sv_verify_bolt12_tagged_host(ctx, ntags, m, f, t.ctypes.data if t is not None else None, blob_p,
                                                blob.size, off.ctypes.data, ln.ctypes.data, x.ctypes.data, s.ctypes.data, n,
                                                st.ctypes.data, None)

    assert call() == SV_OK and list(st) == [0, 0]  # both parse; the all-zero key is not on the curve
    tag_of[0] = 2
    assert call() == SV_ERR_ARG  # tag_of out of range
    tag_of[0] = 1
    assert call(ntags=0) == SV_ERR_ARG  # no tags for two streams
    assert call(t=None) == SV_ERR_ARG
    assert call(m=None) == SV_ERR_ARG and call(f=None) == SV_ERR_ARG
    for arr in (mn, fn):
        keep = arr[1]
        arr[1] = None
        assert call() == SV_ERR_ARG  # a NULL name
        arr[1] = keep
    off[1] = 6
    assert call() == SV_ERR_ARG  # a span past the blob
    off[1] = 5
    assert call(n=0, t=None, blob_p=None) == SV_OK  # n = 0
    assert call(ntags=0, m=None, f=None, n=0, t=None, blob_p=None) == SV_OK
    assert lib.sv_verify_bolt12_tagged_host(None, 2, mn, fn, tag_of.ctypes.data, blob.ctypes.data, blob.size,
                                            off.ctypes.data, ln.ctypes.data, x.ctypes.data, s.ctypes.data, 2,
                                            st.ctypes.data, None) == SV_ERR_ARG
    assert call() == SV_OK and list(st) == [0, 0]  # the context is still good
