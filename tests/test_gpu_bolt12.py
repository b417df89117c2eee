"""BOLT12 signatures on the device (sv_verify_bolt12_host, bolt12_check_signature) against the fixture.

tests/golden/bolt12_vectors.npz carries the reference's status and sighash for every item (tests/test_bolt12_host.py
keeps it honest); here the whole path runs on the GPU: parse, Merkle root and sighash kernels, then BIP-340 through the
small-batch kernel or the throughput kernels, with and without the square-root-free flow.
"""
import ctypes
import time

import numpy as np
import pytest

from tests import bolt12, ecc

pytestmark = pytest.mark.gpu
SV_OK, SV_ERR_ARG = 0, -4


@pytest.fixture(scope="module")
def fx():
    return bolt12.load_fixture()


def _groups(fx):
    """item indices per (messagename, fieldname): one call takes one tag"""
    return [(ni, np.nonzero(fx["names"] == ni)[0]) for ni in range(len(bolt12.NAMES))]


def _run(engine, fx, idx, ni):
    off, ln = fx["off"][idx], fx["len"][idx]
    return engine.verify_bolt12_spans(*bolt12.NAMES[ni], fx["blob"], off, ln, fx["xonly"][idx], fx["sig"][idx],
                                      want_sighash=True)


@pytest.mark.parametrize("small_max", [None, 0], ids=["small_batch_kernel", "throughput_kernels"])
@pytest.mark.parametrize("nosqrt", [1, 0], ids=["nosqrt", "plain"])
def test_fixture_every_item(engine, fx, small_max, nosqrt):
    default = engine.small_max()
    try:
        if small_max is not None:
            engine.set_small_max(small_max)
        engine.set_nosqrt(nosqrt)
        for ni, idx in _groups(fx):
            status, sh = _run(engine, fx, idx, ni)
            np.testing.assert_array_equal(status, fx["status"][idx].astype(np.int32))
            np.testing.assert_array_equal(sh, fx["sighash"][idx])
    finally:
        engine.set_small_max(default)
        engine.set_nosqrt(1)


def test_one_call_per_item(engine, fx):
    n = len(fx["status"])
    for i in list(range(0, n, 17)) + [i for i in range(n) if fx["len"][i] > 20000 or fx["len"][i] == 0]:
        ni = int(fx["names"][i])
        status, sh = _run(engine, fx, np.array([i]), ni)
        assert status[0] == fx["status"][i] and sh[0].tobytes() == fx["sighash"][i].tobytes(), i


class TlvField(ctypes.Structure):
    """struct tlv_field (wire/tlvstream.h:16-27)"""
    _fields_ = [("meta", ctypes.c_void_p), ("numtype", ctypes.c_uint64), ("length", ctypes.c_size_t),
                ("value", ctypes.POINTER(ctypes.c_uint8))]


def test_dropin_bolt12_check_signature(engine, fx):
    """CLN's own signature, driven with tal-style field arrays (the length comes from the tal_bytelen hook)"""
    lib = engine.lib
    sizes = {}
    hook = ctypes.CFUNCTYPE(ctypes.c_size_t, ctypes.c_void_p)(lambda p: sizes[p])
    lib.cln_sigverify_set_tx_hooks.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.bolt12_check_signature.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.bolt12_check_signature.restype = ctypes.c_bool
    lib.cln_sigverify_set_tx_hooks(ctypes.cast(hook, ctypes.c_void_p), None)
    try:
        streams = bolt12.streams(fx)
        checked = 0
        for i in range(0, len(streams), 7):
            if fx["status"][i] < 0:
                continue  # not a stream CLN's parser produces fields from
            conv = ecc.pubkey_convert(b"\x02" + fx["xonly"][i].tobytes())
            if conv is None:
                continue  # no struct pubkey has this x
            xy = conv[1]
            pub = (ctypes.c_uint8 * 64).from_buffer_copy(xy[31::-1] + xy[:31:-1])  # secp256k1_pubkey: LE limbs
            sig = (ctypes.c_uint8 * 64).from_buffer_copy(fx["sig"][i].tobytes())
            fields = bolt12.parse_fields(streams[i])
            arr = (TlvField * max(len(fields), 1))()
            keep = []
            for k, (t, _vo, v) in enumerate(fields):
                buf = (ctypes.c_uint8 * max(len(v), 1)).from_buffer_copy(v + b"\0")
                keep.append(buf)
                arr[k] = TlvField(None, t, len(v), ctypes.cast(buf, ctypes.POINTER(ctypes.c_uint8)))
            sizes[ctypes.addressof(arr)] = len(fields) * ctypes.sizeof(TlvField)
            mn, fn = bolt12.NAMES[fx["names"][i]]
            got = lib.bolt12_check_signature(ctypes.addressof(arr), mn, fn, ctypes.addressof(pub), ctypes.addressof(sig))
            assert got == (fx["status"][i] == 1), i
            checked += 1
        assert checked > 100
    finally:
        lib.cln_sigverify_set_tx_hooks(None, None)


def test_large_tiled_batch(engine, fx):
    """>= 200,000 streams in one call (throughput kernels), tiled from the fixture, with seeded signature corruptions"""
    idx0 = np.nonzero(fx["names"] == 0)[0]
    reps = -(-200_000 // len(idx0))
    idx = np.tile(idx0, reps)
    rng = np.random.default_rng(12)
    sig = fx["sig"][idx].copy()
    want = fx["status"][idx].astype(np.int32)
    # corrupt only items whose answer is then certain: a flipped bit of a valid signature never verifies, and -1 stays -1.
    # (An invalid item may be a fixture variant with one flipped signature bit, which a second flip can undo.)
    bad = (rng.random(len(idx)) < 0.1) & (want != 0)
    pos = rng.integers(0, 64, size=len(idx))
    sig[np.nonzero(bad)[0], pos[bad]] ^= (1 << rng.integers(0, 8, size=int(bad.sum()))).astype(np.uint8)
    want[bad & (want == 1)] = 0
    status, sh = engine.verify_bolt12_spans(*bolt12.NAMES[0], fx["blob"], fx["off"][idx], fx["len"][idx], fx["xonly"][idx],
                                            sig, want_sighash=True)
    assert len(idx) >= 200_000
    np.testing.assert_array_equal(status, want)
    np.testing.assert_array_equal(sh, fx["sighash"][idx])


def test_timing_belongs_to_its_call(engine, fx):
    """the splits of a BOLT12 call fit inside it, and a later verification of ~100,000 signatures leaves them as they
    were"""
    idx = np.nonzero(fx["names"] == 0)[0]
    big = np.tile(idx, -(-100_000 // len(idx)))
    engine.set_profiling(True)
    try:
        _run(engine, fx, idx, 0)  # warm-up
        t = time.perf_counter()
        _run(engine, fx, idx, 0)
        wall = (time.perf_counter() - t) * 1e3
        first = engine.last_bolt12_timing()
        engine.verify(2, fx["sighash"][big], fx["xonly"][big], fx["sig"][big])
        assert engine.last_bolt12_timing() == first
        assert min(first) > 0 and sum(first) <= wall, (first, wall)
    finally:
        engine.set_profiling(False)


def test_arguments(engine):
    lib, ctx = engine.lib, engine._ctx
    blob = np.frombuffer(bolt12.record(1, b"abc"), np.uint8)
    x, s = np.zeros(32, np.uint8), np.zeros(64, np.uint8)
    st = np.zeros(1, np.int32)
    off, ln = np.array([0], np.uint64), np.array([blob.size], np.uint32)
    args = [blob.ctypes.data, blob.size, off.ctypes.data, ln.ctypes.data, x.ctypes.data, s.ctypes.data, 1, st.ctypes.data, None]
    assert lib.sv_verify_bolt12_host(ctx, b"invoice", b"signature", *args) == SV_OK
    assert st[0] == 0  # parses; the all-zero key is not on the curve
    for o, n in ((0, blob.size + 1), (blob.size + 1, 0), (2, blob.size - 1)):
        off[0], ln[0] = o, n
        assert lib.sv_verify_bolt12_host(ctx, b"invoice", b"signature", *args) == SV_ERR_ARG, (o, n)
    off[0], ln[0] = 0, blob.size
    assert lib.sv_verify_bolt12_host(None, b"invoice", b"signature", *args) == SV_ERR_ARG
    assert lib.sv_verify_bolt12_host(ctx, None, b"signature", *args) == SV_ERR_ARG
    assert lib.sv_verify_bolt12_host(ctx, b"invoice", None, *args) == SV_ERR_ARG
    for k in (0, 2, 3, 4, 5, 7):
        a = list(args)
        a[k] = None
        assert lib.sv_verify_bolt12_host(ctx, b"invoice", b"signature", *a) == SV_ERR_ARG, k
    a = list(args)
    a[6] = 0
    a[0] = a[2] = a[3] = a[4] = a[5] = a[7] = None
    assert lib.sv_verify_bolt12_host(ctx, b"invoice", b"signature", *a) == SV_OK  # n = 0
