"""BOLT11 invoice signatures on the device (sv_verify_bolt11_host, bolt11_decode's signature step) against the fixture.

tests/golden/bolt11_vectors.npz carries Core Lightning's answer for every invoice (tests/test_bolt11_host.py keeps it
honest).  Here the whole path runs on the GPU: parse and signing hash, then the `n` invoices through the compressed-key
ECDSA path (small-batch kernel or throughput kernels) and the others through the recovery kernels around the plain-flow
ladder.  Items CLN refuses for a field value the engine does not check are left out of the comparison.
"""
import numpy as np
import pytest

from tests import bolt11

pytestmark = pytest.mark.gpu
SV_OK, SV_ERR_ARG = 0, -4


@pytest.fixture(scope="module")
def fx():
    return bolt11.load_fixture()


def _check(fx, idx, status, node, h):
    e = fx["expected"][idx]
    m = e != bolt11.UNCHECKED
    bad = np.nonzero(m & (status != e))[0]
    assert bad.size == 0, [(int(idx[i]), fx["label_name"][idx[i]], int(status[i]), int(e[i])) for i in bad[:10]]
    signed = m & (e >= 0)
    np.testing.assert_array_equal(h[signed], fx["hash"][idx][signed])
    assert not h[status == -1].any()
    ok = e == 1
    np.testing.assert_array_equal(node[ok], fx["node"][idx][ok])
    assert not node[status != 1].any()


def _run(engine, fx, idx):
    return engine.verify_bolt11_spans(fx["blob"], fx["off"][idx], fx["len"][idx])


@pytest.mark.parametrize("small_max", [None, 0], ids=["small_batch_kernel", "throughput_kernels"])
@pytest.mark.parametrize("nosqrt", [1, 0], ids=["nosqrt", "plain"])
def test_fixture_every_item(engine, fx, small_max, nosqrt):
    default = engine.small_max()
    try:
        if small_max is not None:
            engine.set_small_max(small_max)
        engine.set_nosqrt(nosqrt)
        idx = np.arange(len(fx["ret"]))
        _check(fx, idx, *_run(engine, fx, idx))
    finally:
        engine.set_small_max(default)
        engine.set_nosqrt(1)


def test_batch_sizes(engine, fx):
    """1, 31, 33, 8,192 and 40,000 invoices, and 9,000 `n` invoices: above the small-batch limit on their own"""
    rng = np.random.default_rng(11)
    n_items = len(fx["ret"])
    for size in (1, 31, 33, 8192, 40000):
        idx = rng.integers(0, n_items, size)
        _check(fx, idx, *_run(engine, fx, idx))
    with_n = np.nonzero(fx["label_name"] == "signed_n")[0]
    assert engine.small_max() < 9000
    idx = np.concatenate([with_n[rng.integers(0, len(with_n), 9000)], rng.integers(0, n_items, 1000)])
    _check(fx, idx, *_run(engine, fx, idx))


def test_one_call_per_item(engine, fx):
    for i in range(0, len(fx["ret"]), 29):
        idx = np.array([i])
        _check(fx, idx, *_run(engine, fx, idx))


def test_strings_and_bytes(engine, fx):
    invs = bolt11.invoices(fx)
    idx = np.nonzero(np.isin(fx["label_name"], ["signed", "signed_n", "spec", "long"]))[0]
    given = [invs[i].decode() if k % 2 else invs[i] for k, i in enumerate(idx)]
    _check(fx, idx, *engine.verify_bolt11(given))


def _special(fx):
    """a -1, a 0, an `n` item and a recovery-id-3 item"""
    lab, e = fx["label_name"], fx["expected"]
    # make_bolt11.py builds the recid23 items in pairs, recovery id 2 then 3
    pick = [np.nonzero(lab == "charset")[0][0], np.nonzero(lab == "recid_high")[0][0],
            np.nonzero(lab == "signed_n")[0][0], np.nonzero(lab == "recid23")[0][1]]
    assert [e[i] for i in pick] == [-1, 0, 1, 1]
    return pick


@pytest.mark.parametrize("small_max", [None, 0], ids=["small_batch_kernel", "throughput_kernels"])
def test_isolation(engine, fx, small_max):
    """a -1, a 0, an `n` item and a recovery-id-3 item at every offset of a batch change no other item's answer"""
    base = np.nonzero(np.isin(fx["label_name"], ["signed", "signed_n", "high_s"]))[0][:47]
    default = engine.small_max()
    try:
        if small_max is not None:
            engine.set_small_max(small_max)
        for sp in _special(fx):
            for pos in range(len(base) + 1):
                idx = np.insert(base, pos, sp)
                _check(fx, idx, *_run(engine, fx, idx))
    finally:
        engine.set_small_max(default)


def test_timing(engine, fx):
    engine.set_profiling(True)
    try:
        idx = np.arange(len(fx["ret"]))
        _check(fx, idx, *_run(engine, fx, idx))
        parse_ms, curve_ms = engine.last_bolt11_timing()
        assert parse_ms > 0 and curve_ms > 0
    finally:
        engine.set_profiling(False)


def test_arguments(engine, fx):
    lib, ctx = engine.lib, engine._ctx
    blob = np.frombuffer(bolt11.invoices(fx)[0], np.uint8)
    st = np.zeros(1, np.int32)
    node = np.zeros(33, np.uint8)
    off, ln = np.array([0], np.uint64), np.array([blob.size], np.uint32)
    args = [blob.ctypes.data, blob.size, off.ctypes.data, ln.ctypes.data, 1, st.ctypes.data, node.ctypes.data, None]
    assert lib.sv_verify_bolt11_host(ctx, *args) == SV_OK
    for o, n in ((0, blob.size + 1), (blob.size + 1, 0), (2, blob.size - 1)):
        off[0], ln[0] = o, n
        assert lib.sv_verify_bolt11_host(ctx, *args) == SV_ERR_ARG, (o, n)
    off[0], ln[0] = 0, blob.size
    assert lib.sv_verify_bolt11_host(None, *args) == SV_ERR_ARG
    for k in (0, 2, 3, 5, 6):
        a = list(args)
        a[k] = None
        assert lib.sv_verify_bolt11_host(ctx, *a) == SV_ERR_ARG, k
    a = [None, 0, None, None, 0, None, None, None]
    assert lib.sv_verify_bolt11_host(ctx, *a) == SV_OK  # n = 0
