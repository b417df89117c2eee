"""GPU: signatures forged for 64-byte keys off secp256k1 are refused on every route that takes a 64-byte key.

The cases of tests/golden/invalid_curve.npz (tests/invalid_curve.py) are valid on the key's own curve y^2 = x^3 + b', and
the engine's ladder, which never uses the curve constant, computes exactly what they need: only the key's decode flag keeps
their verdict at 0.  tests/test_invalid_curve_host.py shows that a host build without any one of the four places that
carry that flag into the verdict accepts every case.  Here each case goes through the device's routes among valid 64-byte
-key signatures (device generator, about 1 % of messages flipped), at the first, middle and last positions and on both
sides of the 32-item inversion batch and the 16-item final batch: the forged items get the reference's verdict (0) and
every neighbour keeps its own.  The launch counter pins the route of each call (tests/test_gpu_routes.py).  Kind 1 has no
flow without the square root, so every call runs with that switch on and off and no verdict may move.

Not covered here, because no such forgery exists: the transaction checks (check_tx_sigs, grind_tx_fee), whose message is
a BIP143 digest nobody can steer to 0; 33-byte and x-only keys, whose off-curve x lifts to a fixed point of essentially
random order (the one cheap small order, 3, needs x^3 = -4, and its table meets infinity like the suite's key.x=0 case),
and whose flows without the square root refuse a non-residue by algebra; and the drop-in's check_signed_hash, whose
x || y comes from a parsed struct pubkey."""
import numpy as np
import pytest

from tests import invalid_curve as I
from tests.test_gpu_routes import _mixed_batch, _mixed_routes, _wave, counted, route, synth

pytestmark = pytest.mark.gpu
EDGES = (0, 1, 15, 16, 17, 31, 32, 33)
REACHED = {}  # (route, api) -> {case index}


@pytest.fixture(scope="module")
def fx():
    return I.load()


@pytest.fixture()
def defaults(engine):
    sm = engine.small_max()
    yield sm
    engine.set_small_max(sm)
    engine.set_nosqrt(True)


def _positions(n, count):
    """where the forged items go in a batch of n: the edges of the first 32- and 16-item units, the middle, the end, and
    enough evenly spread positions for `count` items when n allows"""
    pos = {p for p in EDGES if p < n} | {n // 2, n - 1}
    if n >= 4 * count:
        pos |= set(np.linspace(40, n - 2, count, dtype=np.int64).tolist())
    return np.array(sorted(pos))


def _placed(bg, n, fx):
    """the first n background items with forged cases put in (case k % cases at the k-th position): (msg, key, sig, want,
    positions, case index per position)"""
    msg, key, sig, want = (np.ascontiguousarray(a[:n]).copy() for a in bg)
    cases = fx["msg"].shape[0]
    pos = _positions(n, cases)
    idx = np.arange(pos.size) % cases
    msg[pos], key[pos], sig[pos], want[pos] = fx["msg"][idx], fx["key"][idx], fx["sig"][idx], fx["ref_verdict"][idx]
    return msg, key, sig, want, pos, idx


def _check(got, want, pos, what):
    bad = np.nonzero(np.asarray(got) != want)[0]
    forged = sorted(set(bad.tolist()) & set(pos.tolist()))
    assert not bad.size, f"{what}: forged items accepted at {forged[:8]}, neighbour verdicts changed at " \
                         f"{sorted(set(bad.tolist()) - set(forged))[:8]}"


def _reached(r, api, idx):
    REACHED.setdefault((r, api), set()).update(int(i) for i in idx)


def test_verify_and_verify_device(engine, fx, defaults):
    """sv_verify_host and sv_verify_device with a verdict bitmap, kind 1, at n = 1 (each case alone), small_max,
    small_max + 1 and one wave +- 1: the small-batch kernel and k_main<ECDSA_XY>"""
    import torch
    sm = defaults
    sizes = sorted({sm, sm + 1, _wave(engine) - 1, _wave(engine), _wave(engine) + 1})
    assert sm >= 4 * fx["msg"].shape[0]
    (dm, dk, ds), want_all = synth(engine, 1, max(sizes), 9100)
    bg = tuple(t.cpu().numpy() for t in (dm, dk, ds)) + (want_all,)
    cases = fx["msg"].shape[0]
    for nosqrt in (True, False):
        engine.set_nosqrt(nosqrt)
        for i in range(cases):
            got = counted(engine, lambda: engine.verify(1, fx["msg"][i:i + 1], fx["key"][i:i + 1], fx["sig"][i:i + 1]),
                          route(engine, 1, 1, nosqrt))
            assert got[0] == fx["ref_verdict"][i] == 0, (i, nosqrt)
        _reached("small", "verify n=1", range(cases))
        for n in sizes:
            r = route(engine, 1, n, nosqrt)
            msg, key, sig, want, pos, idx = _placed(bg, n, fx)
            assert 0 < want.sum() < n
            got = counted(engine, lambda: engine.verify(1, msg, key, sig), r)
            _check(got, want, pos, f"verify n = {n} nosqrt {nosqrt}")
            _reached(r, "verify", idx)
            d = [torch.from_numpy(a).cuda() for a in (msg, key, sig)]
            nw = (n + 31) // 32
            out = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
            bm = torch.full((nw,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            counted(engine, lambda: engine.verify_device(1, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), n,
                                                         out.data_ptr(), bm.data_ptr()), r, "bitmap")
            engine.sync()
            _check(out.cpu().numpy(), want, pos, f"verify_device n = {n} nosqrt {nosqrt}")
            bits = np.unpackbits(bm.cpu().numpy().view(np.uint8), bitorder="little")[:n]
            _check(bits, want, pos, f"verdict bitmap n = {n} nosqrt {nosqrt}")
            _reached(r, "verify_device", idx)
    for r in ("small", "main_ecdsa_xy"):
        for api in ("verify", "verify_device"):
            assert REACHED[(r, api)] == set(range(cases)), (r, api)
    print(f"sizes {sizes}, small_max {sm}: every one of {cases} cases on " + ", ".join(sorted(f"{r}/{a}" for r, a in REACHED)))


def _mixed_with_forged(engine, counts, seed, fx):
    """an interleaved batch of tests/test_gpu_routes.py with forged items on kind-1 slots: (kinds, msg, key64, sig, want,
    positions)"""
    kinds, msg, key, sig, want = _mixed_batch(engine, counts, seed)
    slots = np.nonzero(kinds == 1)[0]
    sel = slots[_positions(slots.size, fx["msg"].shape[0])]
    idx = np.arange(sel.size) % fx["msg"].shape[0]
    msg[sel], key[sel], sig[sel], want[sel] = fx["msg"][idx], fx["key"][idx], fx["sig"][idx], fx["ref_verdict"][idx]
    return kinds, msg, key, sig, want, sel, idx


def test_mixed_batches(engine, fx, defaults):
    """sv_verify_mixed_host and sv_verify_mixed_device with the forged items among kind-1 items interleaved with kinds 0
    and 2, the kind-1 count on both sides of small_max"""
    import torch
    sm = defaults
    for ci, counts in enumerate([(sm + 1, sm + 1, sm), (sm, sm, sm + 1)]):
        kinds, msg, key, sig, want, pos, idx = _mixed_with_forged(engine, counts, 9200 + 10 * ci, fx)
        n = kinds.shape[0]
        for nosqrt in (True, False):
            engine.set_nosqrt(nosqrt)
            rs = _mixed_routes(engine, counts, nosqrt)
            got = counted(engine, lambda: engine.verify_mixed(kinds, msg, key, sig), *rs)
            _check(got, want, pos, f"verify_mixed counts {counts} nosqrt {nosqrt}")
            st = torch.cuda.Stream()
            dk, dm, dkey, ds = (torch.from_numpy(a).cuda() for a in (kinds, msg, key, sig))
            out = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            rc = counted(engine, lambda: engine.lib.sv_verify_mixed_device(engine._ctx, dk.data_ptr(), dm.data_ptr(),
                                                                           dkey.data_ptr(), ds.data_ptr(), n, out.data_ptr(),
                                                                           st.cuda_stream), *rs)
            assert rc == 0, engine.lib.sv_last_error(engine._ctx)
            st.synchronize()
            _check(out.cpu().numpy(), want, pos, f"sv_verify_mixed_device counts {counts} nosqrt {nosqrt}")
            _reached(route(engine, 1, counts[1], nosqrt), "mixed", idx)
    assert REACHED[("small", "mixed")] == REACHED[("main_ecdsa_xy", "mixed")] == set(range(fx["msg"].shape[0]))


def test_deferral_queue(engine, fx, defaults):
    """enqueue / flush: the forged items among items of all three kinds, the kind-1 count on both sides of small_max"""
    sm = defaults
    for ci, counts in enumerate([(sm + 1, sm + 1, sm), (sm, sm, sm + 1)]):
        kinds, msg, key, sig, want, pos, idx = _mixed_with_forged(engine, counts, 9300 + 10 * ci, fx)
        known = np.nonzero(kinds < 3)[0]
        # positions in the queue: the known items keep their order
        qpos = np.searchsorted(known, pos)
        for nosqrt in (True, False):
            engine.set_nosqrt(nosqrt)
            assert engine.pending() == 0
            for i in known:
                engine.enqueue(int(kinds[i]), msg[i], key[i, :{0: 33, 1: 64, 2: 32}[int(kinds[i])]], sig[i])
            rs = [route(engine, kind, c, nosqrt) for kind, c in enumerate(counts) if c]
            got = counted(engine, engine.flush, *rs)
            _check(got, want[known], qpos, f"flush counts {counts} nosqrt {nosqrt}")
            assert engine.pending() == 0
            _reached(route(engine, 1, counts[1], nosqrt), "flush", idx)
    assert REACHED[("small", "flush")] == REACHED[("main_ecdsa_xy", "flush")] == set(range(fx["msg"].shape[0]))


def test_same_key(engine, fx, defaults):
    """sv_verify_samekey_host with a forged key shared by every signature of the batch: its own cases alone, tiled to
    small_max (small-batch kernel) and to small_max + 1 (k_sharedkey_build + k_main_shared); every verdict 0"""
    sm = defaults
    for g in np.unique(fx["group"]):
        sel = np.nonzero(fx["group"] == g)[0]
        key = fx["key"][sel[0]]
        for nosqrt in (True, False):
            engine.set_nosqrt(nosqrt)
            for n, r in ((sel.size, "small"), (sm, "small"), (sm + 1, "samekey_shared")):
                reps = -(-n // sel.size)
                m, s = (np.ascontiguousarray(np.tile(fx[a][sel], (reps, 1))[:n]) for a in ("msg", "sig"))
                want = np.tile(fx["ref_verdict"][sel], reps)[:n]
                got = counted(engine, lambda: engine.verify_samekey(1, key, m, s), r)
                assert np.array_equal(got, want), (int(g), n, nosqrt, np.nonzero(got)[0][:8])
                _reached(r, "samekey", sel)
    assert REACHED[("small", "samekey")] == REACHED[("samekey_shared", "samekey")] == set(range(fx["msg"].shape[0]))
