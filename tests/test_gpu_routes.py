"""GPU: every verification dispatch route at the batch sizes that select it, and launches that overlap on caller streams.

Each entry point picks its kernels at run time from the batch size and the context settings: the small-batch kernel up
to small_max, the throughput kernels above it (compressed-key ECDSA and BIP-340 with or without the square root), the
shared-key kernel for one-key batches, BIP-340 batch verification with its one-by-one fallback.  Every case here names
the route it must take in LAUNCHES and checks it through the engine's launch counter, so a dispatch change that moves a
case to another kernel fails loudly instead of passing on whichever kernel happens to run.

Inputs of a wave and above come from the device generator (sv_synth_device) with message bytes flipped at known
positions, so their verdicts are known by construction; smaller crafted sets go through the reference."""
import numpy as np
import pytest

from tests import adversarial, util

pytestmark = pytest.mark.gpu
KEYLEN = {0: 33, 1: 64, 2: 32}

# Kernel launches each route adds to engine.info()["launches"] (engine.cu: launch_small, launch_verify,
# sv_verify_samekey_host, mixed_device, sv_verify_schnorr_batch_host).
LAUNCHES = {
    "small": 1,            # k_small
    "main_ecdsa33_ns": 4,  # k_prep_inv, k_prep_finish, k_main<ECDSA33 without square root>, k_final_ecdsa33
    "main_ecdsa33": 3,     # k_prep_inv, k_prep_finish, k_main<ECDSA33>
    "main_ecdsa_xy": 3,    # k_prep_inv, k_prep_finish, k_main<ECDSA_XY>
    "main_schnorr": 3,     # k_prep_schnorr, k_main<SCHNORR with or without square root>, k_final_schnorr(_ns)
    "bitmap": 1,           # k_pack_bitmap
    "samekey_shared": 4,   # k_sharedkey_build, k_prep_inv, k_prep_finish, k_main_shared
    "mixed_split": 1,      # k_mixed_index
    "mixed_kind": 2,       # k_mixed_gather and k_mixed_scatter around each kind present
    "sb_batch": 4,         # k_sb_prep, k_sb_window, k_sb_final, k_sb_verdicts
    "sb_fallback": 2,      # k_sb_gather and k_mixed_scatter around the one-by-one re-verification
}


def main_route(kind, nosqrt):
    if kind == 0:
        return "main_ecdsa33_ns" if nosqrt else "main_ecdsa33"
    return "main_ecdsa_xy" if kind == 1 else "main_schnorr"


def route(engine, kind, n, nosqrt):
    """the route one launch_verify of n items must take: up to small_max the small-batch kernel, above it the throughput
    kernels"""
    return "small" if n <= engine.small_max() else main_route(kind, nosqrt)


def counted(engine, fn, *routes):
    """fn() must add exactly the launches of `routes` to the engine's counter"""
    before = engine.info()["launches"]
    r = fn()
    got = engine.info()["launches"] - before
    want = sum(LAUNCHES[x] for x in routes)
    assert got == want, f"{got} launches, the routes {routes} take {want}"
    return r


@pytest.fixture()
def defaults(engine):
    """restore the context's settings whatever a test switched"""
    sm = engine.small_max()
    yield sm
    engine.set_small_max(sm)
    engine.set_nosqrt(True)


def _wave(engine):
    info = engine.info()
    return info["main_grid"] * info["main_block"]


def _bad(n, seed):
    """known positions whose message gets a flipped bit: both ends, the batch edges of the prep (32) and final (16) kernels,
    and about 1 % at random"""
    rng = np.random.default_rng(seed)
    fixed = np.array([0, 1, 15, 16, 17, 31, 32, 33, n // 2, n - 2, n - 1])
    return np.unique(np.concatenate([fixed[(fixed >= 0) & (fixed < n)], rng.choice(n, size=max(n // 100, 1), replace=False)]))


def synth(engine, kind, n, seed):
    """n generated signatures of `kind` on the device, messages of the _bad positions corrupted.  Returns device tensors
    (msg, key, sig) and the expected verdicts (numpy)."""
    import torch
    msg = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
    key = torch.empty((n, KEYLEN[kind]), dtype=torch.uint8, device="cuda")
    sig = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    engine.synth_device(kind, seed, n, msg.data_ptr(), key.data_ptr(), sig.data_ptr())
    engine.sync()
    bad = _bad(n, seed)
    msg[torch.from_numpy(bad).cuda(), 9] ^= 0x20
    torch.cuda.synchronize()
    want = np.ones(n, np.uint8)
    want[bad] = 0
    return (msg, key, sig), want


def _sizes(engine):
    """small_max, one past it, the first size past it that is 1 mod 16 but not 1 mod 32, one wave and its neighbours"""
    sm, wave = engine.small_max(), _wave(engine)
    return sorted({sm, sm + 1, sm + 17, wave - 1, wave, wave + 1})


def test_verify_and_verify_device_at_route_boundaries(engine, defaults):
    """sv_verify_host and sv_verify_device (with a verdict bitmap) for all three kinds, without the square root and with
    it, at small_max, small_max + 1, small_max + 17 and one wave +- 1: route and verdicts.  Verdict bytes past n, bitmap
    bits past n in the last word and a sentinel word past the bitmap stay as they were."""
    import torch
    sizes = _sizes(engine)
    top = max(sizes)
    # one wave lies above small_max + 17, and the throughput sizes include ones that are 1 mod 32 (SV_PREP_BATCH) and
    # 1 mod 16 but not mod 32 (SV_FINAL_BATCH)
    above = [n for n in sizes if n > defaults]
    assert _wave(engine) > defaults + 18 and any(n % 32 == 1 for n in above) and any(n % 32 == 17 for n in above)
    for kind in (0, 1, 2):
        (msg, key, sig), want_all = synth(engine, kind, top, 7100 + kind)
        hm, hk, hs = (t.cpu().numpy() for t in (msg, key, sig))
        for nosqrt in (True, False):
            engine.set_nosqrt(nosqrt)
            for n in sizes:
                r = route(engine, kind, n, nosqrt)
                want = want_all[:n]
                got = counted(engine, lambda: engine.verify(kind, hm[:n], hk[:n], hs[:n]), r)
                assert np.array_equal(got, want), (kind, nosqrt, n, "verify")
                nw = (n + 31) // 32
                out = torch.full((n + 1,), 0xA5, dtype=torch.uint8, device="cuda")
                bm = torch.full((nw + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                counted(engine, lambda: engine.verify_device(kind, msg.data_ptr(), key.data_ptr(), sig.data_ptr(), n,
                                                             out.data_ptr(), bm.data_ptr()), r, "bitmap")
                engine.sync()
                o, b = out.cpu().numpy(), bm.cpu().numpy().view(np.uint32)
                assert np.array_equal(o[:n], want), (kind, nosqrt, n, "verify_device")
                assert o[n] == 0xA5, (kind, nosqrt, n, "verdict byte past n written")
                bits = np.unpackbits(b[:nw].view(np.uint8), bitorder="little")
                assert np.array_equal(bits[:n], want), (kind, nosqrt, n, "bitmap")
                assert not bits[n:].any(), (kind, nosqrt, n, "bitmap bits past n")
                assert b[nw] == 0x5A5A5A5A, (kind, nosqrt, n, "word past the bitmap written")


def _mixed_batch(engine, counts, seed):
    """an interleaved batch with counts[kind] items of each kind plus four unknown tags: (kinds, msg, key64, sig, want);
    the unused tail of every 64-byte key slot is filled with junk the engine must not read"""
    rng = np.random.default_rng(seed)
    parts = []
    for kind, c in enumerate(counts):
        if c:
            (m, k, s), w = synth(engine, kind, c, seed + kind)
            parts.append((kind, m.cpu().numpy(), k.cpu().numpy(), s.cpu().numpy(), w))
    n = sum(counts) + 4
    kinds = np.zeros(n, np.uint8)
    msg = np.zeros((n, 32), np.uint8)
    key = np.full((n, 64), 0xEE, np.uint8)
    sig = np.zeros((n, 64), np.uint8)
    want = np.zeros(n, np.uint8)
    order = rng.permutation(n)
    pos = 0
    for kind, m, k, s, w in parts:
        sel = order[pos:pos + m.shape[0]]
        pos += m.shape[0]
        kinds[sel], msg[sel], sig[sel], want[sel] = kind, m, s, w
        key[sel, :KEYLEN[kind]] = k
    unknown = order[pos:]
    kinds[unknown] = [3, 9, 200, 255]  # no such kind: verdict 0
    msg[unknown] = parts[0][1][:4]
    sig[unknown] = parts[0][3][:4]
    return kinds, msg, key, sig, want


def _mixed_routes(engine, counts, nosqrt):
    rs = ["mixed_split"]
    for kind, c in enumerate(counts):
        if c:
            rs += ["mixed_kind", route(engine, kind, c, nosqrt)]
    return rs


def test_mixed_batches_per_kind_counts_straddling_the_threshold(engine, defaults):
    """sv_verify_mixed_host and sv_verify_mixed_device (on a caller stream) with per-kind counts on both sides of
    small_max, so that one kind of a batch runs the small-batch kernel while another runs the throughput kernels; unknown
    tags get verdict 0 and the verdict byte past n stays untouched."""
    import torch
    sm = defaults
    lib = engine.lib
    for ci, counts in enumerate([(sm + 1, 1, sm), (0, sm + 1, sm), (sm, sm, sm + 1)]):
        kinds, msg, key, sig, want = _mixed_batch(engine, counts, 7200 + 10 * ci)
        n = kinds.shape[0]
        for nosqrt in (True, False):
            engine.set_nosqrt(nosqrt)
            rs = _mixed_routes(engine, counts, nosqrt)
            got = counted(engine, lambda: engine.verify_mixed(kinds, msg, key, sig), *rs)
            assert np.array_equal(got, want), (counts, nosqrt, "host")
            st = torch.cuda.Stream()
            dk, dm, dkey, ds = (torch.from_numpy(a).cuda() for a in (kinds, msg, key, sig))
            out = torch.full((n + 1,), 0xA5, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            rc = counted(engine, lambda: lib.sv_verify_mixed_device(engine._ctx, dk.data_ptr(), dm.data_ptr(), dkey.data_ptr(),
                                                                    ds.data_ptr(), n, out.data_ptr(), st.cuda_stream), *rs)
            assert rc == 0, engine.lib.sv_last_error(engine._ctx)
            st.synchronize()
            o = out.cpu().numpy()
            assert np.array_equal(o[:n], want) and o[n] == 0xA5, (counts, nosqrt, "device")
        assert 0 < want.sum() < n


def test_flush_per_kind_counts_straddling_the_threshold(engine, defaults):
    """the deferral queue splits by kind and verifies each kind through sv_verify_host: with per-kind counts on both sides
    of small_max one flush takes both routes; verdicts come back in enqueue order"""
    sm = defaults
    for ci, counts in enumerate([(sm + 1, 1, sm), (0, sm + 1, sm)]):
        kinds, msg, key, sig, want = _mixed_batch(engine, counts, 7300 + 10 * ci)
        known = kinds < 3
        kinds, msg, key, sig, want = kinds[known], msg[known], key[known], sig[known], want[known]
        assert engine.pending() == 0
        for i in range(kinds.shape[0]):
            engine.enqueue(int(kinds[i]), msg[i], key[i, :KEYLEN[int(kinds[i])]], sig[i])
        rs = [route(engine, kind, c, True) for kind, c in enumerate(counts) if c]
        got = counted(engine, engine.flush, *rs)
        assert np.array_equal(got, want), counts
        assert engine.pending() == 0


def test_overlapping_launches_on_caller_streams():
    """sv_verify_device calls queued back to back on three caller streams with no host synchronisation between them: all
    kinds, the square-root switch toggled between launches, growing sizes (a launch slot's record array grows while the
    other slot's launch is in flight), one small-batch call, one sv_verify_host call in the middle.  Every output equals
    its known verdicts and the same inputs verified one call at a time.  A context of its own, so that its launch slots
    start empty and grow exactly as planned below."""
    import torch

    import lightning_b200 as L
    engine = L.SigVerifier(0)
    try:
        sm = engine.small_max()
        streams = [torch.cuda.Stream() for _ in range(3)]
        # (kind, n, nosqrt, on the host API).  The throughput calls take the two launch slots in turn, each slot from
        # another stream than its last user; records are allocated for 4096 * 2^k items: 1 -> slot A (16384 records),
        # 2 -> B (32768), 4 -> A grows while 2 runs on B, host -> B, 6 -> A grows, 7 -> B grows while 6 runs on A,
        # 8 -> A, 9 -> B
        plan = [(0, sm + 1, True, False), (2, 2 * sm + 3, False, False), (1, 3000, True, False), (0, 4 * sm + 5, False, False),
                (1, 2 * sm + 1, True, True), (2, 8 * sm + 7, True, False), (1, 16 * sm + 9, False, False),
                (2, 9000, True, False), (0, 2 * sm + 33, True, False)]
        calls = []
        for i, (kind, n, nosqrt, host) in enumerate(plan):
            ins, want = synth(engine, kind, n, 7400 + i)
            out = torch.full((n + 1,), 0xA5, dtype=torch.uint8, device="cuda")
            calls.append((kind, n, nosqrt, host, ins, want, out))
        host_ins = {i: tuple(t.cpu().numpy() for t in c[4]) for i, c in enumerate(calls) if c[3]}
        torch.cuda.synchronize()
        got = {}
        for i, (kind, n, nosqrt, host, (m, k, s), want, out) in enumerate(calls):
            engine.set_nosqrt(nosqrt)
            r = route(engine, kind, n, nosqrt)
            if host:
                got[i] = counted(engine, lambda: engine.verify(kind, *host_ins[i]), r)
                continue
            st = streams[i % 3]
            counted(engine, lambda: engine.verify_device(kind, m.data_ptr(), k.data_ptr(), s.data_ptr(), n, out.data_ptr(),
                                                         stream=st.cuda_stream), r)
        torch.cuda.synchronize()
        for i, (kind, n, nosqrt, host, ins, want, out) in enumerate(calls):
            o = got[i] if host else out.cpu().numpy()
            assert np.array_equal(o[:n], want), (i, kind, n, nosqrt, int((o[:n] != want).sum()))
            assert host or o[n] == 0xA5, (i, "verdict byte past n written")
        # the same inputs one call at a time on the context's own stream
        for i, (kind, n, nosqrt, host, (m, k, s), want, out) in enumerate(calls):
            if host:
                continue
            engine.set_nosqrt(nosqrt)
            one = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            counted(engine, lambda: engine.verify_device(kind, m.data_ptr(), k.data_ptr(), s.data_ptr(), n, one.data_ptr()),
                    route(engine, kind, n, nosqrt))
            engine.sync()
            assert torch.equal(one, out[:n]), (i, kind, n, nosqrt)
    finally:
        engine.close()


def test_adversarial_scalars_through_the_shared_key_kernel(engine, ref, defaults):
    """The crafted signatures that steer the ladder and the comb into their exceptional branches (tests/adversarial.py),
    grouped by key (9 keys), through sv_verify_samekey_host: tiled past small_max so that the shared-key kernel runs, for
    both key forms; once more at group size with the small path off; and with the last message byte flipped, against the
    reference.  One key also at small_max and small_max + 1 (small-batch kernel, then shared-key kernel)."""
    sm = defaults
    msg, _, _, sig = adversarial.load()
    groups = adversarial.by_key()
    assert len(groups) == 9
    for gi, (pub33, pubxy, idx) in enumerate(groups):
        m, s = msg[idx], sig[idx]
        reps = (sm + 1 + len(idx) - 1) // len(idx)
        tile = lambda a: np.ascontiguousarray(np.tile(a, (reps, 1))[:sm + 1])
        m2 = m.copy()
        m2[:, 31] ^= 1
        want2 = util.ref_verify(ref, 0, m2, np.tile(pub33, (len(idx), 1)), s)
        for kind, key in ((0, pub33), (1, pubxy)):
            got = counted(engine, lambda: engine.verify_samekey(kind, key, tile(m), tile(s)), "samekey_shared")
            assert got.all(), (gi, kind, np.nonzero(got == 0)[0][:5] % len(idx))
            got = counted(engine, lambda: engine.verify_samekey(kind, key, tile(m2), tile(s)), "samekey_shared")
            assert np.array_equal(got, tile(want2[:, None])[:, 0]), (gi, kind, "flipped")
            engine.set_small_max(0)
            got = counted(engine, lambda: engine.verify_samekey(kind, key, m, s), "samekey_shared")
            engine.set_small_max(sm)
            assert got.all(), (gi, kind, "small path off")
    pub33, pubxy, idx = groups[0]
    for n, r in ((sm, "small"), (sm + 1, "samekey_shared")):
        reps = (n + len(idx) - 1) // len(idx)
        m, s = (np.ascontiguousarray(np.tile(a[idx], (reps, 1))[:n]) for a in (msg, sig))
        assert counted(engine, lambda: engine.verify_samekey(0, pub33, m, s), r).all(), n
        assert counted(engine, lambda: engine.verify_samekey(1, pubxy, m, s), r).all(), n


def test_bip340_batch_with_points_colliding_in_buckets(engine, ref, defaults):
    """BIP-340 batch verification on the device (counting sort, bucket sums, suffix scan and tree reduction per window)
    with groups whose points meet inside buckets (adversarial.bip340_collision_groups): every group's equation must hold,
    so groups_failed == 0.  A wrong bucket addition would only show there, since failed groups fall back to one-by-one
    verification.  Then one bad signature in each of 12 groups: the fallback re-verifies more than small_max members on
    the throughput kernels, verdicts against the reference."""
    sm = defaults
    groups = adversarial.bip340_collision_groups()
    msg = np.concatenate([g[1] for g in groups])
    key = np.concatenate([g[2] for g in groups])
    sig = np.concatenate([g[3] for g in groups])
    assert util.ref_verify(ref, 2, msg, key, sig, threads=4).all()
    for seed in (bytes(range(32)), bytes(32)):
        v, gt, gf = counted(engine, lambda: engine.verify_schnorr_batch(msg, key, sig, seed32=seed), "sb_batch")
        assert v.all() and gt == len(groups) and gf == 0, (gt, gf)
    for name, m, k, s in groups:
        v, gt, gf = counted(engine, lambda: engine.verify_schnorr_batch(m, k, s, seed32=bytes(range(32))), "sb_batch")
        assert v.all() and gt == 1 and gf == 0, name
    # the same signatures verified one by one: small-batch kernel, then the throughput kernels
    for nosqrt in (True, False):
        engine.set_nosqrt(nosqrt)
        assert counted(engine, lambda: engine.verify(2, msg, key, sig), "small").all()
        engine.set_small_max(0)
        assert counted(engine, lambda: engine.verify(2, msg, key, sig), main_route(2, nosqrt)).all()
        engine.set_small_max(sm)
    engine.set_nosqrt(True)
    # one bad signature in each of 12 groups: 12 x 1024 members go back to one-by-one verification
    m12, k12, s12 = (np.concatenate([a] * 3) for a in (msg, key, sig))
    for g in range(12):
        pos = g * 1024 + (97 * g + 5) % 1024
        if g % 3 == 0:
            m12[pos, g % 32] ^= 1 << (g % 8)
        elif g % 3 == 1:
            s12[pos, 40 + g % 24] ^= 1 << (g % 8)
        else:
            k12[pos] = groups[2][2][(31 * g + 7) % 1024]  # another signer's key (r_eq_p has one key per member)
    want = util.ref_verify(ref, 2, m12, k12, s12, threads=4)
    assert want.sum() == 12 * 1024 - 12 and 12 * 1024 > sm  # every member of the 12 groups is re-verified
    v, gt, gf = counted(engine, lambda: engine.verify_schnorr_batch(m12, k12, s12, seed32=bytes(range(32))),
                        "sb_batch", "sb_fallback", main_route(2, True))
    assert np.array_equal(v, want) and gt == 12 and gf == 12, (gt, gf, np.nonzero(v != want)[0][:5])
