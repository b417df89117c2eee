"""GPU: the fixed-base comb table d * 2^(16 i) * G, entry by entry, and the digit boundaries of every row through its readers.

Every ECDSA and BIP-340 verification adds u1*G (BIP-340: s*G) from one piece of device state: the 34 MiB table that
k_gtable_bases / k_gtable_fill build once per context, 557,056 affine points in the allocation it shares with the two
launch slots' per-thread table slabs, laid out [slab 0 | G table | slab 1].  A wrong entry rejects only the valid
signatures whose u1 has that digit in that row, so random signatures, which draw entries uniformly, would almost never
notice it; neither would they notice a kernel that writes past its slab into the table.  Here:

  (a) every entry, bit-exact against the plain model (tests/gtable_model.py): the single-entry scalar of each entry through
      SV_ST_ECMULT_GEN is one mixed addition from infinity onto the entry and the conversion to affine, so the output is
      the entry itself (the last entry of row 15, reachable only through the carry out of window 14, comes with -B_14);
  (b) the table is unchanged after every route that shares its allocation or reads it, run at sizes that fill the
      persistent grid (the last thread's slab ends where the table begins), in the session's context and in one whose
      smaller grid (SV_MAIN_GRID_RESERVE=2) puts the table at another offset;
  (c) every row's recoding boundaries (window values 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF, with and without a carry in,
      and the carry into row 15's 0x10000) through the digit recoding, ecmult_comb_add, small_comb and ecmult_gen_comb
      against Python, and end to end through the small-batch kernel, the throughput kernels with and without the square
      root, the shared-key kernel, sv_verify_device and mixed batches, against the reference.

The fee grind and the BIP-340 comb (batch verification's window sums) are not steered in (c): the grind's u1 comes from a
sighash and BIP-340's s is fixed by the nonce hash.  Both read the table through the same ecmult_comb_add that (c) tests,
and (b) runs both before checking the table itself.

With $SV_SELFTEST_COVERAGE_DIR set, gtable_coverage.json receives, per row, the entries (a) checked and the boundary digits
(c) reached in each reader."""
import json
import os
import random

import numpy as np
import pytest

from tests import adversarial, bolt12, ecc, feegrind, gossip, txsig, util
from tests import group_cases as C
from tests import group_schedule as S
from tests import gtable_model as M
from tests import selftest_cases as SC
from tests import test_gpu_routes as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
QTAB_ENTRY_BYTES, GE_MEM_BYTES = 96, 64  # sizeof(qtab_entry): x, y, beta*x; sizeof(ge_mem): x, y
WINDOWS = (0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF)
COVERAGE = {"table_checks": {}, "rows": {str(r): {"entries": M.row_size(r), "checked": {}, "boundary_digits": {}}
                                          for r in range(M.ROWS)}}


@pytest.fixture(scope="module", autouse=True)
def _coverage():
    yield
    out = os.environ.get("SV_SELFTEST_COVERAGE_DIR")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "gtable_coverage.json"), "w") as f:
            json.dump(COVERAGE, f, indent=1)


def _reached(reader, digit_lists):
    for gd in digit_lists:
        for row, d in enumerate(gd):
            if d:
                got = COVERAGE["rows"][str(row)]["boundary_digits"].setdefault(reader, [])
                if d not in got:
                    got.append(d)
                    got.sort()


@pytest.fixture(scope="module")
def table():
    """(single-entry scalars as limbs, what SV_ST_ECMULT_GEN must return for them)"""
    model = M.build()
    scalars = M.scalar_limbs([M.scalar_for(e) for e in range(M.ENTRIES)])
    want = model.copy()
    x, y = ecc.base_mult(M.CARRY_SCALAR)
    want[-1] = M.scalar_limbs([x, y]).reshape(16)
    return scalars, want


def check_table(engine, table, label):
    """the whole device table of `engine` against the model, and the layout sizes of engine.info()"""
    scalars, want = table
    info = engine.info()
    assert info["gtable_bytes"] == M.ENTRIES * GE_MEM_BYTES, info
    assert info["scratch_bytes"] == info["main_grid"] * info["main_block"] * 8 * QTAB_ENTRY_BYTES, info
    got = engine.selftest(SC.OPS["ECMULT_GEN"], scalars)
    bad = np.nonzero((got != want).any(axis=1))[0]
    first = [(int(e), *M.row_d(int(e))) for e in bad[:8]]
    assert bad.size == 0, f"{label}: {bad.size} table entries differ; first (entry, row, d): {first}"
    COVERAGE["table_checks"][label] = M.ENTRIES
    for r in range(M.ROWS):
        COVERAGE["rows"][str(r)]["checked"][label] = M.row_size(r)


def test_whole_table_entry_by_entry(engine, table):
    """(a): all 557,056 entries through SV_ST_ECMULT_GEN, bit-exact, and the table and slab sizes of the layout"""
    check_table(engine, table, "fresh")


# ---- (b) every route that shares the table's allocation or reads it -------------------------------------------------
def _throughput_on_two_streams(engine):
    """k_main of all five kinds at one wave + 1 and two waves, sv_verify_device launches alternating between two caller
    streams with no host synchronisation between them, so that both launch slots are in flight at once"""
    import torch
    wave = R._wave(engine)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    calls = []
    for ki, (kind, nosqrt) in enumerate(((0, True), (0, False), (1, True), (2, True), (2, False))):
        ins, want = R.synth(engine, kind, 2 * wave, 7800 + ki)
        for n in (wave + 1, 2 * wave):
            calls.append((kind, nosqrt, n, ins, want[:n], torch.full((n + 1,), 0xA5, dtype=torch.uint8, device="cuda")))
    torch.cuda.synchronize()
    for i, (kind, nosqrt, n, (m, k, s), _, out) in enumerate(calls):
        engine.set_nosqrt(nosqrt)
        R.counted(engine, lambda: engine.verify_device(kind, m.data_ptr(), k.data_ptr(), s.data_ptr(), n, out.data_ptr(),
                                                       stream=streams[i % 2].cuda_stream),
                  R.route(engine, kind, n, nosqrt))
    torch.cuda.synchronize()
    engine.set_nosqrt(True)
    for kind, nosqrt, n, _, want, out in calls:
        o = out.cpu().numpy()
        assert np.array_equal(o[:n], want) and o[n] == 0xA5, (kind, nosqrt, n, int((o[:n] != want).sum()))


def _schnorr_batch_with_one_fallback(engine):
    """two groups of valid BIP-340 signatures, one bad signature in the second: that group falls back"""
    n, seed = 2 * adversarial.BATCH_GROUP, 7810
    (m, k, s), _ = R.synth(engine, 2, n, seed)
    m, k, s = (t.cpu().numpy() for t in (m, k, s))
    m[R._bad(n, seed), 9] ^= 0x20  # undo synth's corruption: every signature valid
    bad = adversarial.BATCH_GROUP + 321
    m[bad, 3] ^= 1
    want = np.ones(n, np.uint8)
    want[bad] = 0
    v, gt, gf = engine.verify_schnorr_batch(m, k, s, seed32=bytes(range(32)))
    assert np.array_equal(v, want) and gt == 2 and gf == 1, (gt, gf, np.nonzero(v != want)[0][:5])


def _fee_grind(engine):
    """one grind over [253, 125000] of an HTLC transaction signed at feerate 2070"""
    from lightning_b200 import SvTx
    vec = json.load(open(os.path.join(ROOT, "tests", "golden", "bolt3_htlc_txs.json")))[0]
    weight = feegrind.HTLC_SUCCESS_WEIGHT if "success" in vec["name"] else feegrind.HTLC_TIMEOUT_WEIGHT
    amount, fee = 5_000_000, feegrind.fee(2070, weight)
    t, blob = feegrind.htlc_tx(vec, 1, amount)
    t.output_amount = amount - fee
    key, sigs = txsig.sign(engine, 0, (0x5EED + 7).to_bytes(32, "big"), (SvTx * 1)(t), blob)
    want = feegrind.grind(253, 125000, weight, amount, lambda f, x: x == fee)
    assert want[0] is not None and engine.grind_tx_fee(0, t, blob, key, bytes(sigs[0]), weight, 253, 125000) == want


def _bolt12_pass(engine):
    fx = bolt12.load_fixture()
    idx = np.nonzero(fx["names"] == 0)[0]
    status = engine.verify_bolt12_spans(*bolt12.NAMES[0], fx["blob"], fx["off"][idx], fx["len"][idx], fx["xonly"][idx],
                                        fx["sig"][idx])
    np.testing.assert_array_equal(status, fx["status"][idx].astype(np.int32))


def run_every_route(engine):
    """every route that reads the table or shares its allocation, once, verdicts checked"""
    sm = engine.small_max()
    wave = R._wave(engine)
    assert wave > sm
    try:
        _throughput_on_two_streams(engine)
        # the small-batch kernel, all three kinds
        for kind in (0, 1, 2):
            ins, want = R.synth(engine, kind, sm, 7820 + kind)
            m, k, s = (t.cpu().numpy() for t in ins)
            assert np.array_equal(R.counted(engine, lambda: engine.verify(kind, m, k, s), "small"), want), kind
        # the shared-key kernel over a whole grid: its key table sits at the head of a launch slot's slab
        msg, _, _, sig = adversarial.load()
        pub33, pubxy, idx = adversarial.by_key()[0]
        reps = (wave + 1 + len(idx) - 1) // len(idx)
        tm, ts = (np.ascontiguousarray(np.tile(a[idx], (reps, 1))[:wave + 1]) for a in (msg, sig))
        for kind, key in ((0, pub33), (1, pubxy)):
            assert R.counted(engine, lambda: engine.verify_samekey(kind, key, tm, ts), "samekey_shared").all(), kind
        # a gossip burst whose node keys repeat (every message six times): key de-duplication, k_main_shared
        engine.set_dedup(True)
        st = engine.verify_gossip_burst(gossip.load_subset() * 6, TESTNET)
        assert not st.any() and engine.last_distinct_keys() > 0
        # a mixed batch with one kind above small_max and the others below
        counts = (sm + 1, 1, sm)
        kinds, msg, key, sig, want = R._mixed_batch(engine, counts, 7830)
        got = R.counted(engine, lambda: engine.verify_mixed(kinds, msg, key, sig), *R._mixed_routes(engine, counts, True))
        assert np.array_equal(got, want)
        _schnorr_batch_with_one_fallback(engine)
        _fee_grind(engine)
        _bolt12_pass(engine)
    finally:
        engine.set_small_max(sm)
        engine.set_nosqrt(True)
        engine.set_dedup(True)


def test_table_unchanged_after_every_route(engine, table):
    """(b): the whole table, bit-exact, after every route has run in the session's context; then the same in a context
    whose grid is two blocks smaller (SV_MAIN_GRID_RESERVE=2, read at sv_create), so that slab 0 is smaller and the
    table starts at another offset"""
    import lightning_b200 as L
    check_table(engine, table, "fresh")
    run_every_route(engine)
    check_table(engine, table, "after_every_route")
    old = os.environ.get("SV_MAIN_GRID_RESERVE")
    os.environ["SV_MAIN_GRID_RESERVE"] = "2"
    try:
        other = L.SigVerifier(0)
    finally:
        if old is None:
            del os.environ["SV_MAIN_GRID_RESERVE"]
        else:
            os.environ["SV_MAIN_GRID_RESERVE"] = old
    try:
        if old is None:
            assert other.info()["main_grid"] == engine.info()["main_grid"] - 2
        check_table(other, table, "reserve_2_fresh")
        run_every_route(other)
        check_table(other, table, "reserve_2_after_every_route")
    finally:
        other.close()


# ---- (c) the recoding boundaries of every row through every reader --------------------------------------------------
def _recoded(j, w, carry_in):
    """the comb digits of window j = w (and window j - 1 = 0x8001 when carry_in), derived by hand: a window above 0x8000
    (below row 15) becomes w - 0x10000 and carries 1 into the next row"""
    gd = [0] * M.ROWS
    if carry_in:
        gd[j - 1] = 0x8001 - 0x10000
    v = w + carry_in
    if j < 15 and v > 0x8000:
        gd[j] = v - 0x10000
        gd[j + 1] = 1
    else:
        gd[j] = v
    return gd


def boundary_scalars():
    """[(u1, its comb digits)]: for every row j, window j in WINDOWS with window j - 1 = 0 or 0x8001 (no carry in, or one),
    and 2^256 - 2^224, whose carry out of window 14 makes row 15's digit 0x10000 without a carry in"""
    out = []
    for j in range(M.ROWS):
        for w in WINDOWS:
            for cin in ((0,) if j == 0 else (0, 1)):
                out.append(((w << (16 * j)) + ((0x8001 << (16 * (j - 1))) if cin else 0), _recoded(j, w, cin)))
    gd = [0] * M.ROWS
    gd[14], gd[15] = -1, 0x10000
    out.append((M.CARRY_SCALAR, gd))
    for u1, gd in out:
        assert 0 < u1 < M.N and S.prepare_u1(u1) == gd, hex(u1)
        assert sum(d << (16 * i) for i, d in enumerate(gd)) == u1
    assert {gd[15] for _, gd in out} >= {0x8000, 0x8001, 0xFFFF, 0x10000}
    return out


def test_boundary_digits_through_the_comb_readers(engine):
    """(c): SV_ST_PREPARE_U1 returns the expected digits; SV_ST_ECMULT_GEN (ecmult_gen_comb), SV_STG_ECMULT_COMB_ADD onto
    infinity and onto a random point, and SV_STG_SMALL_COMB (from infinity) equal u1*G computed in Python"""
    cases = boundary_scalars()
    us = [u for u, _ in cases]
    digits = [gd for _, gd in cases]
    got = engine.selftest(SC.OPS["PREPARE_U1"], M.scalar_limbs(us)).view(np.int32)
    for (u1, gd), row in zip(cases, got):
        assert [int(v) for v in row] == gd, hex(u1)
    _reached("prepare_u1", digits)
    out = engine.selftest(SC.OPS["ECMULT_GEN"], M.scalar_limbs(us))
    for u1, o in zip(us, out):
        assert (C.get(o, 0), C.get(o, 8)) == ecc.base_mult(u1), ("ecmult_gen_comb", hex(u1))
    _reached("ecmult_gen_comb", digits)
    rnd = random.Random(7840)
    starts = [None] * len(us) + [rnd.randrange(1, M.N) for _ in us]
    recs = C.new_records(len(starts))
    for i, (start, u1) in enumerate(zip(starts, us + us)):
        C.put_jac(recs[i], 0, None if start is None else ecc.base_mult(start), C.random_z(rnd), rnd)
        C.put(recs[i], 48, u1)
    out_a = engine.selftest_group(C.OPS["ECMULT_COMB_ADD"], recs)
    out_s = engine.selftest_group(C.OPS["SMALL_COMB"], recs[:len(us)])
    for i, (start, u1) in enumerate(zip(starts, us + us)):
        assert C.get_jac(out_a[i]) == ecc.base_mult((u1 + (start or 0)) % M.N), ("ecmult_comb_add", start, hex(u1))
    for u1, o in zip(us, out_s):
        assert C.get_jac(o) == ecc.base_mult(u1), ("small_comb", hex(u1))
    _reached("ecmult_comb_add", digits)
    _reached("small_comb", digits)


KEYS = (0x1D2C3B4A59687786950A1B2C3D4E5F60718293A4B5C6D7E8F90123456789ABC, 7)


def crafted_boundary_signatures():
    """per key d of KEYS, one ECDSA signature per boundary u1 that the verifier must see with exactly that u1 (the first u2
    of a seeded list for which s comes out low): {d: (msg, pub33, pubxy, sig)}"""
    rnd = random.Random(7850)
    out = {}
    for d in KEYS:
        rows = []
        for u1, _ in boundary_scalars():
            for _ in range(64):
                c = adversarial.craft(d, u1, rnd.randrange(1, M.N), exact=True)
                if c is not None:
                    rows.append(c)
                    break
            else:
                raise AssertionError(("no low-s signature", d, hex(u1)))
        out[d] = tuple(np.stack(col) for col in zip(*rows))
    return out


def test_boundary_digits_end_to_end(engine, ref):
    """(c), end to end: signatures whose u1 is every boundary scalar, for two keys, in both ECDSA key forms, through the
    small-batch kernel, the throughput kernels with and without the square root, the shared-key kernel, sv_verify_device
    and mixed batches.  All are valid by construction; every verdict equals the reference's."""
    import torch
    sm = engine.small_max()
    sigs = crafted_boundary_signatures()
    digits = [gd for _, gd in boundary_scalars()]
    msg = np.concatenate([sigs[d][0] for d in KEYS])
    sig = np.concatenate([sigs[d][3] for d in KEYS])
    keys = {0: np.concatenate([sigs[d][1] for d in KEYS]), 1: np.concatenate([sigs[d][2] for d in KEYS])}
    n = msg.shape[0]
    want = {kind: util.ref_verify(ref, kind, msg, keys[kind], sig) for kind in (0, 1)}
    assert want[0].all() and want[1].all()
    try:
        for kind in (0, 1):
            assert n <= sm
            got = R.counted(engine, lambda: engine.verify(kind, msg, keys[kind], sig), "small")
            assert np.array_equal(got, want[kind]), (kind, "small", np.nonzero(got != want[kind])[0][:5])
            engine.set_small_max(0)
            for nosqrt in (True, False):
                engine.set_nosqrt(nosqrt)
                got = R.counted(engine, lambda: engine.verify(kind, msg, keys[kind], sig), R.main_route(kind, nosqrt))
                assert np.array_equal(got, want[kind]), (kind, nosqrt, np.nonzero(got != want[kind])[0][:5])
                dm, dk, ds = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (msg, keys[kind], sig))
                out = torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                R.counted(engine, lambda: engine.verify_device(kind, dm.data_ptr(), dk.data_ptr(), ds.data_ptr(), n,
                                                               out.data_ptr()), R.main_route(kind, nosqrt))
                engine.sync()
                assert np.array_equal(out.cpu().numpy(), want[kind]), (kind, nosqrt, "verify_device")
            engine.set_nosqrt(True)
            off = 0
            for d in KEYS:
                m, s = sigs[d][0], sigs[d][3]
                key = sigs[d][1][0] if kind == 0 else sigs[d][2][0]
                w = want[kind][off:off + m.shape[0]]
                off += m.shape[0]
                got = R.counted(engine, lambda: engine.verify_samekey(kind, key, m, s), "samekey_shared")
                assert np.array_equal(got, w), (kind, "samekey", d)
            engine.set_small_max(sm)
        # mixed: both key forms interleaved, each kind once below small_max and once on the throughput kernels
        kinds = np.repeat(np.array([0, 1], np.uint8), n)
        order = np.random.default_rng(7860).permutation(2 * n)
        key64 = np.zeros((2 * n, 64), np.uint8)
        key64[:n, :33] = keys[0]
        key64[n:] = keys[1]
        mk, mm, mkey, ms = kinds[order], np.tile(msg, (2, 1))[order], key64[order], np.tile(sig, (2, 1))[order]
        mwant = np.concatenate([want[0], want[1]])[order]
        for small_max in (sm, 0):
            engine.set_small_max(small_max)
            counts = (n, n, 0)
            got = R.counted(engine, lambda: engine.verify_mixed(mk, mm, mkey, ms), *R._mixed_routes(engine, counts, True))
            assert np.array_equal(got, mwant), ("mixed", small_max)
    finally:
        engine.set_small_max(sm)
        engine.set_nosqrt(True)
    for reader in ("small", "main_nosqrt", "main", "verify_device", "samekey_shared", "mixed"):
        _reached("end_to_end." + reader, digits)
