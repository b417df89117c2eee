"""GPU: the funding check of a gossip_store with tables shaped as lightningd exports them (tests/funding_tables.py).

FundingTable.from_lightningd_db keeps utxoset's rows in SQLite's order, and a node's utxoset holds every unspent P2WSH
output of every block it processed.  The engine stages the table as given, sorts the scids with CUB SortPairs carrying
each output's entry index, sorts the heights with SortKeys, refuses neighbouring equal scids (k_funding_dups), and
gf_verdict binary-searches both sorted arrays and reads the amount and script of the entry the sort carried.  So:

  - order: every fixture case with its table reversed, shuffled, in low-bits-first order and shuffled with every height
    twice gives exactly the results of the sorted table; the clean case and one refused case per order also pass the
    whole check of tests/test_gpu_gossip_store_funding.py (model, gossmap's strict load, a second prune deletes nothing)
  - sizes: tables padded with decoys across the radix sort's single-tile and onesweep limits up to 2^22 outputs give
    the model's verdicts and summaries; decoys change nothing
  - duplicates planted anywhere in shuffled tables of up to 2^22 outputs are refused; scids one bit apart are not
  - announcements with features fields of 0 to 1,000 bytes, each with every verdict, whose long features hold another
    funded output's scid and keys where a read that ignored the features length would look
  - a lightningd.sqlite3 with rows in shuffled order, through the exporter, the Python binding and the command line
  - one context reused for a table of 2^22 outputs, then 3, then 2^22 again

The model's signature statuses: the fixture's and the crafted store's messages all verify (asserted against the
engine's own audit), so the model runs without a sigcheck except where CLN's is replayed (check())."""
import os
import subprocess
import sys

import numpy as np
import pytest

from lightning_b200.funding import FundingTable
from tests import funding_tables as ftab
from tests import gossip_store as gs
from tests import gossip_store_funding as gf
from tests import gossip_store_prune as gp
from tests.test_gossip_store_funding_host import make_db
from tests.test_gossip_store_host import load_fixture
from tests.test_gpu_gossip_burst import TESTNET
from tests.test_gpu_gossip_store import TOOL
from tests.test_gpu_gossip_store_funding import check, funding_table
from tests.test_gpu_gossip_store_prune import corrupted_x53

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = sorted(gf.fixture_cases(load_fixture()))
# per order, the refused case that also runs the whole check with CLN's sigcheck and gossmap's strict load
REFUSED_CASE = {"reversed": "no_txout", "shuffled": "script_other_key", "low_bits_first": "amount_off_by_one",
                "shuffled_heights_twice": "refused_holder_then_funded_copy"}


def table(a):
    return FundingTable.from_arrays(*a)


def calls(engine, store, ft):
    """(audit with the table, prune with the table) as the binding returns them"""
    return engine.verify_gossip_store(store, TESTNET, funding=ft), engine.prune_gossip_store(store, TESTNET, funding=ft)


def equal(x, y):
    if isinstance(x, (tuple, list)):
        return len(x) == len(y) and all(equal(a, b) for a, b in zip(x, y))
    if isinstance(x, np.ndarray):
        return np.array_equal(x, y)
    return x == y


def device_verdicts(store, audit, t):
    """the model's verdict for every record the engine's audit gave status 0 as an announcement (GF_NONE elsewhere)"""
    off, typ, st = audit[:3]
    return [gf.verdict(store, int(o), t) if y == 256 and s == 0 else gf.GF_NONE for o, y, s in zip(off, typ, st)]


_MODEL = {}


def model_results(store, t):
    """(audit funding verdicts, funding summary, pruned bytes, prune rows, prune summary, prune verdicts, prune funding
    summary) of the model without a sigcheck, memoized by the table's announced part"""
    key = (hash(store), tuple(sorted(t.outputs.items())), frozenset(t.blocks))
    if key not in _MODEL:
        _, _, fund, fs = gf.audit(store, t)
        out, rows, s, pfund, pfs = gp.prune(store, table=t)
        _MODEL[key] = (fund, fs, out, rows, s, pfund, pfs)
    return _MODEL[key]


def all_good(engine, store, n_msgs):
    """every message of the store verifies (so the model's statuses, all 0 without a sigcheck, are gossipd's)"""
    s = engine.verify_gossip_store(store, TESTNET)[4]
    assert s["good"] == n_msgs and s["stop"] == gs.EOF, s


def agree_with_model(engine, store, a, ann, ft=None):
    """audit and prune with the table a against the model (no sigcheck: every message of these stores verifies)"""
    t = ftab.model(a, ann)
    fund, fs, out, rows, s, pfund, pfs = model_results(store, t)
    au, pr = calls(engine, store, table(a) if ft is None else ft)
    assert [int(x) for x in au[5]] == fund
    assert au[6] == fs
    assert pr[0] == out
    assert [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(*pr[1])] == rows
    assert [int(x) for x in pr[3]] == pfund
    assert pr[4] == pfs
    for k, v in s.items():
        assert pr[2][k] == v, k
    return fs, pfs


# ---- order ------------------------------------------------------------------------------------------------------------
_SORTED = {}


def sorted_results(engine, case):
    if case not in _SORTED:
        store, t = gf.fixture_cases(load_fixture())[case]
        _SORTED[case] = calls(engine, store, funding_table(t))
    return _SORTED[case]


@pytest.mark.parametrize("order", ftab.ORDERS)
@pytest.mark.parametrize("case", CASES)
def test_order_does_not_matter(engine, case, order):
    """the records, verdicts, summaries and pruned bytes of the reordered table are those of the sorted one, and its
    verdicts are the model's"""
    store, t = gf.fixture_cases(load_fixture())[case]
    a = ftab.arrays(t)
    r = ftab.reorder(a, order, seed=CASES.index(case))
    assert not np.array_equal(r[0], a[0])
    got = calls(engine, store, table(r))
    assert equal(got, sorted_results(engine, case))
    assert [int(x) for x in got[0][5]] == device_verdicts(store, got[0], gf.Table.of(funding_table(t)))


@pytest.mark.parametrize("order", ftab.ORDERS)
def test_order_whole_check(engine, order):
    """the clean case and one refused case in each order: the model with CLN's sigcheck, the pruned store under gossmap's
    strict load, a second prune"""
    for case in ("clean", REFUSED_CASE[order]):
        store, t = gf.fixture_cases(load_fixture())[case]
        r = ftab.reorder(ftab.arrays(t), order, seed=1)
        ps, pfs = check(engine, store, ftab.lists(r))
        assert pfs["deleted"] == (0 if case == "clean" else 1), case


def test_tiled_x53_corrupted_table_shuffled(engine):
    """the x53 store with 1 % of the table wrong, shuffled with 100,000 decoys: the sorted table's results"""
    fx = load_fixture()
    t = gf.corrupt_table(gf.table_of_store(fx), 0.01, 53)
    store = corrupted_x53()
    a = ftab.arrays(t)
    r = ftab.reorder(ftab.pad(a, ftab.announced(store), a[0].size + 100000, a[3].size + 1000, seed=53), "shuffled", 53)
    got = calls(engine, store, table(r))
    want = calls(engine, store, funding_table(t))
    assert equal(got, want)
    assert [int(x) for x in got[0][5]] == device_verdicts(store, got[0], gf.Table.of(funding_table(t)))
    assert got[1][4]["deleted"] > 0


# ---- sizes ------------------------------------------------------------------------------------------------------------
def fixture_table(kind):
    fx = load_fixture()
    t = gf.table_of_store(fx)
    return ftab.arrays(t if kind == "clean" else gf.corrupt_table(t, 0.02, 53))


SIZE_CASES = [("no_outputs", 0, None), ("no_heights", None, 0), ("1", 1, None), ("2", 2, None), ("3", 3, None)] + \
    [(str(n), n, n) for n in ftab.SIZES]


@pytest.mark.parametrize("kind", ["clean", "corrupted"])
@pytest.mark.parametrize("name,n,m", SIZE_CASES, ids=[c[0] for c in SIZE_CASES])
def test_sizes(engine, kind, name, n, m):
    """the fixture's table cut down or padded with decoys to n outputs and m heights, shuffled: the model's verdicts
    and summaries, which for a padded table are those of the table without decoys"""
    fx = load_fixture()
    all_good(engine, fx, 3100)
    a = fixture_table(kind)
    ann = ftab.announced(fx)
    p = ftab.pad(a, ann, a[0].size if n is None else n, a[3].size if m is None else m, seed=len(name))
    assert p[0].size == (a[0].size if n is None else n)
    if n is None or n >= a[0].size:
        assert ftab.same_model(a, p, ann) or m == 0
    fs, pfs = agree_with_model(engine, fx, p, ann)
    if kind == "clean" and (n is None or n >= a[0].size) and m != 0:
        assert fs["funded"] == 1500 and pfs["deleted"] == 0
    if n == 0 and kind == "clean":
        assert fs["no_txout"] == 1500
    if m == 0 and kind == "clean":
        assert fs["funded"] == 1500


# ---- duplicates -------------------------------------------------------------------------------------------------------
def plants(n, rng):
    """(positions, same amount?) of planted duplicates: first and last, two random positions, three times"""
    out = [((0, n - 1), True), ((0, n - 1), False)]
    if n > 3:
        i, j = sorted(rng.choice(np.arange(1, n - 1), 2, replace=False).tolist())
        out += [((i, j), True), ((j, i), False)]
    if n >= 3:
        out += [((0, n // 2, n - 1), True), ((n - 1, int(rng.integers(1, n - 1)), 0), False)]
    return out


@pytest.mark.parametrize("n", [2, 3, (1 << 20) + 1, ftab.BIG])
def test_duplicate_scid_refused(engine, n):
    """a scid planted twice or three times (after FundingTable checked), at any positions of a shuffled table, with
    the same amount or another: both entry points refuse the table"""
    fx = load_fixture()
    a = fixture_table("clean")
    p = ftab.pad(a, ftab.announced(fx), n, a[3].size, seed=n)
    ft = table(p)
    rng = np.random.default_rng(n)
    for pos, same in plants(n, rng):
        sc, sa = ft.scid.copy(), ft.satoshis.copy()
        for k in pos[1:]:
            ft.scid[k] = ft.scid[pos[0]]
            ft.satoshis[k] = ft.satoshis[pos[0]] if same else ft.satoshis[pos[0]] ^ np.uint64(1 + k)
        for f in (engine.verify_gossip_store, engine.prune_gossip_store):
            with pytest.raises(Exception, match="twice"):
                f(fx, TESTNET, funding=ft)
        ft.scid[:], ft.satoshis[:] = sc, sa
    # the table itself is fine again
    agree_with_model(engine, fx, p, ftab.announced(fx), ft)


def test_scids_one_bit_apart_not_refused(engine):
    """the fixture's outputs and, for 200 of them, the scid with bit 0 and the scid with bit 63 flipped (each with
    the script and amount of another entry), shuffled: no refusal, the model's verdicts"""
    fx = load_fixture()
    all_good(engine, fx, 3100)
    a = fixture_table("clean")
    ann = ftab.announced(fx)
    rng = np.random.default_rng(63)
    pick = rng.choice(a[0].size, 200, replace=False)
    near = np.concatenate([a[0][pick] ^ np.uint64(1), a[0][pick] ^ np.uint64(1 << 63)])
    near = near[~np.isin(near, ann)]
    src = rng.integers(0, a[0].size, near.size)
    p = (np.concatenate([a[0], near]), np.concatenate([a[1], a[1][src]]), np.concatenate([a[2], a[2][src]]), a[3])
    p = ftab.reorder(p, "shuffled", 63)
    fs, _ = agree_with_model(engine, fx, p, ann)
    assert fs["funded"] == 1500


# ---- features ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ("sorted",) + ftab.ORDERS)
def test_features_fields(engine, order):
    """announcements with features fields of 0 to 1,000 bytes, each with every verdict, with and without decoys: the
    model, the prune, gossmap's strict load of the result (check())"""
    store, a, what = ftab.features_store()
    n = len(ftab.FLENS) * len(ftab.KINDS)
    all_good(engine, store, n)
    if order != "sorted":
        a = ftab.reorder(ftab.pad(a, ftab.announced(store), 5000, 5000, seed=7), order, seed=7)
    ps, pfs = check(engine, store, ftab.lists(a))
    per = len(ftab.FLENS)
    assert (pfs["funded"], pfs["script"], pfs["amount"], pfs["no_txout"], pfs["unchecked"]) == (per,) * 5
    assert pfs["deleted"] == 3 * per
    fund = engine.verify_gossip_store(store, TESTNET, funding=table(a))[5]
    kinds = {"funded": gf.GF_FUNDED, "script": gf.GF_SCRIPT, "amount": gf.GF_AMOUNT, "no_txout": gf.GF_NO_TXOUT,
             "unchecked": gf.GF_UNCHECKED}
    recs = gs.walk(store)[0]
    for (off, typ, _, _), v in zip(recs, fund):
        if typ == 256:
            assert int(v) == kinds[what[gf.ann_keys(store, off + gs.HDR)[0]][1]], what[gf.ann_keys(store, off + gs.HDR)[0]]


# ---- lightningd.sqlite3 -----------------------------------------------------------------------------------------------
def test_export_end_to_end(engine, tmp_path):
    """a lightningd.sqlite3 holding the fixture's outputs (30 of them spent), 20,000 decoys (some spent), spent rows of
    other scripts, and the heights less five of the spent outputs' blocks, every row inserted in shuffled order:
    FundingTable.from_lightningd_db, then the audit and the prune against the model; then the exporter's command line
    and cln_verify_gossip_store --funding"""
    fx = load_fixture()
    all_good(engine, fx, 3100)
    ann = ftab.announced(fx)
    a = fixture_table("clean")
    rng = np.random.default_rng(2026)
    d = ftab.decoys(a, ann, 20000, seed=2026)
    sc = np.concatenate([a[0], d[0]])
    sa = np.concatenate([a[1], d[1] & np.uint64((1 << 63) - 1)])  # sqlite's INTEGER is signed
    sp = np.concatenate([a[2], d[2]])
    spent = set(rng.choice(a[0].size, 30, replace=False).tolist()) | set((a[0].size + rng.choice(
        d[0].size, 500, replace=False)).tolist())
    rows = []
    for k in range(sc.size):
        s = int(sc[k])
        rows.append((s >> 40, (s >> 16) & 0xFFFFFF, s & 0xFFFF, sp[k].tobytes(), int(sa[k]), 800000 if k in spent else None))
    rows += [(1 + k, k, 0, b"\x00\x14" + bytes(20), 1, 800001) for k in range(50)]  # spent, not P2WSH: never read
    spent_ann = sorted(int(a[0][k]) for k in spent if k < a[0].size)
    gone = {s >> 40 for s in spent_ann[:5]}
    heights = [int(h) for h in a[3] if int(h) not in gone] + [int(h) for h in ftab.decoy_heights(ann, 3000, 5)]
    rows = [rows[k] for k in rng.permutation(len(rows))]
    heights = [heights[k] for k in rng.permutation(len(heights))]
    db = tmp_path / "lightningd.sqlite3"
    make_db(str(db), rows, heights)
    ft = FundingTable.from_lightningd_db(str(db))
    unspent = [r for r in rows if r[5] is None]
    assert len(ft) == len(unspent) and not (ft.scid[1:] >= ft.scid[:-1]).all()
    want = {r[0] << 40 | r[1] << 16 | r[2]: (r[4], r[3]) for r in unspent}
    assert {int(s): (int(x), bytes(c)) for s, x, c in zip(ft.scid, ft.satoshis, ft.script)} == want
    assert sorted(int(b) for b in ft.blocks) == sorted(heights)
    arrs = (ft.scid, ft.satoshis, ft.script, ft.blocks)
    fs, pfs = agree_with_model(engine, fx, arrs, ann, ft)
    unchecked = sum(s >> 40 in gone for s in spent_ann)
    assert fs["no_txout"] == 30 - unchecked and fs["unchecked"] == unchecked >= 5 and fs["funded"] == 1470
    assert pfs["deleted"] == 30 - unchecked
    # the command line: export, then the audit with the table file
    out = tmp_path / "funding.tbl"
    r = subprocess.run([sys.executable, "-m", "lightning_b200.funding", "export", str(db), str(out)], cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert f"{len(unspent)} unspent outputs, {len(heights)} processed blocks" in r.stdout
    src = tmp_path / "gossip_store"
    src.write_bytes(fx)
    r = subprocess.run([TOOL, "--chain", TESTNET.hex(), "--funding", str(out), str(src)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 1, r.stdout[-2000:] + r.stderr[-2000:]
    assert (f"{fs['checked']} announcements checked: {fs['funded']} funded, {fs['unchecked']} unchecked, 0 dying, "
            f"{fs['no_txout']} no unspent output, 0 wrong script, 0 wrong amount") in r.stdout, r.stdout[-2000:]


# ---- one context, large then small then large ------------------------------------------------------------------------
def test_one_context_big_small_big(engine):
    """the engine's device buffers sized by a table of 2^22 outputs, then a table of 3, then 2^22 again (the corrupted
    table the second time): each equal to the model"""
    fx = load_fixture()
    all_good(engine, fx, 3100)
    ann = ftab.announced(fx)
    clean, bad = fixture_table("clean"), fixture_table("corrupted")
    for a, n, m in ((clean, ftab.BIG, ftab.BIG), (clean, 3, clean[3].size), (bad, ftab.BIG, 4096)):
        agree_with_model(engine, fx, ftab.pad(a, ann, n, m, seed=n), ann)
