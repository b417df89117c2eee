"""The funding check with tables shaped as lightningd exports them, on the host, no GPU (tests/funding_tables.py).

The engine sorts the table's scids with CUB and carries each output's entry index through the sort; gf_verdict then reads
the amount and script of entry out_idx[i].  Here the host build of gf_verdict (gossip_funding.cuh) gets the sorted scids
with numpy's argsort as that index, for every order and with decoys, against the model (tests/gossip_store_funding.py).
The store whose announcements carry features fields of many lengths goes through it too.  And the helpers themselves
are checked: decoys never hit an announced scid, every single-bit neighbour is there, sizes are exact, and padding or
reordering changes no verdict of the model."""
import ctypes

import numpy as np
import pytest

from tests import funding_tables as ftab
from tests import gossip_store as gs
from tests import gossip_store_funding as gf
from tests.test_gossip_store_funding_host import emul_verdicts
from tests.test_gossip_store_host import load_fixture

CASES = sorted(gf.fixture_cases(load_fixture()))


def ann_offs(store):
    return [off for off, typ, ln, st in gs.walk(store)[0] if typ == 256 and st == 0]


def indexed_verdicts(emul, store, offs, a):
    """the host build's verdicts with the engine's index array: scids sorted, out_idx into the table as given"""
    sc, sa, sp, bl = a
    idx = np.argsort(sc, kind="stable").astype(np.uint32)
    keys = np.ascontiguousarray(sc[idx])
    sa, sp = np.ascontiguousarray(sa), np.ascontiguousarray(sp).reshape(-1)
    if not sp.size:
        sp = np.zeros(1, np.uint8)
    blocks = np.sort(bl)
    offs = np.array(offs, np.uint64)
    out = np.zeros(max(offs.size, 1), np.uint8)
    vp = ctypes.c_void_p
    f = emul.emul_gf_verdict_indexed
    f.argtypes = [ctypes.c_char_p, ctypes.c_uint64, vp, ctypes.c_size_t, vp, vp, vp, vp, ctypes.c_uint64, vp,
                  ctypes.c_uint64, vp]
    f(store, len(store), offs.ctypes.data, offs.size, keys.ctypes.data, idx.ctypes.data, sa.ctypes.data, sp.ctypes.data,
      keys.size, blocks.ctypes.data, blocks.size, out.ctypes.data)
    return [int(x) for x in out[:offs.size]]


def want(store, offs, a, ann):
    table = ftab.model(a, ann)
    return [gf.verdict(store, off, table) for off in offs]


@pytest.mark.parametrize("order", ftab.ORDERS)
@pytest.mark.parametrize("case", CASES)
def test_indexed_verdicts_every_order(emul, case, order):
    """each fixture case, its table in each order with 20,000 decoys mixed in: the host build reading through the index
    array gives the model's verdicts, which are those of the sorted table without decoys"""
    store, t = gf.fixture_cases(load_fixture())[case]
    ann = ftab.announced(store)
    a = ftab.arrays(t)
    padded = ftab.pad(a, ann, a[0].size + 20000, a[3].size + 2000, seed=CASES.index(case))
    r = ftab.reorder(padded, order, seed=7)
    offs = ann_offs(store)
    w = want(store, offs, a, ann)
    assert want(store, offs, r, ann) == w
    assert indexed_verdicts(emul, store, offs, r) == w
    # the index array is not the identity: an entry read at its sorted position instead would be another output
    assert not np.array_equal(np.argsort(r[0], kind="stable"), np.arange(r[0].size))


def test_indexed_corrupted_table_shuffled(emul):
    """2 % of the table wrong (every refused verdict and unchecked), shuffled with decoys, every height twice"""
    fx = load_fixture()
    a = ftab.arrays(gf.corrupt_table(gf.table_of_store(fx), 0.02, 53))
    ann = ftab.announced(fx)
    r = ftab.reorder(ftab.pad(a, ann, 60000, 5000, seed=53), "shuffled_heights_twice", seed=53)
    offs = ann_offs(fx)
    w = want(fx, offs, a, ann)
    assert {gf.GF_NO_TXOUT, gf.GF_UNCHECKED, gf.GF_SCRIPT, gf.GF_AMOUNT} <= set(w)
    assert indexed_verdicts(emul, fx, offs, r) == w
    assert emul_verdicts(emul, fx, offs, (r[0], r[1], [x.tobytes() for x in r[2]], r[3])) == w


@pytest.mark.parametrize("n,m", [(0, None), (None, 0), (1, None), (2, None), (3, None), (ftab.TILE_OUT + 1, ftab.TILE_BLK + 1),
                                 ((1 << 16) + 1, (1 << 16) + 1)])
def test_indexed_sizes(emul, n, m):
    fx = load_fixture()
    a = ftab.arrays(gf.table_of_store(fx))
    ann = ftab.announced(fx)
    p = ftab.pad(a, ann, a[0].size if n is None else n, a[3].size if m is None else m, seed=11)
    offs = ann_offs(fx)
    assert indexed_verdicts(emul, fx, offs, p) == want(fx, offs, p, ann)


def test_features_store(emul):
    """announcements with features fields of 0 to 1,000 bytes, each with every verdict: the host build (sorted and
    through the index array) reads the scid and keys after the features, as the model does"""
    store, a, what = ftab.features_store()
    ann = ftab.announced(store)
    offs = ann_offs(store)
    assert len(offs) == len(ftab.FLENS) * len(ftab.KINDS)
    w = want(store, offs, a, ann)
    kinds = {"funded": gf.GF_FUNDED, "script": gf.GF_SCRIPT, "amount": gf.GF_AMOUNT, "no_txout": gf.GF_NO_TXOUT,
             "unchecked": gf.GF_UNCHECKED}
    assert w == [kinds[what[gf.ann_keys(store, off + gs.HDR)[0]][1]] for off in offs]
    assert {what[gf.ann_keys(store, off + gs.HDR)[0]][0] for off in offs} == set(ftab.FLENS)
    assert emul_verdicts(emul, store, offs, (a[0], a[1], [x.tobytes() for x in a[2]], a[3])) == w
    for order in ftab.ORDERS:
        assert indexed_verdicts(emul, store, offs, ftab.reorder(a, order, 3)) == w, order
    # a read at m + 260, ignoring the features length, would see a funded output for every long-features announcement
    t = ftab.model(a, ann)
    for off in offs:
        flen, kind = what[gf.ann_keys(store, off + gs.HDR)[0]]
        if flen >= 172:
            m = off + gs.HDR
            f = m + 260
            s = int.from_bytes(store[f + 32:f + 40], "big")
            assert s in t.outputs and t.outputs[s][1] == gf.p2wsh_2of2(store[f + 106:f + 139], store[f + 139:f + 172])


# ---- the helpers --------------------------------------------------------------------------------------------------------
def test_decoys_never_hit_and_cover_every_bit():
    fx = load_fixture()
    a = ftab.arrays(gf.table_of_store(fx))
    ann = ftab.announced(fx)
    assert ann.size == 1500
    d = ftab.decoys(a, ann, 200000, seed=5, flips=ann.size)
    assert d[0].size == 200000 and np.unique(d[0]).size == d[0].size
    assert not np.isin(d[0], ann).any()
    got = set(d[0].tolist())
    annset = set(ann.tolist())
    for s in ann.tolist():
        flips = {s ^ (1 << b) for b in range(64)} - annset
        assert flips <= got, s
        blk, tx, out = s >> 40, (s >> 16) & 0xFFFFFF, s & 0xFFFF
        near = {gf_scid(blk, tx + 1, out), gf_scid(blk, tx - 1, out), gf_scid(blk, tx, out + 1), gf_scid(blk, tx, out - 1),
                gf_scid(blk + 1, tx, out), gf_scid(blk - 1, tx, out)} - {None} - annset
        assert near <= got, s
    assert {0, 1, (1 << 64) - 1, ((1 << 24) - 1) << 40} <= got
    # every decoy carries a real entry's script; some amounts have bit 63 set
    scripts = {x.tobytes() for x in a[2]}
    assert all(x.tobytes() in scripts for x in d[2][:1000])
    assert (d[1] >= np.uint64(1 << 63)).any() and (d[1] < np.uint64(1 << 63)).any()
    # a smaller count is a sample of the structured decoys, still never an announced scid
    small = ftab.decoys(a, ann, 500, seed=6)
    assert small[0].size == 500 and not np.isin(small[0], ann).any()
    h = ftab.decoy_heights(ann, 10000, seed=3)
    assert h.size == 10000 and np.unique(h).size == h.size
    assert not np.isin(h, (ann >> np.uint64(40)).astype(np.uint32)).any()


def gf_scid(blk, tx, out):
    if 0 <= blk < 1 << 24 and 0 <= tx < 1 << 24 and 0 <= out < 1 << 16:
        return blk << 40 | tx << 16 | out
    return None


@pytest.mark.parametrize("n", [0, 1, 3, 1499, 1500, 1501] + list(ftab.SIZES[:11]) + [(1 << 16) + 1])
def test_pad_sizes_exact_and_model_unchanged(n):
    fx = load_fixture()
    a = ftab.arrays(gf.table_of_store(fx))
    ann = ftab.announced(fx)
    m = max(n, a[3].size)
    p = ftab.pad(a, ann, n, m, seed=n)
    assert p[0].size == p[1].size == p[2].shape[0] == n and p[3].size == m
    assert np.unique(p[0]).size == n
    if n >= a[0].size:
        assert ftab.same_model(a, p, ann)
    else:  # a subset of the real outputs, with all their heights
        keep = np.isin(a[0], p[0])
        assert keep.sum() == n and ftab.same_model(ftab.take(a, np.nonzero(keep)[0]), p, ann)


@pytest.mark.parametrize("order", ftab.ORDERS)
def test_reorder_keeps_the_table(order):
    fx = load_fixture()
    a = ftab.arrays(gf.table_of_store(fx))
    ann = ftab.announced(fx)
    p = ftab.pad(a, ann, 9000, 3000, seed=1)
    r = ftab.reorder(p, order, seed=2)
    s, rs = ftab.sort(p), ftab.sort(r)
    assert all(np.array_equal(x, y) for x, y in zip(s[:3], rs[:3]))
    assert np.array_equal(np.unique(s[3]), np.unique(rs[3]))
    assert rs[3].size == (2 if order == "shuffled_heights_twice" else 1) * s[3].size
    assert not np.array_equal(r[0], s[0])
    if order == "low_bits_first":
        low = r[0] & np.uint64(0xFFFF)
        assert (np.diff(low.astype(np.int64)) >= 0).all()
    assert ftab.same_model(p, r, ann)
    offs = ann_offs(fx)
    assert want(fx, offs, r, ann) == want(fx, offs, a, ann)
