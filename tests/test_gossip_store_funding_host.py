"""The funding check of a gossip_store on the host, no GPU: the model's script (tests/gossip_store_funding.py) against
Core Lightning's own scriptpubkey_p2wsh(bitcoin_redeem_2of2()) (oracle/funding_harness.c cln_funding_script), the host
build of the per-announcement decision k_store_funding runs (gossip_funding.cuh) against the model, and the table
exporter and file format (lightning_b200/funding.py)."""
import ctypes
import os
import sqlite3
import struct

import numpy as np
import pytest

from lightning_b200.funding import FundingTable
from lightning_b200.funding import main as funding_main
from tests import ecc
from tests import gossip_store as gs
from tests import gossip_store_funding as gf
from tests import oracle_replay
from tests.test_gossip_store_host import A, B, amount, ca, load_fixture, store_of

# cln_funding_script(key1_33, key2_33, out34) -> 1, or 0 if a key does not parse
oracle_replay.SPEC.setdefault("cln_funding_script", (lambda v: {0: 33, 1: 33}, lambda v: {2: 34}, ()))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNDING = os.path.join(ROOT, "oracle", "_ref", "libcln_funding.so")
_O = []


def oracle():
    """the reference's funding script, recorded on this module's `cln` tape"""
    if not _O:
        o = oracle_replay.Oracle("cln")
        o.lib = ctypes.CDLL(FUNDING) if (oracle_replay.RECORD_DIR or os.path.exists(FUNDING)) else None
        _O.append(o)
    return _O[0]


def cln_script(k1, k2):
    out = ctypes.create_string_buffer(34)
    assert oracle().cln_funding_script(k1, k2, out) == 1
    return out.raw


def emul_verdicts(emul, store, offs, t):
    """the host build's verdicts for the announcements at header offsets offs, table t = (scids, sats, scripts, blocks)"""
    order = np.argsort(np.array(t[0], np.uint64), kind="stable")
    scid = np.array(t[0], np.uint64)[order]
    sats = np.array(t[1], np.uint64)[order]
    script = np.frombuffer(b"".join(t[2][k] for k in order), np.uint8).copy() if len(order) else np.zeros(1, np.uint8)
    blocks = np.sort(np.array(t[3], np.uint32))
    offs = np.array(offs, np.uint64)
    out = np.zeros(max(offs.size, 1), np.uint8)
    vp = ctypes.c_void_p
    emul.emul_gf_verdict.argtypes = [ctypes.c_char_p, ctypes.c_uint64, vp, ctypes.c_size_t, vp, vp, vp, ctypes.c_uint64, vp,
                                     ctypes.c_uint64, vp]
    emul.emul_gf_verdict(store, len(store), offs.ctypes.data, offs.size, scid.ctypes.data, sats.ctypes.data,
                         script.ctypes.data, scid.size, blocks.ctypes.data, blocks.size, out.ctypes.data)
    return [int(x) for x in out[:offs.size]]


def key(k):
    return ecc.pubkey_create(k.to_bytes(32, "big"))[0]


def crafted_pairs():
    """key pairs at the edges of pubkey_cmp's memcmp order, in both argument orders: two keys equal up to the last
    byte, the same x under 02 and 03, the same key twice, and two unrelated keys"""
    a = key(11)
    b = next(a[:32] + bytes([a[32] ^ d]) for d in range(1, 256) if ecc.pubkey_convert(a[:32] + bytes([a[32] ^ d])))
    k = key(5)
    twin = bytes([k[0] ^ 1]) + k[1:]
    pairs = [(a, b), (k, twin), (k, k), (key(7), key(8))]
    return pairs + [(y, x) for x, y in pairs]


def test_script_matches_clns_for_every_fixture_announcement():
    fx = load_fixture()
    n = 0
    for off, typ, ln, st in gs.walk(fx)[0]:
        if typ == 256 and st == 0:
            _, k1, k2 = gf.ann_keys(fx, off + gs.HDR)
            assert gf.p2wsh_2of2(k1, k2) == cln_script(k1, k2), off
            n += 1
    assert n == 1500


def test_script_matches_clns_for_crafted_keys(emul):
    for k1, k2 in crafted_pairs():
        want = cln_script(k1, k2)
        assert gf.p2wsh_2of2(k1, k2) == want == gf.p2wsh_2of2(k2, k1)
        out = ctypes.create_string_buffer(34)
        emul.emul_gf_p2wsh_2of2(k1, k2, out)
        assert out.raw == want


@pytest.mark.parametrize("case", sorted(gf.fixture_cases(load_fixture())))
def test_emulated_verdicts_match_model(emul, case):
    """every live announcement of each fixture case (whatever its signature status): the host build's verdict equals the
    model's"""
    store, t = gf.fixture_cases(load_fixture())[case]
    table = gf.Table(zip(t[0], zip(t[1], t[2])), t[3])
    offs = [off for off, typ, ln, st in gs.walk(store)[0] if typ == 256 and st == 0]
    want = [gf.verdict(store, off, table) for off in offs]
    assert emul_verdicts(emul, store, offs, t) == want
    counts = {v: want.count(v) for v in set(want)}
    expect = {"clean": {}, "no_txout": {gf.GF_NO_TXOUT: 1}, "unchecked": {gf.GF_UNCHECKED: 1},
              "script_unsorted_keys": {gf.GF_SCRIPT: 1}, "script_other_key": {gf.GF_SCRIPT: 1},
              "amount_off_by_one": {gf.GF_AMOUNT: 1}, "amount_record_removed": {gf.GF_AMOUNT: 1},
              "amount_record_replaced": {gf.GF_AMOUNT: 1}, "dying": {gf.GF_DYING: 1},
              "refused_holder_then_funded_copy": {gf.GF_AMOUNT: 1}}[case]
    for v, c in expect.items():
        assert counts.get(v, 0) == c, (case, counts)
    assert set(counts) <= {gf.GF_FUNDED} | set(expect)


def test_emulated_verdicts_on_crafted_edges(emul):
    """an amount record cut off by the end of the store, one with another type, a table without outputs or blocks"""
    s = struct.unpack(">Q", A)[0]
    keys_script = gf.p2wsh_2of2(*gf.ann_keys(ca(A), 0)[1:])
    t = ([s], [1000], [keys_script], [s >> 40])
    cases = [store_of(gs.record(ca(A)), gs.record(amount())),
             store_of(gs.record(ca(A)), gs.record(amount()))[:-1],
             store_of(gs.record(ca(A)), gs.record(struct.pack(">HQ", 4107, 1000))),
             store_of(gs.record(ca(A)), gs.record(amount(), flags=gs.COMPLETED | gs.DELETED)),
             store_of(gs.record(ca(A)))]
    want_all = [gf.GF_FUNDED, gf.GF_AMOUNT, gf.GF_AMOUNT, gf.GF_FUNDED, gf.GF_AMOUNT]
    for store, w in zip(cases, want_all):
        table = gf.Table({s: (1000, keys_script)}, [s >> 40])
        assert gf.verdict(store, 1, table) == w
        assert emul_verdicts(emul, store, [1], t) == [w]
    store = cases[0]
    for tt, w in ((([], [], [], []), gf.GF_UNCHECKED), (([], [], [], [s >> 40]), gf.GF_NO_TXOUT),
                  (([struct.unpack(">Q", B)[0]], [1000], [keys_script], []), gf.GF_UNCHECKED)):
        assert gf.verdict(store, 1, gf.Table(zip(tt[0], zip(tt[1], tt[2])), tt[3])) == w
        assert emul_verdicts(emul, store, [1], tt) == [w]


# ---- lightningd.sqlite3 -> FundingTable ------------------------------------------------------------------------------
def make_db(path, rows, heights):
    """a database with the two tables get_txout reads, holding only the columns the exporter asks for"""
    con = sqlite3.connect(path)
    con.execute("CREATE TABLE utxoset (blockheight INTEGER, txindex INTEGER, outnum INTEGER, scriptpubkey BLOB, "
                "satoshis BIGINT, spendheight INTEGER)")
    con.execute("CREATE TABLE blocks (height INTEGER)")
    con.executemany("INSERT INTO utxoset VALUES (?, ?, ?, ?, ?, ?)", rows)
    con.executemany("INSERT INTO blocks VALUES (?)", [(h,) for h in heights])
    con.commit()
    con.close()


def scid_bytes(block, txindex, outnum):
    return struct.pack(">Q", block << 40 | txindex << 16 | outnum)


def test_export_follows_get_txout(tmp_path, emul):
    keys = gf.ann_keys(ca(A), 0)[1:]
    good = gf.p2wsh_2of2(*keys)
    rows = [(700000, 5, 1, good, 50000, None),        # unspent, processed block
            (700000, 6, 0, good, 60000, 700100),      # spent
            (700001, 1, 1, good, 70000, None),        # unspent, in a block the blocks table does not list
            (700002, 2, 0, b"\x00\x14" + bytes(32), 1, 700050)]  # spent, and not P2WSH: spent rows are not read
    db = tmp_path / "lightningd.sqlite3"
    make_db(str(db), rows, [700000, 700002])
    t = FundingTable.from_lightningd_db(str(db))
    assert sorted(int(s) for s in t.scid) == [700000 << 40 | 5 << 16 | 1, 700001 << 40 | 1 << 16 | 1]
    assert sorted(int(b) for b in t.blocks) == [700000, 700002]
    model = gf.Table.of(t)
    arrays = ([int(x) for x in t.scid], [int(x) for x in t.satoshis], [bytes(x) for x in t.script],
              [int(x) for x in t.blocks])
    # one announcement per scid; its verdict follows get_txout: the unspent output; a processed block without it; not
    # processed
    cases = {(700000, 5, 1): gf.GF_FUNDED, (700000, 6, 0): gf.GF_NO_TXOUT, (700001, 1, 1): gf.GF_FUNDED,
             (700002, 2, 0): gf.GF_NO_TXOUT, (700000, 9, 9): gf.GF_NO_TXOUT, (700003, 1, 0): gf.GF_UNCHECKED}
    sats = {(700000, 5, 1): 50000, (700001, 1, 1): 70000}
    for sc, want in cases.items():
        store = store_of(gs.record(ca(scid_bytes(*sc))), gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, sats.get(sc, 1))))
        assert gf.verdict(store, 1, model) == want, sc
        assert emul_verdicts(emul, store, [1], arrays) == [want], sc
    # the command line writes the same table
    out = tmp_path / "funding.tbl"
    assert funding_main(["export", str(db), str(out)]) == 0
    u = FundingTable.load(str(out))
    assert np.array_equal(u.scid, t.scid) and np.array_equal(u.satoshis, t.satoshis)
    assert np.array_equal(u.script, t.script) and np.array_equal(u.blocks, t.blocks)


def test_export_refuses_other_scripts_and_duplicates(tmp_path):
    good = gf.p2wsh_2of2(*gf.ann_keys(ca(A), 0)[1:])
    db = tmp_path / "short.sqlite3"
    make_db(str(db), [(700000, 5, 1, good, 1, None), (700000, 5, 2, b"\x00\x14" + bytes(20), 1, None)], [700000])
    with pytest.raises(ValueError, match="34"):
        FundingTable.from_lightningd_db(str(db))
    db = tmp_path / "dup.sqlite3"
    make_db(str(db), [(700000, 5, 1, good, 1, None), (700000, 5, 1, good, 2, None)], [700000])
    with pytest.raises(ValueError, match="twice"):
        FundingTable.from_lightningd_db(str(db))
    # the database is opened read-only: the exporter never creates one
    with pytest.raises(sqlite3.OperationalError):
        FundingTable.from_lightningd_db(str(tmp_path / "missing.sqlite3"))
    assert not (tmp_path / "missing.sqlite3").exists()


def test_file_round_trip_and_refusals(tmp_path):
    rng = np.random.default_rng(7)
    n = 300
    t = FundingTable.from_arrays(rng.choice(1 << 50, n, replace=False).astype(np.uint64),
                                 rng.integers(0, 1 << 40, n, dtype=np.uint64), rng.integers(0, 256, (n, 34), dtype=np.uint8),
                                 rng.integers(0, 900000, 40, dtype=np.uint32))
    p = tmp_path / "t.tbl"
    t.save(str(p))
    data = p.read_bytes()
    assert data[:8] == b"CLNFUND1" and len(data) == 24 + 50 * n + 4 * 40
    assert struct.unpack_from("<QQ", data, 8) == (n, 40)
    assert struct.unpack_from("<QQ", data, 24) == (int(t.scid[0]), int(t.satoshis[0]))
    u = FundingTable.load(str(p))
    for f in ("scid", "satoshis", "script", "blocks"):
        assert np.array_equal(getattr(u, f), getattr(t, f)), f
    empty = FundingTable.from_arrays([], [], np.zeros((0, 34), np.uint8), [])
    assert len(FundingTable.from_bytes(empty.to_bytes())) == 0
    with pytest.raises(ValueError, match="magic"):
        FundingTable.from_bytes(b"CLNFUND2" + data[8:])
    for cut in (0, 7, 23, 24 + 49, len(data) - 1):
        with pytest.raises(ValueError):
            FundingTable.from_bytes(data[:cut])
    with pytest.raises(ValueError):
        FundingTable.from_bytes(data + b"\x00")
    with pytest.raises(ValueError, match="twice"):
        FundingTable.from_arrays([1, 1], [0, 0], np.zeros((2, 34), np.uint8), [])
