"""GPU: the funding check of a gossip_store (sv_verify_gossip_store_funding_host, sv_prune_gossip_store_funding_host).
The committed store fixture with a table built from its own announcements and amount records, then one deterministic
mutation per verdict, each checked on the device against the model (tests/gossip_store_funding.py, with CLN's own
gossipd/sigcheck.c as its sigcheck).  The pruned store must load under Core Lightning's gossmap.c strictly, as gossipd
loads it at start-up (oracle/gossmap_strict_harness.c), and every channel it holds must be funded, unchecked or dying
in the table, with the capacity the table gives.  Then the same on the fixture tiled x53 with 1 % of the table wrong,
the Python binding without a table, and the command line's exit codes."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200.funding import FundingTable
from tests import gossip_store as gs
from tests import gossip_store_funding as gf
from tests import oracle_replay
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_prune_host import strict_load
from tests.test_gpu_gossip_burst import TESTNET
from tests.test_gpu_gossip_store import TOOL, cln_sigcheck
from tests.test_gpu_gossip_store_prune import _Both, corrupted_x53, memo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOSSMAP = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap_strict.so")
_O = []


def oracle():
    """CLN's sigcheck and its strict gossmap load behind one recorded oracle (this module's `cln` tape)"""
    if not _O:
        o = oracle_replay.Oracle("cln")
        if o.lib is not None and os.path.exists(GOSSMAP):
            o.lib = _Both(o.lib, ctypes.CDLL(GOSSMAP))
        _O.append(o)
    return _O[0]


def funding_table(t):
    return FundingTable.from_arrays(np.array(t[0], np.uint64), np.array(t[1], np.uint64),
                                    np.frombuffer(b"".join(t[2]), np.uint8).reshape(-1, 34) if t[2] else
                                    np.zeros((0, 34), np.uint8), np.array(t[3], np.uint32))


def check(engine, store, t, chain=TESTNET):
    """audit + funding and prune + funding against the model; the pruned store against gossmap's strict load.
    -> (prune summary, funding summary of the prune)"""
    o = oracle()
    sig = memo(cln_sigcheck(o, chain))
    ft = funding_table(t)
    table = gf.Table.of(ft)
    before = bytes(store)
    # the audit: its outputs are the plain audit's, plus the verdicts
    off, typ, st, hold, s, fund, fs = engine.verify_gossip_store(store, chain, funding=ft)
    plain = engine.verify_gossip_store(store, chain)
    for a, b in zip((off, typ, st, hold), plain[:4]):
        assert np.array_equal(a, b)
    assert s == plain[4]
    rows, _, wfund, wfs = gf.audit(store, table, sig)
    assert [int(x) for x in fund] == wfund
    assert fs == wfs
    # the prune
    out, (poff, ptyp, pst, why), ps, pfund, pfs = engine.prune_gossip_store(store, chain, funding=ft)
    assert store == before
    want, wrows, ws, wpfund, wpfs = gf.prune(store, table, sig)
    assert out == want
    assert [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(poff, ptyp, pst, why)] == wrows
    assert [int(x) for x in pfund] == wpfund
    for k, v in ws.items():
        assert ps[k] == v, k
    assert pfs == wpfs
    if pfs["deleted"] == 0:
        p_out, p_recs, p_s = engine.prune_gossip_store(store, chain)
        assert (p_out, p_s) == (out, ps) and all(np.array_equal(a, b) for a, b in zip(p_recs, (poff, ptyp, pst, why)))
    # the result audits clean with the table, and pruning it again deletes nothing
    _, _, _, _, a, _, afs = engine.verify_gossip_store(out, chain, funding=ft)
    assert a["stop"] == gs.EOF and a["end_offset"] == len(out)
    assert (a["bad_signature"], a["malformed"], a["no_channel"], a["wrong_chain"], a["bad_order"],
            a["redundant_announcements"], a["unknown"]) == (0,) * 7
    assert afs["no_txout"] == afs["script"] == afs["amount"] == 0
    again, _, s2, _, fs2 = engine.prune_gossip_store(out, chain, funding=ft)
    assert again == out and s2["pruned"] == 0 and fs2["deleted"] == 0
    # gossmap's strict load accepts it; every channel it holds is funded, unchecked or dying, with the table's capacity
    ref = strict_load(o, out)
    assert ref is not None, "gossmap's strict load refused the pruned store"
    end, chans, _ = ref
    assert end == len(out)
    for scid, cann, _, _ in chans:
        hdr = cann - gs.HDR
        v = gf.verdict(out, hdr, table)
        assert v in (gf.GF_FUNDED, gf.GF_UNCHECKED, gf.GF_DYING), (scid, v)
        if v == gf.GF_FUNDED:
            a = hdr + gs.HDR + struct.unpack(">H", out[hdr + 2:hdr + 4])[0]
            assert struct.unpack(">Q", out[a + gs.HDR + 2:a + gs.HDR + 10])[0] == table.outputs[scid][0]
    return ps, pfs


CASES = sorted(gf.fixture_cases(load_fixture()))


@pytest.mark.parametrize("case", CASES)
def test_mutation(engine, case):
    store, t = gf.fixture_cases(load_fixture())[case]
    ps, pfs = check(engine, store, t)
    refused = {"no_txout": "no_txout", "script_unsorted_keys": "script", "script_other_key": "script",
               "amount_off_by_one": "amount", "amount_record_removed": "amount", "amount_record_replaced": "amount",
               "refused_holder_then_funded_copy": "amount"}
    if case in refused:
        assert pfs[refused[case]] == 1 and pfs["deleted"] == 1
    else:
        assert pfs["deleted"] == 0
    if case == "clean":
        assert pfs["funded"] == pfs["checked"] == 1500 and ps["pruned"] == 0
    if case == "unchecked":
        assert pfs["unchecked"] == 1
    if case == "dying":
        assert pfs["dying"] == 1
    if case == "refused_holder_then_funded_copy":
        assert ps["no_channel"] > 0 and ps["amount"] == 1 and pfs["funded"] == 1500 and pfs["checked"] == 1501


def test_tiled_x53_table_corrupted(engine):
    fx = load_fixture()
    t = gf.corrupt_table(gf.table_of_store(fx), 0.01, 53)
    assert len(t[0]) < 1500
    ps, pfs = check(engine, corrupted_x53(), t)
    assert pfs["deleted"] > 0 and pfs["checked"] > 1500 * 51


def test_without_table_unchanged(engine):
    """funding=None makes exactly the calls without a table; a table that funds everything changes nothing of theirs"""
    fx = load_fixture()
    store, t = gf.fixture_cases(fx)["clean"]
    ft = funding_table(t)
    lib = engine.lib
    n = int(lib.sv_gossip_store_count(store, len(store)))
    a = engine.verify_gossip_store(store, TESTNET)
    b = engine.verify_gossip_store(store, TESTNET, funding=ft)
    assert len(a) == 5 and all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4])) and a[4] == b[4]
    assert a[0].size == n
    p = engine.prune_gossip_store(store, TESTNET)
    q = engine.prune_gossip_store(store, TESTNET, funding=ft)
    assert len(p) == 3 and p[0] == q[0] and p[2] == q[2]


def test_duplicate_scid_refused(engine):
    store, t = gf.fixture_cases(load_fixture())["clean"]
    ft = funding_table(t)
    ft.scid[1] = ft.scid[0]  # the constructor checked; the engine checks again
    with pytest.raises(Exception, match="twice"):
        engine.verify_gossip_store(store, TESTNET, funding=ft)
    with pytest.raises(Exception, match="twice"):
        engine.prune_gossip_store(store, TESTNET, funding=ft)


def test_profiling_reports_funding_time(engine):
    store, t = gf.fixture_cases(load_fixture())["clean"]
    engine.set_profiling(True)
    try:
        engine.verify_gossip_store(store, TESTNET, funding=funding_table(t))
        stage, kernel = engine.last_gossip_funding_timing()
        assert stage > 0 and kernel > 0
    finally:
        engine.set_profiling(False)


def test_cli_funding(tmp_path):
    cases = gf.fixture_cases(load_fixture())
    chain = ["--chain", TESTNET.hex()]

    def run(name, *extra):
        store, t = cases[name]
        src, tbl = tmp_path / f"{name}.store", tmp_path / f"{name}.tbl"
        src.write_bytes(store)
        funding_table(t).save(str(tbl))
        r = subprocess.run([TOOL] + chain + ["--funding", str(tbl)] + list(extra) + [str(src)], capture_output=True,
                           text=True, timeout=300)
        return r, src, store

    r, _, _ = run("clean")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "1500 funded" in r.stdout
    # unchecked and dying never change the exit code
    for name in ("unchecked", "dying"):
        r, _, _ = run(name)
        assert r.returncode == 0, (name, r.stdout[-2000:])
    r, _, _ = run("no_txout")
    assert r.returncode == 1 and "no unspent output" in r.stdout
    dst = tmp_path / "pruned"
    r, src, store = run("amount_off_by_one", "--prune", str(dst))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert src.read_bytes() == store and dst.read_bytes() != store and "clean" in r.stdout
    assert "1 announcement gossipd would refuse" in r.stdout
    # a walk stopped at a bad checksum: 2, as without a table
    store, t = cases["clean"]
    recs = gs.walk(store)[0]
    st = bytearray(store)
    st[recs[1200][0] + gs.HDR + 20] ^= 4
    cases["bad_crc"] = (bytes(st), t)
    r, _, _ = run("bad_crc")
    assert r.returncode == 2, r.stdout[-2000:]
    # OUT not clean: its walk stops at an incomplete last record, which the prune leaves alone
    last = recs[-1][0]
    st = bytearray(store)
    st[last] &= ~(gs.COMPLETED >> 8) & 0xFF
    cases["incomplete_tail"] = (bytes(st), t)
    r, _, _ = run("incomplete_tail", "--prune", str(tmp_path / "pruned2"))
    assert r.returncode == 1 and "NOT clean" in r.stdout, r.stdout[-2000:]
    # a table file that is not one: 3, before the store is read
    bad = tmp_path / "bad.tbl"
    bad.write_bytes(b"CLNFUND2" + bytes(16))
    r = subprocess.run([TOOL, "--funding", str(bad), str(src)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 3
