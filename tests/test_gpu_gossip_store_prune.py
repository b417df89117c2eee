"""GPU: pruning a gossip_store (sv_prune_gossip_store_host).  Deterministic mutations of the committed store fixture,
each pruned on the device and checked against the model (tests/gossip_store_prune.py, with CLN's own gossipd/sigcheck.c
as its sigcheck), against the audit of the result, and against Core Lightning's gossmap.c loading the result strictly as
gossipd does at start-up (oracle/gossmap_strict_harness.c cln_gossmap_load_strict): the load must succeed, and every channel it
holds, every current channel_update and every current node_announcement must verify under CLN's sigcheck.  Then the
same on the fixture tiled x53 with 1 % of its records corrupted."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200.engine import SvGossipPruneSummary
from tests import gossip_store as gs
from tests import gossip_store_prune as gp
from tests import oracle_replay
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_prune_host import strict_load
from tests.test_gpu_gossip_burst import OTHER, TESTNET, _ordered, make_ca, make_cu
from tests.test_gpu_gossip_store import TOOL, cln_sigcheck

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOSSMAP = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap_strict.so")


class _Both:
    """CLN's sigcheck library and its gossmap library behind one recorded oracle (one tape per test module)"""

    def __init__(self, *libs):
        self.libs = libs

    def __getattr__(self, name):
        for lib in self.libs:
            if hasattr(lib, name):
                return getattr(lib, name)
        raise AttributeError(name)


_O = []


def oracle():
    if not _O:
        o = oracle_replay.Oracle("cln")
        if o.lib is not None and os.path.exists(GOSSMAP):
            o.lib = _Both(o.lib, ctypes.CDLL(GOSSMAP))
        _O.append(o)
    return _O[0]


def memo(f):
    """the model's sigcheck, asked once per distinct (message, signer): the tiled store repeats its messages"""
    seen = {}

    def g(m, signer):
        k = (bytes(m), None if signer is None else bytes(signer))
        if k not in seen:
            seen[k] = f(m, signer)
        return seen[k]
    return g


def flip_sig(rec_bytes, k=0):
    """a record with bit 0 of signature k's byte 10 flipped, checksum recomputed"""
    r = bytearray(rec_bytes)
    r[12 + 2 + 64 * k + 10] ^= 1
    gs.reseal(r, 0)
    return bytes(r)


def records_of(store):
    recs = gs.walk(store)[0]
    return recs, lambda i: store[recs[i][0]:recs[i][0] + 12 + recs[i][2]]


def scid_of_update(store, off):
    return store[off + 12 + 98:off + 12 + 106]


def mutations():
    """name -> mutated store, one per case of the prune rules"""
    fx = load_fixture()
    recs, rec = records_of(fx)
    anns = [i for i, r in enumerate(recs) if r[1] == 256]
    upds = [i for i, r in enumerate(recs) if r[1] == 258]
    nanns = [i for i, r in enumerate(recs) if r[1] == 257]
    out = {}
    # a failing holding announcement, then a good redundant copy of it, the channel's updates before and after the copy
    i = anns[100]
    scid = gs.ann_fields(fx, recs[i][0] + 12)[1]
    mine = [u for u in upds if scid_of_update(fx, recs[u][0]) == scid]
    assert mine
    st = bytearray(fx)
    st[recs[i][0]:recs[i][0] + 12 + recs[i][2]] = flip_sig(rec(i), 2)
    out["bad_holder_then_redundant"] = bytes(st) + rec(i) + rec(i + 1) + b"".join(rec(u) for u in mine)
    # a bad newest update after a good one; a bad newest node_announcement after a good one
    out["bad_newest_update"] = fx + flip_sig(rec(upds[300]))
    out["bad_newest_node_announcement"] = fx + flip_sig(rec(nanns[40]))
    # a malformed update (cut short), an update of another chain, an announcement with its node ids out of order
    a, b = _ordered("a", "b")
    A = b"\x00\x00\x01\x00\x00\x02\x00\x01"
    short = make_cu(A, a, 0)[:100]
    out["malformed_chain_order"] = fx + gs.record(make_ca(A, a, b)) + gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 1)) + \
        gs.record(short) + gs.record(make_cu(A, a, 0, chain=OTHER)) + gs.record(make_ca(A[:7] + b"\x02", a, b, swap=True)) + \
        gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 1)) + gs.record(make_cu(A, b, 1))
    # a bad checksum and a truncated record in mid-store, an unknown record type in mid-store
    mid = recs[2300][0]
    st = bytearray(fx)
    st[recs[1200][0] + 12 + 20] ^= 4
    out["bad_crc_and_truncated"] = bytes(st[:mid]) + gs.record(b"\x01") + bytes(st[mid:])
    out["unknown_type"] = fx[:mid] + gs.record(struct.pack(">HI", 4999, 1)) + fx[mid:]
    # an update of a channel a delete_chan removed
    u = upds[500]
    out["update_after_delete_chan"] = fx + gs.record(struct.pack(">H", gs.DELETE_CHAN) + scid_of_update(fx, recs[u][0])) + rec(u)
    return out


def corrupted_x53():
    """the fixture tiled x53 with ~1 % of its records corrupted: a flipped signature bit (checksum recomputed), a
    flipped message bit (checksum left), or an unknown type"""
    fx = load_fixture()
    store = bytearray(fx[:1] + fx[1:] * 53)
    rng = np.random.default_rng(53)
    recs = gs.walk(bytes(store))[0]
    for off, t, ln, _ in recs:
        if rng.random() >= 0.01:
            continue
        k = int(rng.integers(0, 3))
        if k == 0 and t in (256, 257, 258):
            store[off + 12 + 2 + int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
            gs.reseal(store, off)
        elif k == 1:
            store[off + 12 + int(rng.integers(2, ln))] ^= 1
        else:
            store[off + 12:off + 14] = struct.pack(">H", 4999)
            gs.reseal(store, off)
    return bytes(store)


def check(engine, store, chain=TESTNET):
    o = oracle()
    sig = memo(cln_sigcheck(o, chain))
    before = bytes(store)
    out, (off, typ, status, why), s = engine.prune_gossip_store(store, chain)
    assert store == before
    want, rows, ws = gp.prune(store, sig)
    assert out == want
    assert [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(off, typ, status, why)] == rows
    for k, v in ws.items():
        assert s[k] == v, k
    # the audit of the result is clean
    _, _, ast, _, a = engine.verify_gossip_store(out, chain)
    assert a["stop"] == gs.EOF and a["end_offset"] == len(out)
    assert (a["bad_signature"], a["malformed"], a["no_channel"], a["wrong_chain"], a["bad_order"],
            a["redundant_announcements"], a["unknown"]) == (0,) * 7
    # pruning it again deletes nothing
    again, _, s2 = engine.prune_gossip_store(out, chain)
    assert again == out and s2["pruned"] == 0
    # gossmap's strict load accepts it, and what it holds verifies under CLN's sigcheck
    ref = strict_load(o, out)
    assert ref is not None, "gossmap's strict load refused the pruned store"
    end, chans, nodes = ref
    assert end == len(out)
    for _, cann, up0, up1 in chans:
        m = out[cann:cann + struct.unpack(">H", out[cann - 10:cann - 8])[0]]
        assert sig(m, None) == 0
        for d, u in enumerate((up0, up1)):
            if u:
                assert sig(out[u:u + struct.unpack(">H", out[u - 10:u - 8])[0]], gs.ann_fields(m)[2 + d]) == 0
    for n in nodes:
        if n:
            assert sig(out[n:n + struct.unpack(">H", out[n - 10:n - 8])[0]], None) == 0
    return s


@pytest.mark.parametrize("case", sorted(mutations()))
def test_mutation(engine, case):
    store = mutations()[case]
    s = check(engine, store)
    assert s["pruned"] > 0
    expect = {"bad_holder_then_redundant": ("message", "no_channel"), "bad_newest_update": ("signature",),
              "bad_newest_node_announcement": ("message",), "malformed_chain_order": ("message",),
              "bad_crc_and_truncated": ("bad_crc", "truncated"), "unknown_type": ("unknown",),
              "update_after_delete_chan": ("no_channel",)}[case]
    for k in expect:
        assert s[k] > 0, k
    if case == "bad_holder_then_redundant":
        assert s["reverified"] > 0 and s["amount"] == 1


def test_clean_fixture_unchanged(engine):
    fx = load_fixture()
    for chain in (None, TESTNET):
        out, (_, _, _, why), s = engine.prune_gossip_store(fx, chain)
        assert out == fx and s["pruned"] == 0 and not why.any() and s["records"] == 4600


def test_in_place_and_input_untouched(engine):
    """the C call with out == store prunes in place; with another out it leaves the input alone"""
    store = mutations()["bad_newest_update"]
    want = engine.prune_gossip_store(store, TESTNET)[0]
    lib = engine.lib
    n = int(lib.sv_gossip_prune_count(store, len(store)))
    arrs = [np.zeros(n, d) for d in (np.uint64, np.uint16, np.int32, np.uint8)]
    chain = np.frombuffer(TESTNET, np.uint8).copy()
    for in_place in (False, True):
        buf = np.frombuffer(store, np.uint8).copy()
        out = buf if in_place else np.zeros_like(buf)
        s = SvGossipPruneSummary()
        assert lib.sv_prune_gossip_store_host(engine._ctx, buf.ctypes.data, buf.size, chain.ctypes.data, out.ctypes.data,
                                              *(a.ctypes.data for a in arrs), n, ctypes.byref(s)) == 0
        assert out.tobytes() == want
        assert in_place or buf.tobytes() == store
    # argument errors write nothing
    s = SvGossipPruneSummary()
    out = np.zeros(len(store), np.uint8)
    assert lib.sv_prune_gossip_store_host(engine._ctx, store, len(store), None, out.ctypes.data,
                                          *(a.ctypes.data for a in arrs), n - 1, ctypes.byref(s)) != 0
    bad = bytes([0x20]) + store[1:]
    assert lib.sv_prune_gossip_store_host(engine._ctx, bad, len(bad), None, out.ctypes.data,
                                          *(a.ctypes.data for a in arrs), n, ctypes.byref(s)) != 0
    assert not out.any()


def test_tiled_x53_corrupted(engine):
    store = corrupted_x53()
    s = check(engine, store)
    assert s["records"] == 4600 * 53 and s["redundant"] >= 1500 * 51 and s["bad_crc"] > 0 and s["unknown"] > 0


def test_cli_prune(tmp_path):
    src = tmp_path / "gossip_store"
    dst = tmp_path / "pruned"
    store = mutations()["bad_holder_then_redundant"]
    src.write_bytes(store)
    r = subprocess.run([TOOL, "--chain", TESTNET.hex(), "--prune", str(dst), str(src)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert src.read_bytes() == store
    pruned = dst.read_bytes()
    assert len(pruned) == len(store) and pruned != store
    assert "failing message" in r.stdout and "clean" in r.stdout
    r = subprocess.run([TOOL, "--prune", str(src), str(src)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 3 and src.read_bytes() == store
