"""GPU: repairing a torn gossip_store in place (sv_repair_gossip_store_fd), checked against Core Lightning's own gossmap.c.

A store ends in a new channel's channel_announcement, channel_amount, channel_update and node_announcement, as gossipd
appends them.  Its torn versions are what a crash during those appends leaves: the file cut at every byte offset inside the
four records, the last record with GOSSIP_STORE_COMPLETED_BIT cleared, and the whole channel_amount record with flags 0
(gossipd writes a record with flags 0 and sets COMPLETED in a second write: a crash between the two).  The same tears are made on the fixture tiled
x53 with 1 % of its records corrupted (tests/test_gpu_gossip_store_prune.py), at the edges and inside of each record (the
x53 store is 51 MB, so not at every byte).  For each torn store T with cut = sv_gossip_prune_cut of its prune:
  - the repaired file is byte for byte prune(T)[:cut] (prune = SigVerifier.prune_gossip_store on the same bytes), and
    also prune(untorn store[:cut]): the torn tail changes nothing before the cut;
  - cut is where the rule puts it (tests/sigverifyd_fake.py cut_rule), and the record boundary the tear
    lies behind;
  - CLN's strict load (oracle/gossmap_strict_harness.c, expected_len = the new length) accepts the repaired file, and its
    channel table equals that of CLN's lenient load (oracle/gossmap_harness.c) of prune(T) uncut, which stops at the cut:
    the repair keeps exactly what gossmap would have loaded.  The one exception is the incomplete amount record: the
    lenient load stops at it but reads its bytes for the announcement before it, so it holds that one channel more;
  - the strict load's nodes are the endpoints of its channels, and each node's current node_announcement is a live
    node_announcement of the repaired file for that node (or none).
Each torn store goes through SigVerifier.repair_gossip_store_fd, through the drop-in's gossip_store_repair in client mode
through a real cln_sigverifyd (the fd passed over the socket), and through `cln_verify_gossip_store --prune OUT --cut-tail`
(on a subset of the tears of the small store).  A store whose walk ends at a gossip_store_ended record, and the untorn
stores, come out of every path exactly as sv_prune_gossip_store_fd leaves them.  CLN's answers are recorded under
tests/golden/oracle/ (tests/oracle_replay.py)."""
import ctypes
import hashlib
import os
import struct
import subprocess

import pytest

from lightning_b200 import build
from tests import ecc
from tests import gossip_store as gs
from tests import oracle_replay, sigverifyd_daemon
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_prune_host import strict_load
from tests.test_gossmap import gossmap_load
from tests.test_gpu_gossip_burst import PUB, SK, TESTNET, _ordered, _sha256d, make_ca, make_cu
from tests.test_gpu_gossip_store import TOOL
from tests.test_gpu_gossip_store_prune import corrupted_x53
from tests.sigverifyd_fake import case, cut_rule, run_client

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRICT = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap_strict.so")
LENIENT = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap.so")
SCID = b"\x00\x0f\x42\x40\x00\x07\x00\x01"


class _All:
    """CLN's libraries behind one recorded oracle (one tape per test module)"""

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
        libs = [ctypes.CDLL(p) for p in (STRICT, LENIENT) if os.path.exists(p)]
        if o.lib is not None and libs:
            o.lib = _All(o.lib, *libs)
            o.lib.cln_gossmap_load.restype = ctypes.c_longlong
        _O.append(o)
    return _O[0]


# ---- the stores ------------------------------------------------------------------------------------------------------
def make_na(node, ts=1):
    """a signed node_announcement of `node` with no features and no addresses"""
    tail = b"\x00\x00" + ts.to_bytes(4, "big") + PUB[node] + b"\x01\x02\x03" + node.encode().ljust(32, b"\0") + b"\x00\x00"
    return b"\x01\x01" + ecc.ecdsa_sign(SK[node], _sha256d(tail)) + tail


def last_four():
    """a new channel as gossipd appends it: channel_announcement, channel_amount, channel_update, node_announcement"""
    a, b = _ordered("a", "b")
    return [gs.record(make_ca(SCID, a, b)), gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 100000)),
            gs.record(make_cu(SCID, a, 0)), gs.record(make_na(a))]


def _prefix():
    """the fixture's records before its first channel_announcement past record 60"""
    fx = load_fixture()
    recs = gs.walk(fx)[0]
    n = next(i for i in range(60, len(recs)) if recs[i][1] == 256)
    return fx[:recs[n][0]]


_BASES = {}


def base(name):
    """(the untorn store, the offsets of its last four records)"""
    if name not in _BASES:
        head = _prefix() if name == "small" else corrupted_x53()
        four = last_four()
        offs = [len(head) + sum(len(r) for r in four[:k]) for k in range(4)]
        _BASES[name] = (head + b"".join(four), offs)
    return _BASES[name]


def boundary_cut(offs, end, t):
    """where a store torn at byte t must end: at the last record boundary it keeps, and never inside the announcement and
    its amount record (gossmap ignores an announcement whose amount record does not fit)"""
    ca, am, cu, na = offs
    if t in (cu, na, end):
        return t
    return ca if t < cu else cu if t < na else na


_TEARS = {}


def tears(name):
    """tear -> the cut it must get"""
    if name in _TEARS:
        return _TEARS[name]
    store, offs = base(name)
    end = len(store)
    if name == "small":
        cuts = range(offs[0] + 1, end)
    else:
        ends = offs[1:] + [end]
        cuts = sorted({t for o, e in zip(offs, ends) for t in (o + 1, o + 12, o + 13, (o + e) // 2, e - 1)})
    out = {"at_%d" % t: boundary_cut(offs, end, t) for t in cuts}
    out["last_incomplete"] = offs[3]
    out["amount_incomplete"] = offs[0]  # the announcement goes with its incomplete amount record
    _TEARS[name] = out
    return out


def torn(name, k):
    """the torn store of tear k"""
    store, offs = base(name)
    if k == "last_incomplete":
        inc = bytearray(store)
        inc[offs[3]] &= ~(gs.COMPLETED >> 8) & 0xFF
        return bytes(inc)
    if k == "amount_incomplete":
        return store[:offs[1]] + b"\0\0" + store[offs[1] + 2:offs[2]]
    return store[:int(k[3:])]


def cli_subset(name):
    """the tears the command-line tool repairs: every record's first, 12th, 13th and last byte, and the incomplete one"""
    if name != "small":
        return sorted(tears(name))
    store, offs = base(name)
    ends = offs[1:] + [len(store)]
    return ["at_%d" % t for o, e in zip(offs, ends) for t in (o + 1, o + 12, o + 13, e - 1)] + ["last_incomplete",
                                                                                              "amount_incomplete"]


def ended_store():
    """the small store's head, a gossip_store_ended record, and bytes after it (a replaced store: not repaired)"""
    store, offs = base("small")
    return store[:offs[0]] + gs.record(struct.pack(">HQ", gs.ENDED, offs[0])) + store[offs[0]:offs[2] + 40]


class Expected:
    """prune(T) and its summary for every tear, from the host-buffer call.  prune(T) is kept as its part before the cut,
    shared by the tears with the same one, and its own tail: the x53 tears would not fit in memory whole."""

    def __init__(self, engine):
        self.heads, self.tears = {}, {}
        for name in ("small", "x53"):
            for k, cut in tears(name).items():
                pruned, _, s = engine.prune_gossip_store(torn(name, k), TESTNET)
                h = _digest(pruned[:cut])
                self.heads.setdefault(h, pruned[:cut])
                self.tears[name, k] = (s, cut, h, pruned[cut:])

    def __call__(self, name, k):
        """(torn store, prune(T), its summary, cut)"""
        s, cut, h, tail = self.tears[name, k]
        return torn(name, k), self.heads[h] + tail, s, cut


@pytest.fixture(scope="module")
def expected(engine):
    return Expected(engine)


def _digest(b):
    return hashlib.sha256(b).digest()


def _msg(store, off):
    """the message at message offset off"""
    return store[off:off + struct.unpack(">H", store[off - 10:off - 8])[0]]


def check_nodes(store, chans, nodes):
    """gossmap's nodes are the endpoints of its channels; each current node_announcement is a live one of that node"""
    ends = {n for _, cann, _, _ in chans for n in gs.ann_fields(_msg(store, cann))[2:4]}
    assert len(nodes) == len(ends)
    live = {off + gs.HDR for off, t, _, st in gs.walk(store)[0] if t == 257 and st == 0}
    for n in nodes:
        if n:
            m = _msg(store, n)
            flen = struct.unpack(">H", m[66:68])[0]
            assert n in live and m[72 + flen:105 + flen] in ends
    assert len([n for n in nodes if n]) == len({n for n in nodes if n})


# ---- in-process, against gossmap -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "x53"])
def test_repair_in_process_against_gossmap(engine, expected, tmp_path, name):
    o = oracle()
    store, offs = base(name)
    _, _, s0 = engine.prune_gossip_store(store, TESTNET)
    assert s0["stop"] == gs.EOF and s0["end_offset"] == len(store)
    assert name != "small" or s0["pruned"] == 0
    untorn, strict = {}, {}
    f = tmp_path / "gossip_store"
    for k in tears(name):
        t, pruned, s, cut = expected(name, k)
        assert cut == cut_rule(pruned, s) == engine.gossip_prune_cut(s, pruned), k
        f.write_bytes(t)
        fd = os.open(f, os.O_RDWR)
        try:
            rs, new_len = engine.repair_gossip_store_fd(fd, len(t), TESTNET)
        finally:
            os.close(fd)
        repaired = f.read_bytes()
        assert (rs, new_len) == (s, cut), k
        assert repaired == pruned[:cut], k
        if cut not in untorn:
            untorn[cut] = engine.prune_gossip_store(store[:cut], TESTNET)[0]
        assert repaired == untorn[cut], k
        if cut == len(t):
            assert repaired == pruned, k
            continue
        # gossmap: the strict load accepts the repaired file, and holds what the lenient load of prune(T) holds
        if _digest(repaired) not in strict:
            ref = strict_load(o, repaired)
            assert ref is not None, (k, "gossmap's strict load refused the repaired store")
            strict[_digest(repaired)] = ref
        end, chans, nodes = strict[_digest(repaired)]
        assert end == cut, k
        check_nodes(repaired, chans, nodes)
        lenient = gossmap_load(o, pruned)
        assert lenient is not None, k
        if k == "amount_incomplete":  # the lenient load keeps the announcement, reading the incomplete amount's bytes
            assert s["stop"] == gs.INCOMPLETE and s["end_offset"] == offs[1]
            assert lenient[0] == offs[1] and [r for r in lenient[1] if r[1] != offs[0] + gs.HDR] == chans
            assert len(lenient[1]) == len(chans) + 1
            continue
        assert lenient == (cut, chans), k
    assert len(untorn) == 3  # every record boundary a tear can fall back to: before the announcement, update, node_announcement


# ---- through the verifier subdaemon, and the command-line tool -------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "x53"])
def test_repair_through_the_daemon(expected, tmp_path, name):
    """the drop-in's gossip_store_repair in client mode through cln_sigverifyd: each file ends as prune(T)[:cut], with
    the summary and new_len of the host call"""
    tests = sorted(tears(name))
    batch = len(tests) if name == "small" else 1  # the x53 tears one file at a time
    d = tmp_path / "stores"
    d.mkdir()
    with sigverifyd_daemon.running(tmp_path) as sock:
        for i in range(0, len(tests), batch):
            part = tests[i:i + batch]
            for k in part:
                (d / k).write_bytes(torn(name, k))
            got = run_client(tmp_path, build.LIB, "sock:" + sock, [case(d / k, op="repair") for k in part])
            for k, g in zip(part, got):
                t, pruned, s, cut = expected(name, k)
                assert g == [True, 0, s, cut], k
                assert (d / k).read_bytes() == pruned[:cut], k
                if name != "small":
                    (d / k).unlink()


@pytest.mark.parametrize("name", ["small", "x53"])
def test_repair_cli(expected, tmp_path, name):
    """cln_verify_gossip_store --prune OUT --cut-tail FILE writes prune(T)[:cut] and finds it clean"""
    src, dst = tmp_path / "gossip_store", tmp_path / "repaired"
    for k in cli_subset(name):
        t, pruned, s, cut = expected(name, k)
        src.write_bytes(t)
        r = subprocess.run([TOOL, "--chain", TESTNET.hex(), "--prune", str(dst), "--cut-tail", str(src)], capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, (k, r.stdout[-2000:], r.stderr[-2000:])
        assert src.read_bytes() == t, k
        assert dst.read_bytes() == pruned[:cut], k
        assert ("torn tail: %d bytes cut" % (len(t) - cut)) in r.stdout and "clean" in r.stdout, k


def test_ended_and_untorn_stores_are_only_pruned(engine, tmp_path):
    """a store whose walk stops at gossip_store_ended, the untorn stores, and the x53 store: every path leaves the file as
    sv_prune_gossip_store_fd does, with new_len its length"""
    stores = {"ended": ended_store(), "small": base("small")[0], "x53": base("x53")[0]}
    for k, st in stores.items():
        a, b = tmp_path / (k + ".prune"), tmp_path / (k + ".repair")
        a.write_bytes(st)
        b.write_bytes(st)
        fa, fb = os.open(a, os.O_RDWR), os.open(b, os.O_RDWR)
        try:
            sp = engine.prune_gossip_store_fd(fa, len(st), TESTNET)
            sr, new_len = engine.repair_gossip_store_fd(fb, len(st), TESTNET)
        finally:
            os.close(fa)
            os.close(fb)
        assert sr == sp and new_len == len(st), k
        assert b.read_bytes() == a.read_bytes(), k
        if k == "ended":
            assert sp["stop"] == gs.ST_ENDED and sp["end_offset"] < len(st)
        b.write_bytes(st)
        with sigverifyd_daemon.running(tmp_path) as sock:
            got = run_client(tmp_path, build.LIB, "sock:" + sock, [case(b, op="repair")])
        assert got == [[True, 0, sp, len(st)]] and b.read_bytes() == a.read_bytes(), k
        dst = tmp_path / (k + ".cli")
        r = subprocess.run([TOOL, "--chain", TESTNET.hex(), "--prune", str(dst), "--cut-tail", str(b)], capture_output=True,
                           text=True, timeout=300)
        assert dst.read_bytes() == engine.prune_gossip_store(st, TESTNET)[0], k
        assert "torn tail: 0 bytes cut" in r.stdout and r.returncode == (1 if k == "ended" else 0), (k, r.stdout[-2000:])
        for p in (a, b, dst):
            p.unlink()
