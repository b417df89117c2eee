"""GPU: salvaging a gossip_store past damaged record headers (sv_salvage_gossip_store_host, sv_salvage_gossip_store_fd),
on the fixture and on the fixture tiled x53 (each with a gossip_store_uuid record first and one record deleted as gossipd
deletes), for every damage class of tests/test_gossip_store_salvage_host.py: a length bit flipped in the high and in the
low byte, COMPLETED cleared, a header zeroed, 100 KB zeroed, two separate breaks, the first record's length, a deleted
record's length, and damage inside the last record.  For each:
  - the written bytes, the action list and the salvage summary are the model's (tests/gossip_store_salvage.py);
  - the file salvaged in place is byte for byte the file the repair (sv_repair_gossip_store_fd) makes of the model's
    salvage, with the same prune summary and new length, and gossmap's strict load (oracle/gossmap_strict_harness.c,
    expected_len = that length) accepts it;
  - every record outside the damaged bytes keeps the prune status and reason it has in the undamaged store, except an
    update or a later announcement of a channel whose holding announcement was damaged;
  - damage inside the last record is repaired exactly as the repair alone repairs it.
Each of the nine single header flips of the table in INTEGRATION.md §4b is restored and every one of the fixture's 4,600
records kept.  Stores without a break come out of the salvage unchanged, and out of the salvage and repair exactly as
out of the repair; a salvaged store salvages to itself.  The drop-in's gossip_store_salvage, in-process and in client
mode through a real cln_sigverifyd (the fd passed over the socket), leaves every file, summary and new length exactly as
SigVerifier.salvage_gossip_store_fd does.  `cln_verify_gossip_store --prune OUT --salvage` writes what the in-place call
leaves.  CLN's answers are recorded under tests/golden/oracle/ (tests/oracle_replay.py)."""
import os
import subprocess

import pytest

from lightning_b200 import build
from tests import gossip_store as gs
from tests import gossip_store_salvage as sv
from tests import sigverifyd_daemon
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_prune_host import oracle, strict_load
from tests.test_gossip_store_salvage_host import damage_classes, header_flips, kept_changes, with_uuid, x53
from tests.test_gpu_gossip_burst import TESTNET
from tests.test_gpu_gossip_store import TOOL
from tests.test_sigverifyd_salvage_fake import case, run_client

pytestmark = pytest.mark.gpu

_BASES = {}


def base(name):
    if name not in _BASES:
        _BASES[name] = with_uuid(load_fixture() if name == "fixture" else x53())
    return _BASES[name]


_CLASSES = {}


def classes(name):
    if name not in _CLASSES:
        _CLASSES[name] = damage_classes(base(name))
    return _CLASSES[name]


def in_file(tmp_path, data, fn, *args):
    """fn(fd, len(data), *args) on a file holding data -> (its result, the file's bytes after)"""
    f = tmp_path / "gossip_store"
    f.write_bytes(data)
    fd = os.open(f, os.O_RDWR)
    try:
        r = fn(fd, len(data), *args)
    finally:
        os.close(fd)
    out = f.read_bytes()
    f.unlink()
    return r, out


def rows(engine, store):
    off, typ, status, why = engine.prune_gossip_store(store, TESTNET)[1]
    return [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(off, typ, status, why)]


@pytest.mark.parametrize("name", ["fixture", "x53"])
def test_damage_classes(engine, tmp_path, name):
    o = oracle()
    b = base(name)
    want_rows = rows(engine, b)
    for k, (st, span) in classes(name).items():
        model = sv.salvage(st)
        got = engine.salvage_gossip_store(st)
        assert got == model, k
        out, acts, vs = got
        if not k.startswith("last_"):
            assert vs["breaks"] >= 1, k
        # in place: the salvage, then exactly the repair of the salvaged bytes
        (ps, v2, new_len), f = in_file(tmp_path, st, engine.salvage_gossip_store_fd, TESTNET)
        (ps_r, new_len_r), f_r = in_file(tmp_path, out, engine.repair_gossip_store_fd, TESTNET)
        assert (ps, v2, new_len) == (ps_r, vs, new_len_r) and f == f_r and len(f) == new_len, k
        ref = strict_load(o, f)
        assert ref is not None and ref[0] == new_len, (k, "gossmap's strict load refused the salvaged store")
        kept_changes(b, span, want_rows, rows(engine, out))
        if k.startswith("last_"):
            assert acts == [], k
            assert in_file(tmp_path, st, engine.repair_gossip_store_fd, TESTNET) == ((ps, new_len), f), k
        # a salvaged store salvages to itself
        again = engine.salvage_gossip_store(out)
        assert again[0] == out and again[1] == [], k


def test_header_flips_keep_every_record(engine, tmp_path):
    """the nine single header flips of the fixture: each damaged record restored, the store the fixture again, and the
    repair keeps all 4,600 records"""
    fx = load_fixture()
    recs = gs.walk(fx)[0]
    for k, (st, i) in header_flips(fx).items():
        out, acts, vs = engine.salvage_gossip_store(st)
        assert out == fx and acts == [(recs[i][0], recs[i + 1][0], sv.RESTORED)], k
        (ps, _, new_len), f = in_file(tmp_path, st, engine.salvage_gossip_store_fd, TESTNET)
        assert f == fx and new_len == len(fx) and ps["records"] == 4600 and ps["pruned"] == 0, k
        # without the salvage the repair cuts the records after the damaged one
        (pr, cut), _ = in_file(tmp_path, st, engine.repair_gossip_store_fd, TESTNET)
        assert cut < len(fx), k


def test_no_break_is_the_repair(engine, tmp_path):
    """stores without a break (clean, torn tails, a store ended by gossip_store_ended, the prune's mid-store cases): the
    salvage writes nothing, and the salvage and repair leave the file exactly as the repair alone"""
    fx = base("fixture")
    recs = gs.walk(fx)[0]
    mid = recs[2300][0]
    stores = {"clean": fx, "x53": base("x53"),
              "truncated_mid": fx[:mid] + gs.record(b"\x01") + fx[mid:],
              "unknown_mid": fx[:mid] + gs.record(b"\x13\x87\x00\x00") + fx[mid:],
              "ended": fx[:mid] + gs.record(b"\x10\x09" + mid.to_bytes(8, "big")) + fx[mid:mid + 3000]}
    for t in (recs[-3][0] + 5, recs[-2][0] + 12, recs[-1][0] + 13, len(fx) - 1):
        stores["torn_%d" % t] = fx[:t]
    inc = bytearray(fx)
    inc[recs[-1][0]] &= 0xDF
    stores["last_incomplete"] = bytes(inc)
    for k, st in stores.items():
        out, acts, vs = engine.salvage_gossip_store(st)
        assert out == st and acts == [] and vs["breaks"] == 0, k
        assert vs["sound"] == len(sv.sound_offsets(st)), k
        (ps, _, new_len), f = in_file(tmp_path, st, engine.salvage_gossip_store_fd, TESTNET)
        assert in_file(tmp_path, st, engine.repair_gossip_store_fd, TESTNET) == ((ps, new_len), f), k


def test_many_breaks_and_capacity(engine):
    """a store with a break every 50 records, listed whole however small the first room for actions"""
    st = bytearray(base("fixture"))
    recs = gs.walk(bytes(st))[0]
    for i in range(1, len(recs) - 1, 50):
        st[recs[i][0] + 2] ^= 0x02
    st = bytes(st)
    model = sv.salvage(st)
    assert len(model[1]) == len(range(1, len(recs) - 1, 50))
    assert engine.salvage_gossip_store(st, capacity=1) == engine.salvage_gossip_store(st) == model


def test_profiling(engine):
    engine.set_profiling(True)
    try:
        engine.salvage_gossip_store(classes("x53")["zeroed_100k"][0])
        f, c, w = engine.last_gossip_salvage_timing()
        assert f > 0 and c > 0 and w >= 0
    finally:
        engine.set_profiling(False)


def test_cli(engine, tmp_path):
    """--prune OUT --salvage writes the in-place result, names each break and finds OUT clean"""
    src, dst = tmp_path / "src", tmp_path / "out"
    for k in ("len_hi", "zeroed_100k", "two_breaks", "last_length"):
        st = classes("fixture")[k][0]
        out, acts, _ = engine.salvage_gossip_store(st)
        (_, _, new_len), f = in_file(tmp_path, st, engine.salvage_gossip_store_fd, TESTNET)
        src.write_bytes(st)
        r = subprocess.run([TOOL, "--chain", TESTNET.hex(), "--prune", str(dst), "--salvage", str(src)], capture_output=True,
                           text=True, timeout=300)
        assert r.returncode == 0, (k, r.stdout[-2000:], r.stderr[-2000:])
        assert src.read_bytes() == st and dst.read_bytes() == f, k
        for t, q, kind in acts:
            what = "header restored" if kind == sv.RESTORED else "span bridged with deleted fillers"
            assert "break @%d: records resume at %d, %s" % (t, q, what) in r.stdout, k
        assert ("%d breaks" % len(acts)) in r.stdout and "clean" in r.stdout, k


@pytest.mark.parametrize("name", ["fixture", "x53"])
def test_drop_in_and_daemon_agree(engine, tmp_path, name):
    """gossip_store_salvage in-process and through cln_sigverifyd gives the file, both summaries and the new length of
    SigVerifier.salvage_gossip_store_fd (x53: the two single-record classes and the multi-filler bridge)"""
    ks = sorted(classes(name)) if name == "fixture" else ["len_hi", "zeroed_100k"]
    want = {k: in_file(tmp_path, classes(name)[k][0], engine.salvage_gossip_store_fd, TESTNET) for k in ks}
    d = tmp_path / "stores"
    d.mkdir()
    for mode in ("inproc", "daemon"):
        for k in ks:
            (d / k).write_bytes(classes(name)[k][0])
        if mode == "inproc":
            got = run_client(tmp_path, build.LIB, "inproc", [case(d / k) for k in ks])
        else:
            with sigverifyd_daemon.running(tmp_path) as sock:
                got = run_client(tmp_path, build.LIB, "sock:" + sock, [case(d / k) for k in ks])
        for k, g in zip(ks, got):
            (ps, vs, new_len), f = want[k]
            assert g == [True, 0, ps, vs, new_len], (mode, k)
            assert (d / k).read_bytes() == f, (mode, k)
