"""CPU: repairing a gossip_store FILE in place — sv_repair_gossip_store_fd and sv_gossip_prune_cut
(lightning_b200/csrc/gossip_store_fd.c), the verifier subdaemon's sigverifyd_gossip_store_repair (the store's fd passed over
the socket with SCM_RIGHTS) and the drop-in's gossip_store_repair in both modes — built with gcc against the fake prune
(tests/host_emul/fake_engine_prune.c) whose walk stops where gossmap's does on a torn store.  Checked: the cut against a Python statement of
the tail rule on every stop kind; the file ends as the fake's pruned store cut there, with the fake's summary and new_len,
in-process, through a daemon on a socket and through `--fd N`; a client-mode process never creates a context; every
refused file or frame is answered without the daemon exiting, leaves the file as it was and the daemon with no descriptor
more than before; a repair runs on the gossip worker beside channel checks and never beside a prune; the codec of the new
messages."""
import ctypes
import errno
import os
import socket
import struct
import subprocess
import time

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from lightning_b200.engine import SvGossipPruneSummary
from tests import sigverifyd_codec as codec
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.gossip_store import BAD_CRC, EOF, INCOMPLETE, NO_AMOUNT, PARTIAL, ST_ENDED, TRUNCATED
from tests.sigverifyd_fake import (FIELDS, MAX_PRUNE_STORE, PRUNE, TESTNET, back_to, begun, case, cut_rule, fake_prune,
                                   make_store, nfds, prune_frame, run_client, tail_rule, trace, verify_req, wait_trace)


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    return sf.store_bins(tmp_path_factory.mktemp("repair_fake"))


# ---- stores and what the fake makes of them (fake_engine_prune.c) ----------------------------------------------------
def fake_repair(store):
    """(the repaired file, the summary, new_len)"""
    out, s = fake_prune(store)
    cut = cut_rule(out, s)
    return out[:cut], s, cut


def rec(msg, flags=0x2000):
    return struct.pack(">HHII", flags, len(msg), 0, 0) + msg


def torn_stores():
    """name -> store: clean, and each way an append can be torn, plus an ended store and a deleted record past the end"""
    rng = np.random.default_rng(11)
    base = make_store(rng, 40)
    ann = rec(b"\x01\x00" + bytes(200))
    amount = rec(struct.pack(">HQ", 4101, 10))
    upd = rec(b"\x01\x02" + bytes(134))
    out = {"clean": base, "clean_ann_amount": base + ann + amount}
    for k in (1, 5, 12):
        out["torn_header_%d" % k] = base + upd[:k]
    for k in (13, 14, 100, len(upd) - 1):
        out["partial_%d" % k] = base + upd[:k]
    out["incomplete"] = base + rec(b"\x01\x02" + bytes(134), flags=0)
    out["incomplete_then_bytes"] = base + rec(b"\x01\x02" + bytes(134), flags=0) + upd
    for k in (0, 12, 21):
        out["no_amount_%d" % k] = base + ann + amount[:k]
    # a crash between the two writes of the amount's append: the whole amount record, flags 0.  The fake deletes entry 40
    # (the announcement here), so only the announcement at entry 41 is live and must go with the amount record
    out["amount_incomplete"] = base + ann + rec(struct.pack(">HQ", 4101, 10), flags=0)
    out["amount_incomplete_live"] = base + upd + ann + rec(struct.pack(">HQ", 4101, 10), flags=0)
    out["ended"] = base + rec(struct.pack(">HQ", 4105, 7)) + upd[:50]
    out["deleted_past_end"] = base + rec(b"\x01\x02" + bytes(134), flags=0xA000)[:60]
    return out


def repair_frame(rid, length, chain=TESTNET):
    return W.encode("sigverifyd_gossip_store_repair", req_id=rid, has_chain=1 if chain else 0, chain_hash=chain or bytes(32),
                    len=length)


# ---- the cut ---------------------------------------------------------------------------------------------------------
def test_cut_rule(bins):
    """sv_gossip_prune_cut equals the Python statement of the tail rule for every stop kind, with end_offset before, at
    and past the store's length"""
    lib = ctypes.CDLL(bins["inproc"])
    lib.sv_gossip_prune_cut.restype = ctypes.c_uint64
    lib.sv_gossip_prune_cut.argtypes = [ctypes.POINTER(SvGossipPruneSummary), ctypes.c_char_p, ctypes.c_uint64]
    stops = (EOF, 16, 17, 18, 19, INCOMPLETE, PARTIAL, TRUNCATED, BAD_CRC, ST_ENDED, NO_AMOUNT, 0, 1, -1, 99)
    for stop in stops:
        for length in (1, 13, 977, 70001):
            zeros = bytes(length)  # records of type 0: no announcement to back off from
            for end in {0, 1, length - 12, length - 1, length, length + 1, length + 60000}:
                if end < 0:
                    continue
                s = SvGossipPruneSummary(stop=stop, end_offset=end, records=3)
                assert lib.sv_gossip_prune_cut(ctypes.byref(s), zeros, length) == tail_rule(stop, end, length), (stop, end)
    assert lib.sv_gossip_prune_cut(None, b"\0" * 77, 77) == 77 and lib.sv_gossip_prune_cut(ctypes.byref(s), None, 77) == 77
    # the back-off: an announcement the cut leaves with fewer than 22 bytes after it goes, a deleted one stays, and one
    # before it goes too when the same holds for it; a cut of nothing (len) never backs off
    head = make_store(np.random.default_rng(12), 5)
    ann = rec(b"\x01\x00" + bytes(200))
    for tail, flags, want in ((b"", 0x2000, 0), (bytes(21), 0x2000, 0), (bytes(22), 0x2000, None), (b"", 0xA000, None),
                              (rec(b"\x01\x00" + bytes(6)), 0x2000, 0)):
        a = rec(b"\x01\x00" + bytes(200), flags=flags)
        pruned = head + a + tail + bytes(40)
        cut = len(head) + len(a) + len(tail)
        s = SvGossipPruneSummary(stop=INCOMPLETE, end_offset=cut, records=6)
        got = lib.sv_gossip_prune_cut(ctypes.byref(s), pruned, len(pruned))
        assert got == (len(head) if want == 0 else cut) == cut_rule(pruned, {"stop": INCOMPLETE, "end_offset": cut}), tail
    pruned = head + ann + ann + bytes(30)
    s = SvGossipPruneSummary(stop=EOF, end_offset=len(pruned), records=7)
    assert lib.sv_gossip_prune_cut(ctypes.byref(s), pruned[:-30], len(pruned) - 30) == len(pruned) - 30
    # what the cut means on the stores below
    cuts = {k: fake_repair(v)[2] for k, v in torn_stores().items()}
    base = len(torn_stores()["clean"])
    assert cuts["clean"] == base and cuts["clean_ann_amount"] == len(torn_stores()["clean_ann_amount"])
    for k, v in cuts.items():
        if k.startswith(("torn_header", "partial", "incomplete", "no_amount")):
            assert v == base, k
    ts = torn_stores()
    assert cuts["amount_incomplete"] == len(ts["clean"]) + len(ann) and fake_prune(ts["amount_incomplete"])[0][base] & 0x80
    assert cuts["amount_incomplete_live"] == base + len(rec(b"\x01\x02" + bytes(134)))
    assert cuts["ended"] == len(torn_stores()["ended"]) and cuts["deleted_past_end"] == len(torn_stores()["deleted_past_end"])


# ---- the file after a repair -----------------------------------------------------------------------------------------
def test_file_repaired_every_way(tmp_path, bins):
    """in-process, through a daemon on a socket and through `--fd N`: each store's file ends as the fake's pruned store cut
    by the tail rule, with the fake's summary and new_len; a second repair deletes and cuts nothing more"""
    stores = torn_stores()
    names = sorted(stores)
    want = {k: fake_repair(v) for k, v in stores.items()}
    assert all(want[k][1]["pruned"] for k in names)
    d = {}
    for how in ("inproc", "sock", "fd"):
        d[how] = tmp_path / how
        d[how].mkdir()
        for k in names:
            (d[how] / k).write_bytes(stores[k])
    cases = lambda how: [c for k in names for c in (case(d[how] / k, op="repair"),
                                                    case(d[how] / k, want[k][2], op="repair"))]
    got = {"inproc": run_client(tmp_path, bins["inproc"], "inproc", cases("inproc"))}
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        got["sock"] = run_client(tmp_path, bins["client"], "sock:" + sock, cases("sock"))
        assert sock.proc.poll() is None
    parent, child = socket.socketpair()
    dm = subprocess.Popen([bins["daemon"], "--fd", str(child.fileno()), "0"], pass_fds=(child.fileno(),), env=sf.env(tmp_path),
                          stderr=subprocess.PIPE)
    child.close()
    try:
        got["fd"] = run_client(tmp_path, bins["client"], "fd:%d" % parent.fileno(), cases("fd"), pass_fds=(parent.fileno(),))
        parent.close()
        assert dm.wait(timeout=30) == 0
    finally:
        if dm.poll() is None:
            dm.kill()
            dm.wait(timeout=10)
    for how in got:
        for i, k in enumerate(names):
            out, s, cut = want[k]
            assert (d[how] / k).read_bytes() == out, (how, k)
            first, second = got[how][2 * i], got[how][2 * i + 1]
            assert first == [True, 0, s, cut], (how, k)
            assert second[:2] == [True, 0] and second[3] == cut and second[2]["pruned"] == 0, (how, k)


def test_clean_store_repair_is_the_prune(tmp_path, bins):
    """on a store without a torn tail (clean or ended) the repair leaves the file exactly as the prune does"""
    for name in ("clean", "clean_ann_amount", "ended", "deleted_past_end"):
        st = torn_stores()[name]
        a, b = tmp_path / (name + ".p"), tmp_path / (name + ".r")
        a.write_bytes(st)
        b.write_bytes(st)
        p, r = run_client(tmp_path, bins["inproc"], "inproc", [case(a), case(b, op="repair")])
        assert a.read_bytes() == b.read_bytes() and p[2] == r[2] and r[3] == len(st), name


def test_client_mode_never_creates_a_context(tmp_path, bins):
    f = tmp_path / "gossip_store"
    f.write_bytes(torn_stores()["partial_100"])
    r = run_client(tmp_path, bins["client"], "inproc", [case(f, op="repair")], check=False)
    assert r.returncode != 0 and "sv_create called" in r.stderr


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refused_files(tmp_path, bins):
    """a read-only fd (EBADF), a pipe (EINVAL), a length past the end of the file (EINVAL), a store the engine refuses
    (EINVAL), a store above the daemon's cap (EFBIG, never reaching the engine) and a closed descriptor (EBADF, nothing
    sent): false with that errno, in-process and through the daemon; no file changes or shrinks, and the daemon stays up
    with its descriptor count back where it was"""
    store = torn_stores()["partial_100"]
    ro, short, v1, good = (tmp_path / x for x in ("ro", "short", "v1", "good"))
    for f in (ro, short, good):
        f.write_bytes(store)
    v1.write_bytes(bytes([0x20]) + store[1:])
    big = tmp_path / "big"
    with open(big, "wb") as fh:
        fh.truncate(MAX_PRUNE_STORE + 4096)
    cases = [case(ro, kind="ro", op="repair"), case("", 64, None, kind="pipe", op="repair"),
             case(short, len(store) + 1, op="repair"), case(v1, op="repair"), case(big, op="repair"),
             case("", 10, None, kind="closed", op="repair"), case(short, 0, op="repair"), case(good, op="repair")]
    want_err = [errno.EBADF, errno.EINVAL, errno.EINVAL, errno.EINVAL, errno.EFBIG, errno.EBADF, errno.EINVAL]
    before = {f: f.read_bytes() for f in (ro, short, v1)}
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        got = run_client(tmp_path, bins["client"], "sock:" + sock, cases)
        assert sock.proc.poll() is None
        assert back_to(sock.proc, base) == base
    assert [g[:2] for g in got[:-1]] == [[False, e] for e in want_err]
    out, s, cut = fake_repair(store)
    assert got[-1] == [True, 0, s, cut] and good.read_bytes() == out and cut < len(store)
    for f, b in before.items():
        assert f.read_bytes() == b, f
    assert os.path.getsize(big) == MAX_PRUNE_STORE + 4096
    assert [c[3] for c in sf.calls(tmp_path / "engine.log") if c[0] == PRUNE] == [len(store)]
    good.write_bytes(store)
    local = run_client(tmp_path, bins["inproc"], "inproc", cases[:4] + cases[5:])
    assert [g[:2] for g in local[:-1]] == [[False, e] for e in want_err[:4] + want_err[5:]]
    assert local[-1] == got[-1]
    for f, b in before.items():
        assert f.read_bytes() == b, f


def test_refused_frames(tmp_path, bins):
    """a repair frame without an fd is answered sigverifyd_error and the connection keeps serving; a repair frame with one
    is answered sigverifyd_gossip_store_repair_reply"""
    rng = np.random.default_rng(5)
    f = tmp_path / "gossip_store"
    store = torn_stores()["incomplete"]
    f.write_bytes(store)
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        c.settimeout(30)
        c.connect(sock)
        c.sendall(repair_frame(1, len(store)))
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=1, code=1))
        vf, vw = verify_req(rng, 2, 0, 2)
        c.sendall(vf)
        assert W.read_msg(c) == vw
        assert f.read_bytes() == store
        fd = os.open(f, os.O_RDWR)
        try:
            socket.send_fds(c, [repair_frame(3, len(store))], [fd])
        finally:
            os.close(fd)
        name, m = W.read_msg(c)
        out, s, cut = fake_repair(store)
        assert name == "sigverifyd_gossip_store_repair_reply" and m["req_id"] == 3 and m["err"] == 0
        assert {k: m[k] for k in FIELDS} == s and m["new_len"] == cut
        c.close()
        assert back_to(sock.proc, base) == base
    assert f.read_bytes() == out


def test_repair_beside_channel_checks_never_beside_a_prune(tmp_path, bins):
    """a repair held 600 ms on the fake: another client's verify request is answered while it runs, and another client's
    prune begins only after it ends; both files end as they should"""
    rng = np.random.default_rng(6)
    stores = [torn_stores()["partial_100"], make_store(rng, 45)]
    files = [tmp_path / "a", tmp_path / "b"]
    for f, s in zip(files, stores):
        f.write_bytes(s)
    fds = [os.open(f, os.O_RDWR) for f in files]
    try:
        with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path, {PRUNE: 600})) as sock:
            a, b, v = (socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) for _ in range(3))
            for c in (a, b, v):
                c.settimeout(30)
                c.connect(sock)
            socket.send_fds(a, [repair_frame(1, len(stores[0]))], [fds[0]])
            wait_trace(tmp_path, begun(PRUNE))
            socket.send_fds(b, [prune_frame(2, len(stores[1]))], [fds[1]])
            for k in range(3):
                f, want = verify_req(rng, 10 + k, 0, 3)
                v.sendall(f)
                assert W.read_msg(v) == want
            assert not any(e[:2] == ("end", PRUNE) for e in trace(tmp_path))
            name, m = W.read_msg(a)
            assert name == "sigverifyd_gossip_store_repair_reply" and m["err"] == 0 and m["new_len"] == fake_repair(stores[0])[2]
            name, m = W.read_msg(b)
            assert name == "sigverifyd_gossip_store_prune_reply" and m["err"] == 0
            for c in (a, b, v):
                c.close()
    finally:
        for fd in fds:
            os.close(fd)
    assert [e[0] for e in trace(tmp_path) if e[1] == PRUNE] == ["begin", "end", "begin", "end"]
    assert files[0].read_bytes() == fake_repair(stores[0])[0]
    assert files[1].read_bytes() == fake_prune(stores[1])[0]


# ---- the codec -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return codec.build_shim(tmp_path_factory.mktemp("wire"))


def test_codec_round_trip(shim):
    """the C codec (sigverifyd_wiregen.h) and the Python one (sigverifyd_wire.py) give the same bytes for both messages and
    read each other's; a short or long message, or another type, is refused (tests/sigverifyd_codec.py)"""
    rng = np.random.default_rng(8)
    for _ in range(50):
        rid, has, ln = int(rng.integers(0, 2**63)), int(rng.integers(0, 2)), int(rng.integers(0, 2**64, dtype=np.uint64))
        chain = rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()
        req = dict(req_id=rid, has_chain=has, chain_hash=chain, len=ln)
        vals = [rid, int(rng.integers(0, 2**32)), int(rng.integers(0, 2**32)), int(rng.integers(0, 2**32))] + [
            int(x) for x in rng.integers(0, 2**64, size=13, dtype=np.uint64)]
        rep = dict(zip(["req_id", "err"] + FIELDS + ["new_len"], vals))
        for name, m in (("sigverifyd_gossip_store_repair", req), ("sigverifyd_gossip_store_repair_reply", rep)):
            codec.agree(shim, name, m)
            codec.refused(shim, name, m)
            codec.wrong_type_refused(shim, name, m)
