"""CPU: salvaging a gossip_store FILE through the drop-in's gossip_store_salvage in both modes and through the verifier
subdaemon's sigverifyd_gossip_store_salvage (the store's fd passed over the socket with SCM_RIGHTS), built with gcc against
the CPU salvage of tests/host_emul/fake_engine_salvage.cpp (gossip_salvage.cuh's rule, every offset checked on the host)
and the fake prune of tests/host_emul/fake_engine_prune.c, with lightning_b200/csrc/gossip_salvage_fd.c and
gossip_store_fd.c as the library has them.  Checked: the file ends as the fake repair of the model's salvage
(tests/gossip_store_salvage.py), with the fake's summary, the model's salvage summary and the repair's new length,
in-process, through a daemon on a socket and through `--fd N`; a second call mends nothing; a client-mode process never
creates a context; every refused file or frame is answered without the daemon exiting and leaves the file as it was; a
salvage runs on the gossip worker beside channel checks and never beside a prune; the reply's codec."""
import errno
import os
import socket
import subprocess
import time

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import gossip_store_salvage as sv
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.gossip_store import load_fixture
from tests.gossip_store_salvage import damage_classes, with_uuid
from tests.sigverifyd_fake import (FIELDS, MAX_PRUNE_STORE, PRUNE, TESTNET, back_to, begun, cut_rule, fake_prune, make_store,
                                   nfds, prune_frame, run_client, trace, verify_req, wait_trace)
from tests.sigverifyd_fake import salvage_case as case


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    return sf.store_bins(tmp_path_factory.mktemp("salvage_fake"), salvage=True)


def salvage_frame(rid, length, chain=TESTNET):
    return W.encode("sigverifyd_gossip_store_salvage", req_id=rid, has_chain=1 if chain else 0,
                    chain_hash=chain or bytes(32), len=length)


def fake_salvage(store):
    """(the file after the salvage and the fake repair, the repair summary, the salvage summary, new_len)"""
    out, _, v = sv.salvage(store)
    pruned, s = fake_prune(out)
    cut = cut_rule(pruned, s)
    return pruned[:cut], s, v, cut


_STORES = {}


def stores():
    """a clean store, a restored header, a span bridged by several fillers, two breaks"""
    if not _STORES:
        base = with_uuid(load_fixture())
        cls = damage_classes(base)
        _STORES.update(clean=base, len_hi=cls["len_hi"][0], zeroed_100k=cls["zeroed_100k"][0],
                       two_breaks=cls["two_breaks"][0])
    return _STORES


# ---- the file after a salvage ----------------------------------------------------------------------------------------
def test_file_salvaged_every_way(tmp_path, bins):
    """in-process, through a daemon on a socket and through `--fd N`: each file ends as the fake repair of the model's
    salvage, with the fake's summary, the model's salvage summary and the cut; a second call mends nothing"""
    st = stores()
    names = sorted(st)
    want = {k: fake_salvage(v) for k, v in st.items()}
    assert all(want[k][2]["breaks"] for k in names if k != "clean") and want["zeroed_100k"][2]["fillers"] > 1
    d = {}
    for how in ("inproc", "sock", "fd"):
        d[how] = tmp_path / how
        d[how].mkdir()
        for k in names:
            (d[how] / k).write_bytes(st[k])
    cases = lambda how: [c for k in names for c in (case(d[how] / k), case(d[how] / k, want[k][3]))]
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
            out, s, v, cut = want[k]
            assert (d[how] / k).read_bytes() == out, (how, k)
            first, second = got[how][2 * i], got[how][2 * i + 1]
            assert first == [True, 0, s, v, cut], (how, k)
            assert second[:2] == [True, 0] and second[3]["breaks"] == 0 and second[4] == cut, (how, k)


def test_client_mode_never_creates_a_context(tmp_path, bins):
    f = tmp_path / "gossip_store"
    f.write_bytes(stores()["len_hi"])
    r = run_client(tmp_path, bins["client"], "inproc", [case(f)], check=False)
    assert r.returncode != 0 and "sv_create called" in r.stderr


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refused_files(tmp_path, bins):
    """a read-only fd (EBADF), a pipe (EINVAL), a length past the end of the file (EINVAL), a store the engine refuses
    (EINVAL), a store above the daemon's cap (EFBIG, never reaching the engine), a closed descriptor (EBADF, nothing sent)
    and a length of 0 (EINVAL): false with that errno, in-process and through the daemon; no file changes or shrinks, and
    the daemon stays up with its descriptor count back where it was"""
    store = stores()["len_hi"]
    ro, short, v1, good = (tmp_path / x for x in ("ro", "short", "v1", "good"))
    for f in (ro, short, good):
        f.write_bytes(store)
    v1.write_bytes(bytes([0x20]) + store[1:])
    big = tmp_path / "big"
    with open(big, "wb") as fh:
        fh.truncate(MAX_PRUNE_STORE + 4096)
    cases = [case(ro, kind="ro"), case("", 64, None, kind="pipe"), case(short, len(store) + 1), case(v1), case(big),
             case("", 10, None, kind="closed"), case(short, 0), case(good)]
    want_err = [errno.EBADF, errno.EINVAL, errno.EINVAL, errno.EINVAL, errno.EFBIG, errno.EBADF, errno.EINVAL]
    before = {f: f.read_bytes() for f in (ro, short, v1)}
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        got = run_client(tmp_path, bins["client"], "sock:" + sock, cases)
        assert sock.proc.poll() is None
        assert back_to(sock.proc, base) == base
    assert [g[:2] for g in got[:-1]] == [[False, e] for e in want_err]
    out, s, v, cut = fake_salvage(store)
    assert got[-1] == [True, 0, s, v, cut] and good.read_bytes() == out
    for f, b in before.items():
        assert f.read_bytes() == b, f
    assert os.path.getsize(big) == MAX_PRUNE_STORE + 4096
    good.write_bytes(store)
    local = run_client(tmp_path, bins["inproc"], "inproc", cases[:4] + cases[5:])
    assert [g[:2] for g in local[:-1]] == [[False, e] for e in want_err[:4] + want_err[5:]]
    assert local[-1] == got[-1]
    for f, b in before.items():
        assert f.read_bytes() == b, f


def test_frames(tmp_path, bins):
    """a salvage frame without an fd is answered sigverifyd_error and the connection keeps serving; one with an fd is
    answered sigverifyd_gossip_store_salvage_reply, whose fields the Python codec reads as the daemon's C codec wrote
    them"""
    rng = np.random.default_rng(5)
    f = tmp_path / "gossip_store"
    store = stores()["zeroed_100k"]
    f.write_bytes(store)
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        c.settimeout(60)
        c.connect(sock)
        c.sendall(salvage_frame(1, len(store)))
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=1, code=1))
        vf, vw = verify_req(rng, 2, 0, 2)
        c.sendall(vf)
        assert W.read_msg(c) == vw
        assert f.read_bytes() == store
        fd = os.open(f, os.O_RDWR)
        try:
            socket.send_fds(c, [salvage_frame(3, len(store))], [fd])
        finally:
            os.close(fd)
        name, m = W.read_msg(c)
        out, s, v, cut = fake_salvage(store)
        assert name == "sigverifyd_gossip_store_salvage_reply" and m["req_id"] == 3 and m["err"] == 0
        assert {k: m[k] for k in FIELDS} == s and {k: m[k] for k in sv.FIELDS} == v and m["new_len"] == cut
        c.close()
        assert back_to(sock.proc, base) == base
    assert f.read_bytes() == out
    body = W.encode("sigverifyd_gossip_store_salvage", req_id=7, has_chain=1, chain_hash=TESTNET, len=99)[4:]
    assert len(body) == 2 + 8 + 1 + 32 + 8 and body[:2] == (3012).to_bytes(2, "big")


def test_salvage_beside_channel_checks_never_beside_a_prune(tmp_path, bins):
    """a salvage held 600 ms on the fake prune: another client's verify request is answered while it runs, and another
    client's prune begins only after it ends"""
    rng = np.random.default_rng(6)
    st = [stores()["len_hi"], make_store(rng, 45)]
    files = [tmp_path / "a", tmp_path / "b"]
    for f, s in zip(files, st):
        f.write_bytes(s)
    fds = [os.open(f, os.O_RDWR) for f in files]
    try:
        with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path, {PRUNE: 600})) as sock:
            a, b, vv = (socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) for _ in range(3))
            for c in (a, b, vv):
                c.settimeout(60)
                c.connect(sock)
            socket.send_fds(a, [salvage_frame(1, len(st[0]))], [fds[0]])
            wait_trace(tmp_path, begun(PRUNE))
            socket.send_fds(b, [prune_frame(2, len(st[1]))], [fds[1]])
            for k in range(3):
                f, want = verify_req(rng, 10 + k, 0, 3)
                vv.sendall(f)
                assert W.read_msg(vv) == want
            assert not any(e[:2] == ("end", PRUNE) for e in trace(tmp_path))
            name, m = W.read_msg(a)
            assert name == "sigverifyd_gossip_store_salvage_reply" and m["err"] == 0 and m["restored"] == 1
            name, m = W.read_msg(b)
            assert name == "sigverifyd_gossip_store_prune_reply" and m["err"] == 0
            for c in (a, b, vv):
                c.close()
    finally:
        for fd in fds:
            os.close(fd)
    assert [e[0] for e in trace(tmp_path) if e[1] == PRUNE] == ["begin", "end", "begin", "end"]
    assert files[0].read_bytes() == fake_salvage(st[0])[0]
    assert files[1].read_bytes() == fake_prune(st[1])[0]
