"""CPU: pruning a gossip_store FILE in place — sv_prune_gossip_store_fd (lightning_b200/csrc/gossip_store_fd.c), the
verifier subdaemon's sigverifyd_gossip_store_prune (the store's fd passed over the socket with SCM_RIGHTS) and the drop-in's
gossip_store_prune in both modes — built with gcc against a fake prune (tests/host_emul/fake_engine_prune.c) that deletes a
fixed set of records.  Checked: the file changes only in bit 0x8000 of the flags of the records the
fake deleted, the same way in-process, through a daemon on a socket and through `--fd N`; a client-mode process never
creates a context; every refused file or frame is answered without the daemon exiting, leaves the file as it was, and
leaves the daemon with no descriptor more than before; a prune runs beside channel checks and never beside another
prune; the codec of the new messages."""
import errno
import os
import socket
import subprocess
import time

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_codec as codec
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.gossip_store_prune import REASONS
from tests.sigverifyd_fake import (FIELDS, MAX_PRUNE_STORE, PRUNE, back_to, begun, case, fake_prune, make_store, nfds,
                                   prune_frame, run_client, trace, verify_req, wait_trace)


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    return sf.store_bins(tmp_path_factory.mktemp("prune_fake"))


# ---- the file after a prune ------------------------------------------------------------------------------------------
STORES = [(0, 40, 0), (1, 200, 0), (2, 61, 37), (3, 0, 0)]  # seed, records, bytes of a cut-short last record


@pytest.mark.parametrize("seed,n,tail", STORES)
def test_file_pruned_in_place_every_way(tmp_path, bins, seed, n, tail):
    """in-process, through a daemon on a socket and through `--fd N`: the file ends as the fake's pruned store (only bit
    0x8000 of the deleted records' flags differs), with the fake's summary; a second prune deletes nothing"""
    store = make_store(np.random.default_rng(seed), n, tail=tail)
    want, summary = fake_prune(store)
    diff = [i for i in range(len(store)) if store[i] != want[i]]
    assert all(store[i] ^ want[i] == 0x80 for i in diff) and len(diff) == summary["pruned"]
    assert n < 3 or summary["pruned"]
    files = {}
    for how in ("inproc", "sock", "fd"):
        files[how] = tmp_path / ("gossip_store." + how)
        files[how].write_bytes(store)
    got = {"inproc": run_client(tmp_path, bins["inproc"], "inproc", [case(files["inproc"])] * 2)}
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        got["sock"] = run_client(tmp_path, bins["client"], "sock:" + sock, [case(files["sock"])] * 2)
        assert sock.proc.poll() is None
    parent, child = socket.socketpair()
    d = subprocess.Popen([bins["daemon"], "--fd", str(child.fileno()), "0"], pass_fds=(child.fileno(),), env=sf.env(tmp_path),
                         stderr=subprocess.PIPE)
    child.close()
    try:
        got["fd"] = run_client(tmp_path, bins["client"], "fd:%d" % parent.fileno(), [case(files["fd"])] * 2,
                               pass_fds=(parent.fileno(),))
        parent.close()
        assert d.wait(timeout=30) == 0  # the parent went away: the daemon ends
    finally:
        if d.poll() is None:
            d.kill()
            d.wait(timeout=10)
    again = dict(summary, pruned=0, reverified=0, **{r: 0 for r in REASONS})
    for how in files:
        assert files[how].read_bytes() == want, how
        assert got[how] == [[True, 0, summary, None], [True, 0, again, None]], how


def test_client_mode_never_creates_a_context(tmp_path, bins):
    """the client-mode library's sv_create aborts: the prunes above went through the daemon only, and an in-process call
    with that library does reach it"""
    f = tmp_path / "gossip_store"
    f.write_bytes(make_store(np.random.default_rng(9), 10))
    r = run_client(tmp_path, bins["client"], "inproc", [case(f)], check=False)
    assert r.returncode != 0 and "sv_create called" in r.stderr


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refused_files(tmp_path, bins):
    """a read-only fd (EBADF), a pipe (EINVAL), a length past the end of the file (EINVAL), a store the engine refuses
    (EINVAL), a store above the daemon's cap (EFBIG, never reaching the engine) and a closed descriptor (EBADF, nothing
    sent): false with that errno, in-process and through the daemon; the daemon stays up, no file changes, and the
    daemon's descriptor count returns to what it was"""
    store = make_store(np.random.default_rng(4), 30)
    ro, short, v1, good = (tmp_path / x for x in ("ro", "short", "v1", "good"))
    for f in (ro, short, good):
        f.write_bytes(store)
    v1.write_bytes(bytes([0x20]) + store[1:])  # major version 1
    big = tmp_path / "big"
    with open(big, "wb") as fh:  # sparse: no data blocks
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
    assert got[-1] == [True, 0, fake_prune(store)[1], None]
    for f, b in before.items():
        assert f.read_bytes() == b, f
    assert os.path.getsize(big) == MAX_PRUNE_STORE + 4096
    assert [c[3] for c in sf.calls(tmp_path / "engine.log") if c[0] == PRUNE] == [len(store)]  # v1: refused before the log line; big: never sent
    # in-process: the same answers, except the cap, which is the daemon's
    for f in (short, good):
        f.write_bytes(store)
    local = run_client(tmp_path, bins["inproc"], "inproc", cases[:4] + cases[5:])
    assert [g[:2] for g in local[:-1]] == [[False, e] for e in want_err[:4] + want_err[5:]]
    assert local[-1] == got[-1]
    for f, b in before.items():
        assert f.read_bytes() == b, f


def _closed(c):
    c.settimeout(20)
    try:
        return c.recv(1) == b""
    except ConnectionResetError:
        return True


def test_refused_frames(tmp_path, bins):
    """on the wire: a prune frame without an fd and an fd sent with a verify frame are answered sigverifyd_error and the
    connection keeps serving (the stray fd closed); two fds in one message, or more fds waiting than the daemon keeps, drop
    that client.  The file never changes and the daemon's descriptor count returns to what it was after each case"""
    rng = np.random.default_rng(5)
    f = tmp_path / "gossip_store"
    store = make_store(rng, 20)
    f.write_bytes(store)
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        fd = os.open(f, os.O_RDWR)
        try:
            c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            c.settimeout(30)
            c.connect(sock)
            base_c = back_to(sock.proc, base + 1)
            c.sendall(prune_frame(1, len(store)))                                 # no fd
            assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=1, code=1))
            vf, vw = verify_req(rng, 2, 0, 2)
            socket.send_fds(c, [vf], [fd])                                        # an fd with a verify frame
            assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=2, code=1))
            assert back_to(sock.proc, base_c) == base_c
            vf, vw = verify_req(rng, 3, 1, 2)
            c.sendall(vf)                                                         # still serving
            assert W.read_msg(c) == vw
            c.close()
            assert back_to(sock.proc, base) == base
            for how in ("two", "many"):
                c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
                c.connect(sock)
                frame = prune_frame(4, len(store))
                if how == "two":
                    socket.send_fds(c, [frame], [fd, fd])
                else:  # one byte of the frame per message, each with an fd: they all wait for the frame to end
                    for k in range(6):
                        try:
                            socket.send_fds(c, [frame[k:k + 1]], [fd])
                        except OSError:
                            break
                        time.sleep(0.05)
                assert _closed(c), how
                c.close()
                assert sock.proc.poll() is None
                assert back_to(sock.proc, base) == base, how
        finally:
            os.close(fd)
    assert f.read_bytes() == store
    assert not (tmp_path / "engine.log").exists() or PRUNE not in (tmp_path / "engine.log").read_text()


# ---- the gossip worker -----------------------------------------------------------------------------------------------
def test_prune_beside_channel_checks(tmp_path, bins):
    """the prune is held 600 ms on the fake: another client's verify request is answered while it runs, and a second
    client's prune begins only after the first ends; both files end pruned"""
    rng = np.random.default_rng(6)
    stores = [make_store(rng, 30), make_store(rng, 45)]
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
            socket.send_fds(a, [prune_frame(1, len(stores[0]))], [fds[0]])
            wait_trace(tmp_path, begun(PRUNE))
            socket.send_fds(b, [prune_frame(2, len(stores[1]))], [fds[1]])
            for k in range(3):
                f, want = verify_req(rng, 10 + k, 0, 3)
                v.sendall(f)
                assert W.read_msg(v) == want
            assert not any(e[:2] == ("end", PRUNE) for e in trace(tmp_path))  # answered while the prune runs
            for c, rid, s in ((a, 1, stores[0]), (b, 2, stores[1])):
                name, m = W.read_msg(c)
                assert name == "sigverifyd_gossip_store_prune_reply" and m["req_id"] == rid and m["err"] == 0
                assert {k: m[k] for k in FIELDS} == fake_prune(s)[1]
            for c in (a, b, v):
                c.close()
    finally:
        for fd in fds:
            os.close(fd)
    assert [e[0] for e in trace(tmp_path) if e[1] == PRUNE] == ["begin", "end", "begin", "end"]  # never two at once
    for f, s in zip(files, stores):
        assert f.read_bytes() == fake_prune(s)[0]


def test_client_leaving_with_a_prune_in_flight(tmp_path, bins):
    """a client that closes its connection while its prune runs, and one that closes while its prune waits behind it: both
    jobs finish, the daemon stays up, and its descriptor count returns to what it was"""
    rng = np.random.default_rng(7)
    stores = [make_store(rng, 25), make_store(rng, 26)]
    files = [tmp_path / "a", tmp_path / "b"]
    for f, s in zip(files, stores):
        f.write_bytes(s)
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path, {PRUNE: 400})) as sock:
        time.sleep(0.2)
        base = nfds(sock.proc)
        for f, s in zip(files, stores):
            fd = os.open(f, os.O_RDWR)
            c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            c.connect(sock)
            socket.send_fds(c, [prune_frame(1, len(s))], [fd])
            os.close(fd)
            if f is files[0]:
                wait_trace(tmp_path, begun(PRUNE))
            c.close()
        wait_trace(tmp_path, lambda t: sum(1 for e in t if e[:2] == ("end", PRUNE)) == 2)
        assert back_to(sock.proc, base) == base
        assert sock.proc.poll() is None
        f2, want = verify_req(rng, 5, 2, 1)
        c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        c.settimeout(30)
        c.connect(sock)
        c.sendall(f2)
        assert W.read_msg(c) == want
        c.close()
    for f, s in zip(files, stores):
        assert f.read_bytes() == fake_prune(s)[0]


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
            int(x) for x in rng.integers(0, 2**64, size=12, dtype=np.uint64)]
        rep = dict(zip(["req_id", "err"] + FIELDS, vals))
        for name, m in (("sigverifyd_gossip_store_prune", req), ("sigverifyd_gossip_store_prune_reply", rep)):
            codec.agree(shim, name, m)
            codec.refused(shim, name, m)
            codec.wrong_type_refused(shim, name, m)
