"""CPU: the verifier subdaemon's two engine workers (sigverifyd.c), built with gcc against the fake engine
(tests/host_emul/fake_engine.c) with time added: a delay on chosen entry points ($FAKE_ENGINE_DELAY) and a trace of every
call's begin and end with its context ($FAKE_ENGINE_TRACE).  Checked: a burst on one worker does not hold another client's
check behind it, replies leave in each client's request order whichever job ends first, two passes run on the two
contexts at once, two gossip jobs never overlap, a pending list at MAX_PENDING loses nothing, and a client that leaves
with jobs in flight (or the --fd parent) is handled without a crash or a process left behind."""
import select
import socket
import subprocess
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.sigverifyd_fake import TAGS, begun, bolt12_req, burst_req, calls, short, tx_req, verify_req, wait_trace

MAX_PENDING = 4096
BURST = "sv_verify_gossip_burst_host"


@pytest.fixture(scope="module")
def daemon_bin(tmp_path_factory):
    return sf.daemon(tmp_path_factory.mktemp("workers") / "cln_sigverifyd")


def _open_calls(events):
    """per event index, the calls open just before it: a list of (function, context)"""
    open_, out = [], []
    for ev, fn, ctx in events:
        out.append(list(open_))
        if ev == "begin":
            open_.append((fn, ctx))
        else:
            open_.remove((fn, ctx))
    return out


def _readable(sock):
    return bool(select.select([sock], [], [], 0)[0])


def test_burst_does_not_hold_another_clients_check(tmp_path, daemon_bin):
    """client A's burst is held 500 ms on the device; client B's tx request, sent after the burst began, is answered
    first, and its engine call begins on the other context while the burst's call is still open"""
    rng = np.random.default_rng(1)
    with sigverifyd_daemon.running(tmp_path, daemon_bin, env=sf.env(tmp_path, {BURST: 500})) as sock:
        a, b = sigverifyd_daemon.connect(sock), sigverifyd_daemon.connect(sock)
        burst, burst_want = burst_req(rng, 1, 40)
        tx, tx_want = tx_req(rng, 2, 0, [(60, 40, 0, 0), (30, 20, 72, 8)], 1)
        a.sendall(burst)
        wait_trace(tmp_path, begun(BURST))
        b.sendall(tx)
        assert W.read_msg(b) == tx_want
        assert not _readable(a)  # the burst is still on the device
        assert W.read_msg(a) == burst_want
        a.close()
        b.close()
    trace = sf.trace(tmp_path)
    i = next(k for k, e in enumerate(trace) if e[:2] == ("begin", "sv_verify_tx_host"))
    burst_ctx = next(e[2] for e in trace if e[1] == BURST)
    assert (BURST, burst_ctx) in _open_calls(trace)[i] and trace[i][2] != burst_ctx


def _per_client_frames(rng):
    burst, bw = burst_req(rng, 1, 30)
    ver, vw = verify_req(rng, 2, 1, 4)
    b12, b12w = bolt12_req(rng, 3, *TAGS[1], [50, 0, 7], 1)
    stats = W.encode("sigverifyd_stats", req_id=4)
    bad = short(verify_req(rng, 5, 0, 2)[0])
    return burst + ver + b12 + stats + bad, [bw, vw, b12w]


def test_replies_leave_in_request_order(tmp_path, daemon_bin):
    """one client writes a burst (held 400 ms), a verify, a BOLT12 request, a stats request and a malformed frame: the
    verify call ends first, yet the replies come in request order, the stats reply counts the three requests before
    it, and every reply is the one a daemon without delays gives"""
    replies = {}
    for how, delays in (("delayed", {BURST: 400}), ("plain", {})):
        d = tmp_path / how
        d.mkdir()
        frames, want = _per_client_frames(np.random.default_rng(2))
        with sigverifyd_daemon.running(d, daemon_bin, env=sf.env(d, delays)) as sock:
            c = sigverifyd_daemon.connect(sock)
            c.sendall(frames)
            replies[how] = [W.read_msg(c) for _ in range(5)]
            c.close()
        assert replies[how][:3] == want
        assert replies[how][3] == ("sigverifyd_stats_reply", dict(req_id=4, requests=3, launches=3, signatures=4 + 3 + 30,
                                                                  max_coalesced=1))
        assert replies[how][4] == ("sigverifyd_error", dict(req_id=5, code=1))
        if how == "delayed":
            ends = [e[1] for e in sf.trace(d) if e[0] == "end"]
            assert ends.index("sv_verify_host") < ends.index(BURST)
    assert replies["delayed"] == replies["plain"]


def test_two_passes_in_flight(tmp_path, daemon_bin):
    """with sv_verify_host held 400 ms, a request arriving while one pass runs forms a second pass on the other context:
    the two calls overlap"""
    rng = np.random.default_rng(3)
    with sigverifyd_daemon.running(tmp_path, daemon_bin, env=sf.env(tmp_path, {"sv_verify_host": 400})) as sock:
        a, b = sigverifyd_daemon.connect(sock), sigverifyd_daemon.connect(sock)
        ra, rb = verify_req(rng, 1, 0, 3), verify_req(rng, 2, 2, 5)
        a.sendall(ra[0])
        wait_trace(tmp_path, begun("sv_verify_host"))
        b.sendall(rb[0])
        assert W.read_msg(b) == rb[1]
        assert W.read_msg(a) == ra[1]
        a.close()
        b.close()
    trace = [e for e in sf.trace(tmp_path) if e[1] == "sv_verify_host"]
    assert [e[0] for e in trace] == ["begin", "begin", "end", "end"]
    assert trace[0][2] != trace[1][2]


def test_one_gossip_job_at_a_time(tmp_path, daemon_bin):
    """two clients send bursts at once while a third keeps sending verify requests: the bursts' calls never overlap, and
    passes run beside each of them"""
    rng = np.random.default_rng(4)
    with sigverifyd_daemon.running(tmp_path, daemon_bin, env=sf.env(tmp_path, {BURST: 300, "sv_verify_host": 20})) as sock:
        g1, g2, v = (sigverifyd_daemon.connect(sock) for _ in range(3))
        bursts = [burst_req(rng, 10 + k, 20) for k in range(4)]
        g1.sendall(bursts[0][0] + bursts[1][0])
        g2.sendall(bursts[2][0] + bursts[3][0])
        done, errors = threading.Event(), []

        def passes():
            j = 0
            while not done.is_set():
                f, want = verify_req(rng, 100 + j, 1, 2)
                v.sendall(f)
                got = W.read_msg(v)
                if got != want:
                    errors.append((got, want))
                j += 1

        th = threading.Thread(target=passes)
        th.start()
        try:
            assert [W.read_msg(g1) for _ in range(2)] == [bursts[0][1], bursts[1][1]]
            assert [W.read_msg(g2) for _ in range(2)] == [bursts[2][1], bursts[3][1]]
        finally:
            done.set()
            th.join(timeout=30)
        assert not errors
        for c in (g1, g2, v):
            c.close()
    trace = sf.trace(tmp_path)
    opened = _open_calls(trace)
    beside = 0
    for i, (ev, fn, ctx) in enumerate(trace):
        if ev == "begin" and fn == BURST:
            assert not any(f == BURST for f, _ in opened[i]), trace
        if ev == "begin" and fn == "sv_verify_host" and any(f == BURST for f, _ in opened[i]):
            beside += 1
    assert sum(1 for e in trace if e[:2] == ("begin", BURST)) == 4
    assert beside >= 4


def test_full_pending_list_loses_nothing(tmp_path, daemon_bin):
    """both workers held 1.5 s, then 5,000 verify requests from one client: the pending list stops at MAX_PENDING, the
    rest waits unread; every request is answered in order and the stats counts are exact"""
    rng = np.random.default_rng(5)
    n = 5000
    with sigverifyd_daemon.running(tmp_path, daemon_bin, env=sf.env(tmp_path, {"sv_verify_host": 1500})) as sock:
        holders = [sigverifyd_daemon.connect(sock) for _ in range(2)]
        held = [verify_req(rng, 1 + k, 0, 1) for k in range(2)]
        for k, h in enumerate(holders):
            h.sendall(held[k][0])
            wait_trace(tmp_path, begun("sv_verify_host", k + 1))
        reqs = [verify_req(rng, 1000 + j, 2, 1) for j in range(n)]
        c = sigverifyd_daemon.connect(sock)
        sender = threading.Thread(target=c.sendall, args=(b"".join(f for f, _ in reqs),))
        sender.start()
        got = [W.read_msg(c) for _ in range(n)]
        sender.join(timeout=60)
        for k, h in enumerate(holders):
            assert W.read_msg(h) == held[k][1]
            h.close()
        assert got == [w for _, w in reqs]
        st = sigverifyd_daemon.stats(sock)
        c.close()
    log = calls(tmp_path / "engine.log")
    assert st["requests"] == n + 2 and st["signatures"] == n + 2 and st["launches"] == len(log) >= 4
    assert st["max_coalesced"] == MAX_PENDING
    assert sum(x[2] for x in log) == n + 2 and max(x[2] for x in log) == MAX_PENDING


def test_clients_leaving_with_jobs_in_flight(tmp_path, daemon_bin):
    """a client that closes with a burst and a pass in flight, and one that half-closes and still reads its answers:
    the daemon stays up, answers the second, and serves new clients on freed slots"""
    rng = np.random.default_rng(6)
    with sigverifyd_daemon.running(tmp_path, daemon_bin, env=sf.env(tmp_path, {BURST: 400, "sv_verify_host": 200})) as sock:
        gone = sigverifyd_daemon.connect(sock)
        gone.sendall(burst_req(rng, 1, 10)[0] + verify_req(rng, 2, 0, 2)[0])
        wait_trace(tmp_path, lambda t: begun(BURST)(t) and begun("sv_verify_host")(t))
        gone.close()
        half = sigverifyd_daemon.connect(sock)
        reqs = [burst_req(rng, 3, 5), verify_req(rng, 4, 1, 1), tx_req(rng, 5, 1, [(9, 9, 0, 0)], 0)]
        half.sendall(b"".join(f for f, _ in reqs))
        half.shutdown(socket.SHUT_WR)
        assert [W.read_msg(half) for _ in reqs] == [w for _, w in reqs]
        assert half.recv(1) == b""
        half.close()
        for k in range(20):  # new clients, one of them on the slot the first one left
            c = sigverifyd_daemon.connect(sock)
            f, want = verify_req(rng, 100 + k, 2, 1)
            c.sendall(f)
            assert W.read_msg(c) == want
            c.close()
        assert sigverifyd_daemon.stats(sock)["requests"] == 2 + 3 + 20


@pytest.mark.parametrize("how", ["half_close", "close"])
def test_fd_mode_exits_after_its_jobs(tmp_path, daemon_bin, how):
    """--fd mode: the parent goes away with a burst and a pass in flight.  With a half-close it still gets every answer;
    either way the daemon finishes the jobs, exits with 0 and leaves no process behind"""
    rng = np.random.default_rng(7)
    parent, child = socket.socketpair()
    d = subprocess.Popen([daemon_bin, "--fd", str(child.fileno()), "0"], pass_fds=(child.fileno(),),
                         env=sf.env(tmp_path, {BURST: 400, "sv_verify_host": 200}), stderr=subprocess.PIPE)
    child.close()
    try:
        reqs = [burst_req(rng, 1, 8), verify_req(rng, 2, 0, 3), bolt12_req(rng, 3, *TAGS[0], [20], 0)]
        parent.sendall(b"".join(f for f, _ in reqs))
        wait_trace(tmp_path, lambda t: begun(BURST)(t) and begun("sv_verify_host")(t))
        if how == "half_close":
            parent.shutdown(socket.SHUT_WR)
            parent.settimeout(30)
            assert [W.read_msg(parent) for _ in reqs] == [w for _, w in reqs]
            assert parent.recv(1) == b""
        parent.close()
        assert d.wait(timeout=30) == 0, d.stderr.read()
    finally:
        if d.poll() is None:
            d.kill()
            d.wait(timeout=10)
    trace = sf.trace(tmp_path)
    assert sum(1 for e in trace if e[0] == "end") == sum(1 for e in trace if e[0] == "begin") == 3
