"""GPU: pruning a gossip_store FILE in place.  Every mutated store of tests/test_gpu_gossip_store_prune.py, and the fixture
tiled x53 with 1 % of its records corrupted, written to a file and pruned there by SigVerifier.prune_gossip_store_fd, by
the drop-in's gossip_store_prune in-process, and by gossip_store_prune in client mode through cln_sigverifyd (the file's
descriptor passed over the socket): the file must end byte for byte as the `out` of SigVerifier.prune_gossip_store on the
same bytes (which tests/test_gpu_gossip_store_prune.py ties to CLN's strict gossmap.c load), with the same summary, and a
second prune of it must delete nothing.  Then the x53 store is pruned through the daemon while 4 clients send
commitment_signed checks: every verdict they get is the in-process engine's."""
import os
import socket
import threading

import numpy as np
import pytest

from lightning_b200 import build
from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_daemon, txsig
from tests.test_gpu_gossip_burst import TESTNET
from tests.test_gpu_gossip_store_prune import corrupted_x53, mutations
from tests.sigverifyd_fake import FIELDS, case, prune_frame, run_client

pytestmark = pytest.mark.gpu

_STORES = {}


def stores():
    if not _STORES:
        _STORES.update(mutations())
        _STORES["x53_corrupted_1pct"] = corrupted_x53()
    return _STORES


@pytest.fixture(scope="module")
def host(engine):
    """per store: (the pruned bytes, the summary) of the host-buffer call"""
    out = {}
    for name, st in stores().items():
        pruned, _, s = engine.prune_gossip_store(st, TESTNET)
        assert s["pruned"] > 0, name
        out[name] = (pruned, s)
    return out


def _nothing_more(s):
    return dict(s, pruned=0, reverified=0, bad_crc=0, truncated=0, message=0, redundant=0, no_channel=0, signature=0,
                amount=0, unknown=0)


def test_python_prune_fd(engine, host, tmp_path):
    """SigVerifier.prune_gossip_store_fd: the file ends as the host call's out, the summaries are equal, and a second
    prune deletes nothing; a read-only descriptor and a length past the end raise OSError and change nothing"""
    for name, st in stores().items():
        f = tmp_path / name
        f.write_bytes(st)
        fd = os.open(f, os.O_RDWR)
        try:
            s = engine.prune_gossip_store_fd(fd, len(st), TESTNET)
            again = engine.prune_gossip_store_fd(fd, len(st), TESTNET)
        finally:
            os.close(fd)
        assert f.read_bytes() == host[name][0], name
        assert s == host[name][1], name
        assert again == _nothing_more(again) and {k: again[k] for k in ("records", "end_offset", "stop")} == \
            {k: s[k] for k in ("records", "end_offset", "stop")}, name
    st = stores()["bad_newest_update"]
    f = tmp_path / "refused"
    f.write_bytes(st)
    for flags, length in ((os.O_RDONLY, len(st)), (os.O_RDWR, len(st) + 1)):
        fd = os.open(f, flags)
        try:
            with pytest.raises(OSError):
                engine.prune_gossip_store_fd(fd, length, TESTNET)
        finally:
            os.close(fd)
    assert f.read_bytes() == st


def test_dropin_in_process_and_through_the_daemon(host, tmp_path):
    """the drop-in's gossip_store_prune on each store, in a process with a context of its own and in client mode through
    a cln_sigverifyd on a socket: the file ends as the host call's out, with its summary; the second prune deletes
    nothing"""
    names = sorted(stores())
    got = {}
    for how in ("inproc", "daemon"):
        d = tmp_path / how
        d.mkdir()
        cases = []
        for name in names:
            (d / name).write_bytes(stores()[name])
            cases += [case(d / name)] * 2
        if how == "inproc":
            got[how] = run_client(d, build.LIB, "inproc", cases)
        else:
            with sigverifyd_daemon.running(d) as sock:
                got[how] = run_client(d, build.LIB, "sock:" + sock, cases)
                st = sigverifyd_daemon.stats(sock)
            assert st["requests"] == st["launches"] == 2 * len(names) and st["signatures"] == 0
        for k, name in enumerate(names):
            pruned, s = host[name]
            assert (d / name).read_bytes() == pruned, (how, name)
            first, second = got[how][2 * k], got[how][2 * k + 1]
            assert first == [True, 0, s, None], (how, name)
            assert second[:2] == [True, 0] and second[2] == _nothing_more(second[2]), (how, name)


def test_x53_through_the_daemon_beside_commitment_signed(engine, host, tmp_path):
    """the x53 store pruned through the daemon while 4 clients send commitment_signed checks (a commitment transaction
    and 30 HTLC transactions, one HTLC signature of every other request corrupted) back to back: each verdict equals the
    in-process engine's, and the file ends as the host call's out"""
    name = "x53_corrupted_1pct"
    st = stores()[name]
    f = tmp_path / "gossip_store"
    f.write_bytes(st)
    (ctx_, cblob), (htx, hblob) = txsig.commitment_signed(np.random.default_rng(30), 30)
    ckey, csig = txsig.sign(engine, 1, bytes([0x21]) * 32, ctx_, cblob)
    hkey, hsig = txsig.sign(engine, 1, bytes([0x22]) * 32, htx, hblob)
    bad = hsig.copy()
    bad[7, 20] ^= 0x10
    want = {False: txsig.expected(engine, 1, hkey, htx, hblob, hsig)[0], True: txsig.expected(engine, 1, hkey, htx, hblob, bad)[0]}
    assert list(want[False]) == [1] * 30 and want[True][7] == 0
    stop, errors, served = threading.Event(), [], []

    def channeld(ci, sock):
        c = sigverifyd_daemon.connect(sock)
        rid, n = 0, 0
        try:
            while not stop.is_set() or n < 5:
                corrupt = (n + ci) % 2 == 1
                rid += 2
                c.sendall(txsig.request(rid - 1, 1, ckey, ctx_, cblob, csig) +
                          txsig.request(rid, 1, hkey, htx, hblob, bad if corrupt else hsig))
                a, b = W.read_msg(c), W.read_msg(c)
                if a != ("sigverifyd_tx_reply", dict(req_id=rid - 1, n=1, verdicts=b"\x01", nsighash=0, sighashes=b"")) or \
                        b[0] != "sigverifyd_tx_reply" or b[1]["req_id"] != rid or bytes(b[1]["verdicts"]) != bytes(want[corrupt]):
                    errors.append((ci, n, a, b))
                n += 1
        finally:
            c.close()
            served.append(n)

    with sigverifyd_daemon.running(tmp_path) as sock:
        th = [threading.Thread(target=channeld, args=(ci, sock)) for ci in range(4)]
        for t in th:
            t.start()
        fd = os.open(f, os.O_RDWR)
        try:
            c = sigverifyd_daemon.connect(sock)
            socket.send_fds(c, [prune_frame(1, len(st))], [fd])
            name_, m = W.read_msg(c)
            c.close()
        finally:
            os.close(fd)
            stop.set()
            for t in th:
                t.join(timeout=300)
    assert not errors, errors[:3]
    assert len(served) == 4 and min(served) >= 5
    assert name_ == "sigverifyd_gossip_store_prune_reply" and m["err"] == 0
    assert {k: m[k] for k in FIELDS if k != "stop"} == {k: v for k, v in host[name][1].items() if k != "stop"}
    assert f.read_bytes() == host[name][0]
