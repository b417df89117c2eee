"""CPU: the drop-in's non-blocking client mode (the _start functions, cln_sigverify_process / _drain / _events / _fd of
cln_dropin.h), built with gcc against the fake engine (tests/host_emul/fake_engine.c) as test_sigverifyd_fake_engine.py
builds it.  Every answer of a ticket must be the answer of the blocking function on the same inputs (which that file pins
to the fake's hash), callbacks must come in ticket order and exactly once, requests a process keeps in flight must share
the daemon's engine calls, and a lost or misbehaving peer must abort the process."""
import json
import os
import signal
import subprocess
import sys

import pytest

from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The client: python -c DRIVER <library> <mode> [args].  It builds seeded random inputs for every function that has a
# _start, runs them as tickets and / or blocking calls as the mode says, and prints what it saw as JSON.
DRIVER = r"""
import ctypes, json, os, socket, subprocess, sys, signal
import numpy as np
from lightning_b200 import sigverifyd_wire as W
from tests.txsig import WallyIn, WallyOut, WallyTx, BitcoinTx
lib = ctypes.CDLL(sys.argv[1])
mode = sys.argv[2]
vp, sz, b_ = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_bool
DONE = ctypes.CFUNCTYPE(None, vp)
for f in ("check_signed_hash", "check_signed_hash_nodeid", "check_schnorr_sig", "check_tx_sig", "bolt12_check_signature"):
    getattr(lib, f).restype = b_
    getattr(lib, f + "_start").restype = ctypes.c_uint64
lib.sigcheck_gossip_batch_start.restype = ctypes.c_uint64
for f in ("check_signed_hash", "check_signed_hash_nodeid", "check_schnorr_sig"):
    getattr(lib, f).argtypes = [vp, vp, vp]
    getattr(lib, f + "_start").argtypes = [vp, vp, vp, vp, DONE, vp]
lib.check_tx_sig.argtypes = [vp, sz, vp, vp, vp, vp]
lib.check_tx_sig_start.argtypes = [vp, sz, vp, vp, vp, vp, vp, DONE, vp]
lib.bolt12_check_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp]
lib.bolt12_check_signature_start.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp, vp, DONE, vp]
lib.sigcheck_gossip_batch.argtypes = [vp, vp, vp, sz, vp, vp, vp]
lib.sigcheck_gossip_batch_start.argtypes = [vp, vp, vp, sz, vp, vp, vp, DONE, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
lib.cln_sigverify_connect_fd.argtypes = [ctypes.c_int]
lib.cln_sigverify_events.restype = ctypes.c_short
lib.cln_sigverify_process.restype = sz
keep, sizes = [], {}
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: sizes[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
rng = np.random.default_rng(int(os.environ.get("SEED", "5")))
def rand(n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return ctypes.addressof(x)
def fields_arr(fields):
    arr = (ctypes.c_uint64 * max(4 * len(fields), 1))()
    for j, (t, v) in enumerate(fields):
        arr[4 * j + 1], arr[4 * j + 2], arr[4 * j + 3] = t, len(v), buf(v) if v else 0
    keep.append(arr)
    sizes[ctypes.addressof(arr)] = 4 * 8 * len(fields)
    return ctypes.addressof(arr)
def make_tx(sht, witness):
    nin, nout = int(rng.integers(1, 4)), int(rng.integers(1, 5))
    ins = (WallyIn * nin)()
    for j in range(nin):
        ins[j].txhash[:] = list(rand(32)); ins[j].index = int(rng.integers(0, 5)); ins[j].sequence = int(rng.integers(0, 2**32))
    outs = (WallyOut * nout)()
    for j in range(nout):
        s = rand(int(rng.choice([0, 22, 34, 300])))
        outs[j].satoshi = int(rng.integers(0, 2**40)); outs[j].script = buf(s) if s else None; outs[j].script_len = len(s)
    w = WallyTx(2, int(rng.integers(0, 2**31)), ctypes.addressof(ins), nin, nin, ctypes.addressof(outs), nout, nout)
    tx = BitcoinTx(ctypes.pointer(w), None, None)
    keep.extend([ins, outs, w, tx])
    sizes[ctypes.addressof(tx)] = int(rng.integers(0, 2**45))
    script = rand(int(rng.choice([1, 71, 300])))
    sp = buf(script)
    sizes[sp] = len(script)
    args = (None, sp) if witness else (sp, None)
    return ctypes.addressof(tx), int(rng.integers(0, nin)), args, buf(rand(64)), buf(rand(64) + int(sht).to_bytes(4, "little"))

class Item:
    # one check of a random kind: .blocking() answers it with the blocking function, .start(arg) starts it as a ticket
    # whose answer .answer() reads once its callback ran
    def __init__(self, kind=None, big=0):
        self.kind = kind or ["signed", "nodeid", "schnorr", "tx", "bolt12", "burst"][int(rng.integers(0, 6))]
        k = self.kind
        if k == "signed":
            self.a = (buf(rand(32)), buf(rand(64)), buf(rand(64)))
        elif k == "nodeid":
            self.a = (buf(rand(32)), buf(rand(64)), buf(rand(33)))
        elif k == "schnorr":
            self.a = (buf(rand(32)), buf(rand(64)), buf(rand(64)))
        elif k == "tx":
            tx, inp, (rs, ws), key, sig = make_tx(int(rng.choice([1, 0x83])), True)
            self.a = (tx, inp, rs, ws, key, sig)
        elif k == "bolt12":
            types = sorted(int(t) for t in rng.choice(70000, 1 if big else int(rng.integers(1, 5)), replace=False))
            fields = [(t, rand(big or int(rng.choice([0, 3, 40, 300])))) for t in types]
            self.a = (fields_arr(fields), [b"invoice", b"invoice_request", b"offer"][int(rng.integers(0, 3))], b"signature",
                      buf(rand(64)), buf(rand(64)))
        else:
            n = int(rng.integers(1, 20))
            msgs = [rand(int(rng.integers(2, 200))) for _ in range(n)]
            ptrs = buf(b"".join(buf(m).to_bytes(8, "little") for m in msgs))
            lens = buf(b"".join(len(m).to_bytes(8, "little") for m in msgs))
            kinds = buf(bytes(int(x) for x in rng.integers(0, 3, size=n))) if rng.random() < 0.5 else None
            self.a = (buf(TESTNET), ptrs, lens, n, kinds, buf(rand(33 * n)) if kinds else None)
            self.n = n
        self.out = (ctypes.c_int * self.n)(*([99] * self.n)) if k == "burst" else b_(True)
    def fn(self):
        return {"signed": "check_signed_hash", "nodeid": "check_signed_hash_nodeid", "schnorr": "check_schnorr_sig",
                "tx": "check_tx_sig", "bolt12": "bolt12_check_signature", "burst": "sigcheck_gossip_batch"}[self.kind]
    def blocking(self):
        if self.kind == "burst":
            st = (ctypes.c_int * self.n)()
            lib.sigcheck_gossip_batch(*self.a, st)
            return list(st)
        return bool(getattr(lib, self.fn())(*self.a))
    def start(self, arg):
        return int(getattr(lib, self.fn() + "_start")(*self.a, ctypes.addressof(self.out), cb, arg))
    def answer(self):
        return list(self.out) if self.kind == "burst" else bool(self.out.value)

order, hooks = [], {}
def on_done(arg):
    order.append(arg)
    if arg in hooks:
        hooks.pop(arg)()
cb = DONE(on_done)
out = {}

def socketpair_client():
    a, b = socket.socketpair()
    assert lib.cln_sigverify_connect_fd(a.detach()) == 0
    return b

if mode == "mixed":  # tickets of every kind, then the same checks blocking
    items = [Item() for _ in range(60)]
    out["tickets"] = [it.start(i + 1) for i, it in enumerate(items)]
    out["order_after_start"] = list(order)
    lib.cln_sigverify_drain()
    out["order"] = order
    out["async"] = [it.answer() for it in items]
    out["blocking"] = [it.blocking() for it in items]
    out["kinds"] = [it.kind for it in items]
elif mode == "window":  # k of each kind in flight before the daemon starts, or the same checks blocking
    k, blocking = int(sys.argv[3]), sys.argv[4] == "blocking"
    items = [Item(kind) for kind in ("signed", "bolt12", "tx") for _ in range(k)]
    b = socketpair_client()
    if not blocking:
        out["tickets"] = [it.start(i + 1) for i, it in enumerate(items)]
    d = subprocess.Popen([sys.argv[5], "--fd", str(b.fileno()), "0"], pass_fds=(b.fileno(),))
    b.close()
    if blocking:
        out["answers"] = [it.blocking() for it in items]
    else:
        lib.cln_sigverify_drain()
        out["answers"] = [it.answer() for it in items]
        out["order"] = order
    lib.cln_sigverify_shutdown()  # the daemon's --fd peer goes away: it exits
    out["daemon_rc"] = d.wait(timeout=60)
elif mode == "interleave":  # blocking calls between tickets, and inside a callback that starts tickets of its own
    items = [Item() for _ in range(40)]
    for k in (3, 12):
        items[k] = Item("burst")
    tk = {}
    for i in range(10):
        tk[i] = items[i].start(i + 1)
    before = items[3].answer()
    got = {10: items[10].blocking()}
    out["earlier_written"] = before == [99] * items[3].n and items[3].answer() != before
    out["no_callback_in_blocking"] = order == []
    def inner():
        for i in range(20, 25):
            tk[i] = items[i].start(i + 1)
        got[25] = items[25].blocking()
        tk[26] = items[26].start(27)
    hooks[5] = inner
    for i in range(11, 20):
        tk[i] = items[i].start(i + 1)
    got[12] = items[12].blocking()  # the same burst again, the blocking way, while its ticket is outstanding
    lib.cln_sigverify_drain()
    out["order"] = order
    out["tickets"] = [tk[i] for i in sorted(tk)]
    out["ticket_index"] = sorted(tk)
    out["async"] = {i: items[i].answer() for i in tk}
    out["async_blocking"] = {i: got[i] for i in got}
    out["blocking"] = {i: items[i].blocking() for i in list(tk) + list(got)}
elif mode == "gates":  # answered locally: 0, the answer written, nothing sent
    ok = b_(True)
    tx, inp, (rs, ws), key, sig = make_tx(2, True)
    r = [lib.check_tx_sig_start(tx, inp, rs, ws, key, sig, ctypes.addressof(ok), cb, 1), ok.value]
    ok.value = True
    tx, inp, (rs, ws), key, sig = make_tx(0x83, False)  # SINGLE|ANYONECANPAY needs a witness script
    r += [lib.check_tx_sig_start(tx, inp, rs, ws, key, sig, ctypes.addressof(ok), cb, 2), ok.value]
    for fields in ([(5, b"a"), (5, b"b")], [(9, b"a"), (3, b"b")], []):
        ok.value = True
        r += [lib.bolt12_check_signature_start(fields_arr(fields), b"invoice", b"signature", buf(rand(64)), buf(rand(64)),
                                               ctypes.addressof(ok), cb, 3), ok.value]
    r.append(lib.sigcheck_gossip_batch_start(buf(TESTNET), None, None, 0, None, None, None, cb, 4))
    out["gates"] = r
    out["process"] = lib.cln_sigverify_process()
    out["events"] = lib.cln_sigverify_events()
    out["order"] = order
elif mode == "pressure":  # a peer that never reads: nothing blocks below the cap
    b = socketpair_client()
    signal.alarm(60)
    it = Item("bolt12", big=60000)  # one 60 kB field per request: 1,024 of them stay below 64 MiB
    tickets = [it.start(i + 1) for i in range(1024)]
    out["distinct"] = len(set(tickets)) == 1024 and min(tickets) > 0
    out["events"] = lib.cln_sigverify_events()
    out["outstanding"] = lib.cln_sigverify_process()
    out["order"] = order
    print(json.dumps(out), flush=True)
    os._exit(0)
elif mode == "lost":  # the peer goes away with tickets outstanding
    b = socketpair_client()
    for i in range(3):
        Item("signed").start(i + 1)
    b.close()
    lib.cln_sigverify_drain()
    print("drained", flush=True)
elif mode == "order":  # a peer that answers the second request before the first
    b = socketpair_client()
    items = [Item("signed"), Item("signed")]
    t = [it.start(i + 1) for i, it in enumerate(items)]
    ids = [W.read_msg(b)[1]["req_id"] for _ in t]
    assert ids == t, (ids, t)
    b.sendall(W.encode("sigverifyd_verify_reply", req_id=t[1], n=1, verdicts=b"\x01"))
    b.sendall(W.encode("sigverifyd_verify_reply", req_id=t[0], n=1, verdicts=b"\x01"))
    lib.cln_sigverify_drain()
    print("drained", flush=True)
elif mode == "inprocess":  # no daemon: every _start answers at once
    items = [Item(k) for k in ("signed", "nodeid", "schnorr", "tx", "burst") for _ in range(4)]
    out["fd"] = lib.cln_sigverify_fd()
    out["tickets"] = [it.start(i + 1) for i, it in enumerate(items)]
    out["async"] = [it.answer() for it in items]
    out["blocking"] = [it.blocking() for it in items]
    out["events"] = lib.cln_sigverify_events()
    out["process"] = lib.cln_sigverify_process()
    lib.cln_sigverify_drain()
    out["order"] = order
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    d = tmp_path_factory.mktemp("async_client")
    return dict(daemon=sf.daemon(d / "cln_sigverifyd"), lib=sf.dropin(d / "libcln_dropin_fake.so"),
                inproc=sf.dropin(d / "libcln_dropin_inproc.so", client=False))


def _env(**kw):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.pop("CLN_SIGVERIFYD_SOCKET", None)
    env.update(kw)
    return env


def _run(lib, mode, *args, env=None, ok=True):
    r = subprocess.run([sys.executable, "-c", DRIVER, lib, mode, *map(str, args)], env=env or _env(), capture_output=True,
                       text=True, timeout=300)
    if not ok:
        return r
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.splitlines()[-1])


@pytest.fixture
def fake(tmp_path, bins):
    """a daemon on the fake engine, and the engine's call log"""
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        yield sock, tmp_path / "engine.log"


def test_mixed_tickets_match_blocking_calls(fake, bins):
    """60 tickets of every kind (the three verify kinds, bolt12, tx, gossip burst) from one connection: every answer is
    the blocking call's, callbacks run only from cln_sigverify_drain, in ticket order, each once"""
    sock, _ = fake
    out = _run(bins["lib"], "mixed", env=_env(CLN_SIGVERIFYD_SOCKET=sock))
    assert out["async"] == out["blocking"]
    assert out["order_after_start"] == []
    assert out["order"] == list(range(1, 61))
    assert out["tickets"] == sorted(out["tickets"]) and len(set(out["tickets"])) == 60 and min(out["tickets"]) > 0
    assert set(out["kinds"]) == {"signed", "nodeid", "schnorr", "tx", "bolt12", "burst"}
    flat = [a for a in out["async"] if isinstance(a, bool)]
    assert any(flat) and not all(flat)
    assert sigverifyd_daemon.stats(sock)["requests"] == 120


@pytest.mark.parametrize("k", [1, 5])
def test_a_window_shares_engine_calls(tmp_path, bins, k):
    """k requests of each of three types written into a socketpair before the daemon starts on it (--fd): one engine call
    per type for the whole window, where k blocking calls make k calls each; the answers are the same"""
    logs, outs = {}, {}
    for how in ("tickets", "blocking"):
        log = tmp_path / ("engine_%s.log" % how)
        outs[how] = _run(bins["lib"], "window", k, how, bins["daemon"], env=_env(FAKE_ENGINE_LOG=str(log)))
        assert outs[how]["daemon_rc"] == 0
        logs[how] = [c[:3] for c in sf.calls(log)]
    assert outs["tickets"]["answers"] == outs["blocking"]["answers"]
    assert outs["tickets"]["order"] == list(range(1, 3 * k + 1))
    assert logs["tickets"] == [("sv_verify_host", 1, k), ("sv_verify_bolt12_tagged_host", 0, k), ("sv_verify_tx_host", 1, k)]
    assert sorted(logs["blocking"]) == sorted([("sv_verify_host", 1, 1)] * k + [("sv_verify_bolt12_tagged_host", 0, 1)] * k +
                                              [("sv_verify_tx_host", 1, 1)] * k)


def test_blocking_calls_between_tickets(fake, bins):
    """blocking calls with tickets outstanding write the earlier tickets' answers but run no callback; a callback that
    starts tickets and makes a blocking call itself; every answer is the blocking call's"""
    sock, _ = fake
    out = _run(bins["lib"], "interleave", env=_env(CLN_SIGVERIFYD_SOCKET=sock))
    assert out["earlier_written"] and out["no_callback_in_blocking"]
    assert out["tickets"] == sorted(out["tickets"])
    # callbacks in ticket order: 1..20, the callback of 5 started 21..25 and 27, which come after 20
    assert out["order"] == [i + 1 for i in out["ticket_index"]]
    assert out["async"] == {i: out["blocking"][i] for i in out["async"]}
    assert out["async_blocking"] == {i: out["blocking"][i] for i in out["async_blocking"]}


def test_local_gates_send_nothing(fake, bins):
    """check_tx_sig's sighash-type gate, an empty or not strictly ascending BOLT12 field array and an empty gossip burst
    answer at once (0, false) and send nothing"""
    sock, _ = fake
    out = _run(bins["lib"], "gates", env=_env(CLN_SIGVERIFYD_SOCKET=sock))
    assert out["gates"] == [0, False] * 5 + [0]
    assert out["process"] == 0 and out["events"] == 0 and out["order"] == []
    assert sigverifyd_daemon.stats(sock)["requests"] == 0


def test_back_pressure_below_the_cap(bins):
    """a peer that never reads: 1,024 tickets of about 60 kB each all start without blocking (an alarm would end the
    process), the rest of the bytes wait unsent (POLLOUT) and every ticket is outstanding"""
    out = _run(bins["lib"], "pressure")
    assert out["distinct"] and out["order"] == []
    assert out["events"] == 0x001 | 0x004  # POLLIN | POLLOUT
    assert out["outstanding"] == 1024


@pytest.mark.parametrize("mode,message", [("lost", "verifier subdaemon: "), ("order", "reply out of order")])
def test_lost_peer_or_reply_out_of_order_aborts(bins, mode, message):
    """the peer closing with tickets outstanding, or answering the second request first, aborts the process: an answer is
    never made up"""
    r = _run(bins["lib"], mode, ok=False)
    assert r.returncode == -signal.SIGABRT, (r.returncode, r.stderr[-2000:])
    assert message in r.stderr and "drained" not in r.stdout


def test_in_process_mode_answers_at_once(bins):
    """the fake engine linked in and no daemon: every _start returns 0 with the blocking call's answer, there is no socket
    to watch and no callback"""
    out = _run(bins["inproc"], "inprocess")
    assert out["fd"] == -1 and out["tickets"] == [0] * 20
    assert out["async"] == out["blocking"]
    assert out["events"] == 0 and out["process"] == 0 and out["order"] == []
