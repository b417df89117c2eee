"""CPU: pruning a gossip_store FILE in place — sv_prune_gossip_store_fd (lightning_b200/csrc/gossip_store_fd.c), the
verifier subdaemon's sigverifyd_gossip_store_prune (the store's fd passed over the socket with SCM_RIGHTS) and the drop-in's
gossip_store_prune in both modes — built with gcc against a fake prune (tests/host_emul/fake_engine_prune.c) that deletes a
fixed set of records.  Checked: the file changes only in bit 0x8000 of the flags of the records the fake deleted, the same
way in-process, through a daemon on a socket and through `--fd N`; a client-mode process never creates a context; every
refused file or frame is answered without the daemon exiting, leaves the file as it was, and leaves the daemon with no
descriptor more than before; a prune runs beside channel checks and never beside another prune; the codec of the new
messages."""
import contextlib
import ctypes
import errno
import json
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest

from lightning_b200 import build
from lightning_b200 import sigverifyd_wire as W
from lightning_b200.engine import SvGossipPruneSummary
from tests.test_sigverifyd_fake_engine import verify_req

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HE = os.path.join(ROOT, "tests", "host_emul")
STORE_FD = os.path.join(build.CSRC, "gossip_store_fd.c")
PRUNE = "sv_prune_gossip_store_host"
FIELDS = [f for f, _ in SvGossipPruneSummary._fields_]
REASONS = ("bad_crc", "truncated", "message", "redundant", "no_channel", "signature", "amount", "unknown")  # SV_GP_1..8
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
MAX_PRUNE_STORE = 4 << 30  # sigverifyd_proto.h
GS_EOF, GS_PARTIAL = 0, 33


# ---- stores and what the fake prune makes of them (fake_engine_prune.c) ----------------------------------------------
def make_store(rng, n, version=0x0C, tail=0):
    """a version byte, n records of random messages (some already deleted), then `tail` bytes of a record cut short"""
    out = bytearray([version])
    for _ in range(n):
        flags = (0x8000 if rng.random() < 0.15 else 0) | 0x2000
        msg = rng.integers(0, 256, size=int(rng.integers(2, 300)), dtype=np.uint8).tobytes()
        out += flags.to_bytes(2, "big") + len(msg).to_bytes(2, "big") + rng.integers(0, 2**32, size=2, dtype=np.uint64).astype(
            ">u4").tobytes() + msg
    if tail:
        out += (0x2000).to_bytes(2, "big") + (tail + 100).to_bytes(2, "big") + bytes(8) + bytes(tail)
    return bytes(out)


def fake_prune(store):
    """(the pruned store, the summary dict) the fake engine gives"""
    out, s = bytearray(store), dict.fromkeys(FIELDS, 0)
    off, r = 1, 0
    s["version"], s["stop"] = store[0], GS_EOF
    while off + 12 <= len(store):
        mlen = int.from_bytes(store[off + 2:off + 4], "big")
        if off + 12 + mlen > len(store):
            s["stop"] = GS_PARTIAL
            break
        if r % 3 == 1 and not store[off] & 0x80:
            why = 1 + (r // 3) % 8
            out[off] |= 0x80
            s["pruned"] += 1
            s[REASONS[why - 1]] += 1
            s["reverified"] += why == 6
        r += 1
        off += 12 + mlen
    s["end_offset"], s["records"] = min(off, len(store)), r
    return bytes(out), s


# ---- builds, daemons and client processes ---------------------------------------------------------------------------
def _gcc(args):
    r = subprocess.run(["gcc"] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    d = tmp_path_factory.mktemp("prune_fake")
    out = dict(daemon=str(d / "cln_sigverifyd"), inproc=str(d / "libdropin_inproc.so"), client=str(d / "libdropin_client.so"),
               shim=str(d / "libwire_shim_prune.so"))
    prune = [os.path.join(HE, "fake_engine_prune.c"), STORE_FD]
    _gcc(build.DAEMON_CFLAGS + [os.path.join(build.CSRC, "sigverifyd.c"), os.path.join(HE, "fake_engine_timed.c")] + prune +
         ["-o", out["daemon"]])
    dropin = build.DROPIN_CFLAGS + ["-shared", os.path.join(build.CSRC, "cln_dropin.c"), os.path.join(HE, "fake_engine.c")] + prune
    _gcc(dropin + ["-o", out["inproc"]])
    _gcc(dropin + ["-DFAKE_ENGINE_NO_CONTEXT", "-o", out["client"]])  # its sv_create aborts
    _gcc(["-O2", "-shared", "-fPIC", "-Wall", os.path.join(HE, "wire_shim_prune.c"), "-o", out["shim"]])
    return out


def _env(tmp_path, delay_ms=0):
    return dict(os.environ, FAKE_ENGINE_LOG=str(tmp_path / "engine.log"), FAKE_ENGINE_TRACE=str(tmp_path / "trace"),
                FAKE_ENGINE_DELAY="%s=%d" % (PRUNE, delay_ms))


@contextlib.contextmanager
def serve(tmp_path, binary, env):
    """the daemon on a socket of its own: yields (process, socket path); stopped however the block ends"""
    sock = os.path.join(str(tmp_path), "sv.sock")
    if len(os.fsencode(sock)) >= 100:
        sock = os.path.join("/tmp", "svp%d.sock" % os.getpid())
    proc = subprocess.Popen([binary, sock, "0"], stderr=subprocess.PIPE, env=env)
    try:
        for _ in range(300):
            if os.path.exists(sock) or proc.poll() is not None:
                break
            time.sleep(0.05)
        assert os.path.exists(sock), "daemon did not come up"
        yield proc, sock
    finally:
        proc.terminate()
        try:
            proc.wait(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.wait(timeout=10)
        if os.path.exists(sock) and sock.startswith("/tmp/svp"):
            os.unlink(sock)


def nfds(proc):
    return len(os.listdir("/proc/%d/fd" % proc.pid))


def back_to(proc, base, timeout=10):
    """the daemon's descriptor count, once it is back at base (or the timeout passed)"""
    end = time.time() + timeout
    while nfds(proc) != base and time.time() < end:
        time.sleep(0.02)
    return nfds(proc)


CLIENT = r"""
import ctypes, json, os, sys
from lightning_b200.engine import SvGossipPruneSummary
lib = ctypes.CDLL(sys.argv[1], use_errno=True)
lib.gossip_store_prune.restype = ctypes.c_bool
lib.gossip_store_prune.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p, ctypes.POINTER(SvGossipPruneSummary)]
lib.cln_sigverify_connect.argtypes = [ctypes.c_char_p]
mode = sys.argv[2]
if mode.startswith("sock:"):
    assert lib.cln_sigverify_connect(mode[5:].encode()) == 0
elif mode.startswith("fd:"):
    assert lib.cln_sigverify_connect_fd(int(mode[3:])) == 0
out = []
for c in json.load(open(sys.argv[3])):
    if c["kind"] == "pipe":
        fd, w = os.pipe()
        os.write(w, bytes(64))
    elif c["kind"] == "closed":
        fd = os.open(os.devnull, os.O_RDONLY)
        os.close(fd)
    else:
        fd = os.open(c["path"], os.O_RDWR if c["kind"] == "rw" else os.O_RDONLY)
    s = SvGossipPruneSummary()
    chain = bytes.fromhex(c["chain"]) if c["chain"] else None
    ok = lib.gossip_store_prune(fd, c["len"], chain, ctypes.byref(s))
    e = ctypes.get_errno()
    if c["kind"] != "closed":
        os.close(fd)
    if c["kind"] == "pipe":
        os.close(w)
    out.append([ok, 0 if ok else e, {f: getattr(s, f) for f, _ in SvGossipPruneSummary._fields_} if ok else None])
print(json.dumps(out))
"""


def run_client(tmp_path, lib, mode, cases, pass_fds=(), check=True):
    path = tmp_path / ("cases%d.json" % time.monotonic_ns())
    path.write_text(json.dumps(cases))
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", CLIENT, lib, mode, str(path)], env=env, capture_output=True, text=True,
                       timeout=120, pass_fds=pass_fds)
    if check:
        assert r.returncode == 0, r.stderr[-3000:]
        return json.loads(r.stdout)
    return r


def case(path, length=None, chain=TESTNET, kind="rw"):
    return dict(kind=kind, path=str(path), len=os.path.getsize(path) if length is None else length,
                chain=chain.hex() if chain else None)


def prune_frame(rid, length, chain=TESTNET):
    return W.encode("sigverifyd_gossip_store_prune", req_id=rid, has_chain=1 if chain else 0, chain_hash=chain or bytes(32),
                    len=length)


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
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        got["sock"] = run_client(tmp_path, bins["client"], "sock:" + sock, [case(files["sock"])] * 2)
        assert proc.poll() is None
    parent, child = socket.socketpair()
    d = subprocess.Popen([bins["daemon"], "--fd", str(child.fileno()), "0"], pass_fds=(child.fileno(),), env=_env(tmp_path),
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
        assert got[how] == [[True, 0, summary], [True, 0, again]], how


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
    cases = [case(ro, kind="ro"), dict(kind="pipe", path="", len=64, chain=None), case(short, len(store) + 1),
             case(v1), case(big), dict(kind="closed", path="", len=10, chain=None), case(short, 0), case(good)]
    want_err = [errno.EBADF, errno.EINVAL, errno.EINVAL, errno.EINVAL, errno.EFBIG, errno.EBADF, errno.EINVAL]
    before = {f: f.read_bytes() for f in (ro, short, v1)}
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        time.sleep(0.2)
        base = nfds(proc)
        got = run_client(tmp_path, bins["client"], "sock:" + sock, cases)
        assert proc.poll() is None
        assert back_to(proc, base) == base
    assert [g[:2] for g in got[:-1]] == [[False, e] for e in want_err]
    assert got[-1] == [True, 0, fake_prune(store)[1]]
    for f, b in before.items():
        assert f.read_bytes() == b, f
    assert os.path.getsize(big) == MAX_PRUNE_STORE + 4096
    calls = [line.split() for line in (tmp_path / "engine.log").read_text().splitlines()]
    assert [int(c[3]) for c in calls if c[0] == PRUNE] == [len(store)]  # v1: refused before the log line; big: never sent
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
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        time.sleep(0.2)
        base = nfds(proc)
        fd = os.open(f, os.O_RDWR)
        try:
            c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            c.settimeout(30)
            c.connect(sock)
            base_c = back_to(proc, base + 1)
            c.sendall(prune_frame(1, len(store)))                                 # no fd
            assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=1, code=1))
            vf, vw = verify_req(rng, 2, 0, 2)
            socket.send_fds(c, [vf], [fd])                                        # an fd with a verify frame
            assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=2, code=1))
            assert back_to(proc, base_c) == base_c
            vf, vw = verify_req(rng, 3, 1, 2)
            c.sendall(vf)                                                         # still serving
            assert W.read_msg(c) == vw
            c.close()
            assert back_to(proc, base) == base
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
                assert proc.poll() is None
                assert back_to(proc, base) == base, how
        finally:
            os.close(fd)
    assert f.read_bytes() == store
    assert not (tmp_path / "engine.log").exists() or PRUNE not in (tmp_path / "engine.log").read_text()


# ---- the gossip worker -----------------------------------------------------------------------------------------------
def _trace(tmp_path):
    p = tmp_path / "trace"
    return [tuple(line.split()) for line in p.read_text().splitlines()] if p.exists() else []


def _wait(pred, timeout=30):
    end = time.time() + timeout
    while time.time() < end:
        if pred():
            return
        time.sleep(0.01)
    raise AssertionError("condition not reached")


def _begun(tmp_path, fn, count=1):
    return lambda: sum(1 for e in _trace(tmp_path) if e[:2] == ("begin", fn)) >= count


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
        with serve(tmp_path, bins["daemon"], _env(tmp_path, 600)) as (proc, sock):
            a, b, v = (socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) for _ in range(3))
            for c in (a, b, v):
                c.settimeout(30)
                c.connect(sock)
            socket.send_fds(a, [prune_frame(1, len(stores[0]))], [fds[0]])
            _wait(_begun(tmp_path, PRUNE))
            socket.send_fds(b, [prune_frame(2, len(stores[1]))], [fds[1]])
            for k in range(3):
                f, want = verify_req(rng, 10 + k, 0, 3)
                v.sendall(f)
                assert W.read_msg(v) == want
            assert not any(e[:2] == ("end", PRUNE) for e in _trace(tmp_path))  # answered while the prune runs
            for c, rid, s in ((a, 1, stores[0]), (b, 2, stores[1])):
                name, m = W.read_msg(c)
                assert name == "sigverifyd_gossip_store_prune_reply" and m["req_id"] == rid and m["err"] == 0
                assert {k: m[k] for k in FIELDS} == fake_prune(s)[1]
            for c in (a, b, v):
                c.close()
    finally:
        for fd in fds:
            os.close(fd)
    assert [e[0] for e in _trace(tmp_path) if e[1] == PRUNE] == ["begin", "end", "begin", "end"]  # never two at once
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
    with serve(tmp_path, bins["daemon"], _env(tmp_path, 400)) as (proc, sock):
        time.sleep(0.2)
        base = nfds(proc)
        for f, s in zip(files, stores):
            fd = os.open(f, os.O_RDWR)
            c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
            c.connect(sock)
            socket.send_fds(c, [prune_frame(1, len(s))], [fd])
            os.close(fd)
            if f is files[0]:
                _wait(_begun(tmp_path, PRUNE))
            c.close()
        _wait(lambda: sum(1 for e in _trace(tmp_path) if e == ("end", PRUNE, "0")) == 2)
        assert back_to(proc, base) == base
        assert proc.poll() is None
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
def test_codec_round_trip(bins):
    """the C codec (sigverifyd_wiregen.h) and the Python one (sigverifyd_wire.py) give the same bytes for both messages and
    read each other's; a short or long message, or another type, is refused"""
    shim = ctypes.CDLL(bins["shim"])
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    shim.shim_towire_prune.restype = sz
    shim.shim_towire_prune.argtypes = [vp, sz, ctypes.c_uint64, ctypes.c_uint8, vp, ctypes.c_uint64]
    shim.shim_fromwire_prune.argtypes = [vp, sz, vp, vp]
    shim.shim_towire_prune_reply.restype = sz
    shim.shim_towire_prune_reply.argtypes = [vp, sz, vp]
    shim.shim_fromwire_prune_reply.argtypes = [vp, sz, vp]
    rng = np.random.default_rng(8)
    for _ in range(50):
        rid, has, ln = int(rng.integers(0, 2**63)), int(rng.integers(0, 2)), int(rng.integers(0, 2**64, dtype=np.uint64))
        chain = rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()
        body = prune_frame(rid, ln, chain)[4:] if has else W.encode("sigverifyd_gossip_store_prune", req_id=rid, has_chain=0,
                                                                     chain_hash=chain, len=ln)[4:]
        assert len(body) == 2 + 8 + 1 + 32 + 8 and body[:2] == (3010).to_bytes(2, "big")
        out = (ctypes.c_uint8 * 64)()
        cb = (ctypes.c_uint8 * 32).from_buffer_copy(chain)
        n = shim.shim_towire_prune(out, 64, rid, has, cb, ln)
        assert bytes(out[:n]) == body
        u, co = (ctypes.c_uint64 * 3)(), ctypes.c_size_t()
        assert shim.shim_fromwire_prune(body, len(body), u, ctypes.byref(co)) == 1
        assert list(u) == [rid, has, ln] and body[co.value:co.value + 32] == chain
        assert W.decode(body) == ("sigverifyd_gossip_store_prune", dict(req_id=rid, has_chain=has, chain_hash=chain, len=ln))
        for bad in (body[:-1], body + b"\0", (3110).to_bytes(2, "big") + body[2:]):
            assert shim.shim_fromwire_prune(bad, len(bad), u, ctypes.byref(co)) == 0
        vals = [rid, int(rng.integers(0, 2**32)), int(rng.integers(0, 2**32)), int(rng.integers(0, 2**32))] + [
            int(x) for x in rng.integers(0, 2**64, size=12, dtype=np.uint64)]
        names = ["req_id", "err"] + FIELDS
        rb = W.encode("sigverifyd_gossip_store_prune_reply", **dict(zip(names, vals)))[4:]
        assert len(rb) == 2 + 8 + 3 * 4 + 12 * 8
        out = (ctypes.c_uint8 * 200)()
        n = shim.shim_towire_prune_reply(out, 200, (ctypes.c_uint64 * 16)(*vals))
        assert bytes(out[:n]) == rb
        v = (ctypes.c_uint64 * 16)()
        assert shim.shim_fromwire_prune_reply(rb, len(rb), v) == 1 and list(v) == vals
        assert W.decode(rb) == ("sigverifyd_gossip_store_prune_reply", dict(zip(names, vals)))
        for bad in (rb[:-1], rb + b"\0", (3010).to_bytes(2, "big") + rb[2:]):
            assert shim.shim_fromwire_prune_reply(bad, len(bad), v) == 0
