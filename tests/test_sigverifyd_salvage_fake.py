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
from tests import gossip_store_salvage as sv
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_salvage_host import damage_classes, with_uuid
from tests.test_sigverifyd_fake_engine import verify_req
from tests.test_sigverifyd_prune_fake import (FIELDS, HE, MAX_PRUNE_STORE, PRUNE, ROOT, STORE_FD, TESTNET, _begun, _env,
                                              _trace, _wait, back_to, fake_prune, make_store, nfds, prune_frame, serve)
from tests.test_sigverifyd_repair_fake import cut_rule

SALVAGE_FD = os.path.join(build.CSRC, "gossip_salvage_fd.c")


def _run(args):
    r = subprocess.run(args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    d = tmp_path_factory.mktemp("salvage_fake")
    salv_o = str(d / "fake_engine_salvage.o")
    _run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-c",
          os.path.join(HE, "fake_engine_salvage.cpp"), "-o", salv_o])
    out = dict(daemon=str(d / "cln_sigverifyd"), inproc=str(d / "libdropin_inproc.so"), client=str(d / "libdropin_client.so"))
    engine = [os.path.join(HE, "fake_engine_prune.c"), STORE_FD, SALVAGE_FD, salv_o, "-lstdc++"]
    _run(["gcc"] + build.DAEMON_CFLAGS + [os.path.join(build.CSRC, "sigverifyd.c"), os.path.join(HE, "fake_engine_timed.c")] +
         engine + ["-o", out["daemon"]])
    dropin = ["gcc"] + build.DROPIN_CFLAGS + ["-shared", os.path.join(build.CSRC, "cln_dropin.c"),
                                              os.path.join(HE, "fake_engine.c")] + engine
    _run(dropin + ["-o", out["inproc"]])
    _run(dropin + ["-DFAKE_ENGINE_NO_CONTEXT", "-o", out["client"]])  # its sv_create aborts
    return out


CLIENT = r"""
import ctypes, json, os, sys
from lightning_b200.engine import SvGossipPruneSummary, SvGossipSalvageSummary
lib = ctypes.CDLL(sys.argv[1], use_errno=True)
lib.gossip_store_salvage.restype = ctypes.c_bool
lib.gossip_store_salvage.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p, ctypes.POINTER(SvGossipPruneSummary),
                                     ctypes.POINTER(SvGossipSalvageSummary), ctypes.POINTER(ctypes.c_uint64)]
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
    s, v, n = SvGossipPruneSummary(), SvGossipSalvageSummary(), ctypes.c_uint64(12345)
    chain = bytes.fromhex(c["chain"]) if c["chain"] else None
    ok = lib.gossip_store_salvage(fd, c["len"], chain, ctypes.byref(s), ctypes.byref(v), ctypes.byref(n))
    e = ctypes.get_errno()
    if c["kind"] != "closed":
        os.close(fd)
    if c["kind"] == "pipe":
        os.close(w)
    out.append([ok, 0 if ok else e, {f: getattr(s, f) for f, _ in s._fields_} if ok else None,
                {f: getattr(v, f) for f, _ in v._fields_} if ok else None, n.value if ok else None])
print(json.dumps(out))
"""


def run_client(tmp_path, lib, mode, cases, pass_fds=(), check=True):
    """each case's [ok, errno, repair summary, salvage summary, new_len] from a process of its own"""
    path = tmp_path / ("cases%d.json" % time.monotonic_ns())
    path.write_text(json.dumps(cases))
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", CLIENT, lib, mode, str(path)], env=env, capture_output=True, text=True,
                       timeout=300, pass_fds=pass_fds)
    if check:
        assert r.returncode == 0, r.stderr[-3000:]
        return json.loads(r.stdout)
    return r


def case(path, length=None, chain=TESTNET, kind="rw"):
    return dict(kind=kind, path=str(path), len=os.path.getsize(path) if length is None else length,
                chain=chain.hex() if chain else None)


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
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        got["sock"] = run_client(tmp_path, bins["client"], "sock:" + sock, cases("sock"))
        assert proc.poll() is None
    parent, child = socket.socketpair()
    dm = subprocess.Popen([bins["daemon"], "--fd", str(child.fileno()), "0"], pass_fds=(child.fileno(),), env=_env(tmp_path),
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
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        time.sleep(0.2)
        base = nfds(proc)
        got = run_client(tmp_path, bins["client"], "sock:" + sock, cases)
        assert proc.poll() is None
        assert back_to(proc, base) == base
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
    with serve(tmp_path, bins["daemon"], _env(tmp_path)) as (proc, sock):
        time.sleep(0.2)
        base = nfds(proc)
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
        assert back_to(proc, base) == base
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
        with serve(tmp_path, bins["daemon"], _env(tmp_path, 600)) as (proc, sock):
            a, b, vv = (socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) for _ in range(3))
            for c in (a, b, vv):
                c.settimeout(60)
                c.connect(sock)
            socket.send_fds(a, [salvage_frame(1, len(st[0]))], [fds[0]])
            _wait(_begun(tmp_path, PRUNE))
            socket.send_fds(b, [prune_frame(2, len(st[1]))], [fds[1]])
            for k in range(3):
                f, want = verify_req(rng, 10 + k, 0, 3)
                vv.sendall(f)
                assert W.read_msg(vv) == want
            assert not any(e[:2] == ("end", PRUNE) for e in _trace(tmp_path))
            name, m = W.read_msg(a)
            assert name == "sigverifyd_gossip_store_salvage_reply" and m["err"] == 0 and m["restored"] == 1
            name, m = W.read_msg(b)
            assert name == "sigverifyd_gossip_store_prune_reply" and m["err"] == 0
            for c in (a, b, vv):
                c.close()
    finally:
        for fd in fds:
            os.close(fd)
    assert [e[0] for e in _trace(tmp_path) if e[1] == PRUNE] == ["begin", "end", "begin", "end"]
    assert files[0].read_bytes() == fake_salvage(st[0])[0]
    assert files[1].read_bytes() == fake_prune(st[1])[0]
