"""The verifier subdaemon (cln_sigverifyd) for tests: a fresh daemon on a socket of its own, connections to it and its
sigverifyd_stats counters."""
import contextlib
import os
import shutil
import socket
import subprocess
import tempfile
import time

import pytest

from lightning_b200 import build
from lightning_b200 import sigverifyd_wire as W


@contextlib.contextmanager
def running(tmp_path, binary=build.DAEMON, env=None):
    """runs `binary <dir>/sv.sock 0` and yields the socket path once it is up; the daemon is stopped (killed if need be)
    however the block ends.  The socket goes under tmp_path when its path fits a unix socket address (108 bytes with the
    NUL), else into a short directory of its own under /tmp, removed afterwards."""
    short = None
    if len(os.fsencode(tmp_path / "sv.sock")) >= 100:
        short = tempfile.mkdtemp(prefix="sv", dir="/tmp")
    sock_path = os.path.join(short or str(tmp_path), "sv.sock")
    proc = subprocess.Popen([binary, sock_path, "0"], stderr=subprocess.PIPE, env=env)
    try:
        for _ in range(600):
            if os.path.exists(sock_path) or proc.poll() is not None:
                break
            time.sleep(0.1)
        assert os.path.exists(sock_path), "daemon did not come up"
        yield sock_path
    finally:
        proc.terminate()
        try:
            proc.wait(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.wait(timeout=10)
        if short:
            shutil.rmtree(short, ignore_errors=True)


@pytest.fixture
def daemon(tmp_path):
    """a fresh cln_sigverifyd on a socket under tmp_path"""
    with running(tmp_path) as sock_path:
        yield sock_path


def connect(path):
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.settimeout(120)
    c.connect(path)
    return c


def stats(path):
    c = connect(path)
    c.sendall(W.encode("sigverifyd_stats", req_id=77))
    name, st = W.read_msg(c)
    c.close()
    assert name == "sigverifyd_stats_reply"
    return st
