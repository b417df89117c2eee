"""Time sha256_double and pubkey_from_der through the verifier subdaemon against a context per process; prints one JSON
line.

What client mode costs every fromwire_pubkey and bitcoin_txid is the latency of one call through the daemon, so the
workloads are single calls of the drop-in library (libcln_sigverify.so through ctypes), as a CLN daemon makes them:
sha256_double on a 32-, 174- (a featureless channel_announcement's signed part) and 4,000-byte buffer, and
pubkey_from_der on a valid 33-byte key.  For k client processes, k in {1, 4, 16}:
  daemon       each process calls cln_sigverify_connect() to one cln_sigverifyd, then calls the function in a loop; every
               call is one request and one reply;
  in_process   each process has an engine context of its own (created by its first call, before the timed window).
Reported per workload: calls/s over all processes and p50 / p99 latency per call (host clock around each call).  The
card's name and power limit are read in the same run (nvidia-smi --query-gpu).  Every answer is checked against hashlib /
the key's known point.  Fails if there is no GPU.

    python tools/measure_sigverifyd_misc.py [--clients 1,4,16] [--calls 2000]
"""
import argparse
import ctypes
import hashlib
import json
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_bolt12 import card  # noqa: E402

WORKLOADS = ["sha256_double_32", "sha256_double_174", "sha256_double_4000", "pubkey_from_der"]
KEY_SK = bytes([0x41]) * 32


def _client(sock_path, ncalls, start, q):
    """one client process: for each workload, wait for the others, then time ncalls single calls"""
    from lightning_b200 import engine
    from tests import ecc
    lib = ctypes.CDLL(engine.LIB_PATH)
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.sha256_double.argtypes = [vp, vp, sz]
    lib.pubkey_from_der.restype = ctypes.c_bool
    lib.pubkey_from_der.argtypes = [vp, sz, vp]
    if sock_path and lib.cln_sigverify_connect(sock_path.encode()) != 0:
        raise RuntimeError("cannot connect to " + sock_path)
    pub33, xy = ecc.pubkey_create(KEY_SK)
    key = (ctypes.c_uint8 * 33).from_buffer_copy(pub33)
    want_pk = xy[31::-1] + xy[:31:-1]  # struct pubkey: x and y as little-endian limbs
    rng = np.random.default_rng(os.getpid())
    out = (ctypes.c_uint8 * 64)()
    for w in WORKLOADS:
        if w == "pubkey_from_der":
            def call():
                if not lib.pubkey_from_der(key, 33, out) or bytes(out) != want_pk:
                    raise AssertionError("pubkey_from_der")
        else:
            data = bytes(rng.integers(0, 256, size=int(w.rsplit("_", 1)[1]), dtype=np.uint8))
            buf = (ctypes.c_uint8 * len(data)).from_buffer_copy(data)
            want = hashlib.sha256(hashlib.sha256(data).digest()).digest()

            def call():
                lib.sha256_double(out, buf, len(data))
                if bytes(out[:32]) != want:
                    raise AssertionError("sha256_double")
        for _ in range(50):  # warm-up; in_process: the context is created here
            call()
        start.wait()
        lat = np.empty(ncalls)
        for i in range(ncalls):
            t0 = time.perf_counter()
            call()
            lat[i] = time.perf_counter() - t0
        q.put(lat)
    lib.cln_sigverify_shutdown()


def _run_clients(k, sock_path, ncalls):
    ctx = mp.get_context("spawn")
    start, q = ctx.Barrier(k + 1), ctx.Queue()
    procs = [ctx.Process(target=_client, args=(sock_path, ncalls, start, q)) for _ in range(k)]
    for p in procs:
        p.start()
    rows = []
    try:
        for w in WORKLOADS:
            start.wait(timeout=900)
            t0 = time.perf_counter()
            lats = [q.get(timeout=900) for _ in procs]
            wall = time.perf_counter() - t0
            lat = np.concatenate(lats) * 1e3
            rows.append({"mode": "daemon" if sock_path else "in_process", "workload": w, "clients": k,
                         "calls": int(lat.size), "calls_per_s": round(lat.size / wall, 1),
                         "p50_ms": round(float(np.percentile(lat, 50)), 4),
                         "p99_ms": round(float(np.percentile(lat, 99)), 4)})
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    if any(p.exitcode for p in procs):
        raise RuntimeError("a client process failed")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", default="1,4,16")
    ap.add_argument("--calls", type=int, default=2000, help="timed calls per client process and workload")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_misc: no GPU")
    name, power = card()
    clients = [int(x) for x in a.clients.split(",")]
    from lightning_b200 import build
    rows = []
    with tempfile.TemporaryDirectory() as d:
        sock_path = os.path.join(d, "sv.sock")
        daemon = subprocess.Popen([build.DAEMON, sock_path, "0"], stderr=subprocess.DEVNULL)
        try:
            for _ in range(600):
                if os.path.exists(sock_path) or daemon.poll() is not None:
                    break
                time.sleep(0.1)
            assert os.path.exists(sock_path), "daemon did not come up"
            for k in clients:
                rows += _run_clients(k, sock_path, a.calls)
        finally:
            daemon.terminate()
            try:
                daemon.wait(timeout=30)
            except subprocess.TimeoutExpired:
                daemon.kill()
                daemon.wait(timeout=30)
    for k in clients:
        rows += _run_clients(k, None, a.calls)
    print(json.dumps({"metric": "sigverifyd_misc", "gpu": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
