"""Time channeld's commitment_signed checks through the verifier subdaemon against a context per process; prints one JSON
line.

A request is what one commitment_signed makes channeld check: the commitment transaction (one input, its outputs
serialised, SIGHASH_ALL, signed with the funding key; check_tx_sig) and H HTLC transactions (SIGHASH_SINGLE|ANYONECANPAY,
signed with the one HTLC key; check_tx_sigs_bip143_batch), H in {0, 30, 483}.  For k client processes, k in
{1, 4, 16, 64}:
  daemon       each process sends the request as sigverifyd_tx messages (one per key) to one cln_sigverifyd and waits for
               the replies before it sends the next, as the drop-in's client mode does;
  in_process   each process has an engine context of its own and calls sv_verify_tx_host once per key.
Reported: requests/s over all processes, p50 / p99 latency per request, and the device memory one context takes
(cudaMemGetInfo around sv_create, and after its first request, in a fresh process).  The card's name and power limit are
read in the same run (nvidia-smi --query-gpu).  Every verdict is checked.  Fails if there is no GPU.

    python tools/measure_sigverifyd_tx.py [--clients 1,4,16,64] [--htlcs 0,30,483] [--requests 100]
"""
import argparse
import ctypes
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

FUNDING_SK, HTLC_SK = bytes([0x21]) * 32, bytes([0x22]) * 32


def workload(htlcs):
    """per H: the commitment transaction and the H HTLC transactions, each (record bytes, blob, key, signatures), all
    signatures valid (made over the device's sighashes in this process)"""
    import lightning_b200 as LB
    from tests import txsig
    eng = LB.SigVerifier(0)
    out = {}
    for h in htlcs:
        (ctx_, cblob), (htx, hblob) = txsig.commitment_signed(np.random.default_rng(h), h)
        ckey, csig = txsig.sign(eng, 1, FUNDING_SK, ctx_, cblob)
        parts = [(bytes(ctx_), cblob, ckey, csig.tobytes())]
        if h:
            hkey, hsig = txsig.sign(eng, 1, HTLC_SK, htx, hblob)
            parts.append((bytes(htx), hblob, hkey, hsig.tobytes()))
        out[h] = parts
    eng.close()
    return out


def _records(part):
    import lightning_b200 as LB
    raw, blob, key, sigs = part
    n = len(raw) // ctypes.sizeof(LB.SvTx)
    return (LB.SvTx * n).from_buffer_copy(raw), blob, key, np.frombuffer(sigs, np.uint8).reshape(n, 64)


def _client_daemon(sock_path, parts, nreq, start, q):
    import socket
    from lightning_b200 import sigverifyd_wire as W
    from tests import txsig
    frames = []
    for k, part in enumerate(parts):
        txs, blob, key, sigs = _records(part)
        frames.append(bytearray(txsig.request(k, 1, key, txs, blob, sigs)))
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    rid = 0

    def one():
        nonlocal rid
        ids = []
        for f in frames:
            rid += 1
            f[6:14] = rid.to_bytes(8, "big")  # after the length prefix and the message type
            c.sendall(f)
            ids.append(rid)
        for r in ids:
            name, v = W.read_msg(c)
            assert name == "sigverifyd_tx_reply" and v["req_id"] == r and all(v["verdicts"]), (name, r)

    for _ in range(5):  # warm-up
        one()
    start.wait()
    lat = []
    for _ in range(nreq):
        t0 = time.perf_counter()
        one()
        lat.append(time.perf_counter() - t0)
    c.close()
    q.put(lat)


def _client_inprocess(parts, nreq, start, q):
    import lightning_b200 as LB
    eng = LB.SigVerifier(0)
    calls = []
    for part in parts:
        txs, blob, key, sigs = _records(part)
        keys = np.frombuffer(key * len(txs), np.uint8).reshape(len(txs), len(key))
        calls.append((txs, blob, keys, sigs))

    def one():
        for txs, blob, keys, sigs in calls:
            assert eng.check_tx_sigs(1, txs, blob, keys, sigs).all()

    for _ in range(5):
        one()
    start.wait()
    lat = []
    for _ in range(nreq):
        t0 = time.perf_counter()
        one()
        lat.append(time.perf_counter() - t0)
    eng.close()
    q.put(lat)


def _run_clients(k, target, args):
    ctx = mp.get_context("spawn")
    start, q = ctx.Barrier(k + 1), ctx.Queue()
    procs = [ctx.Process(target=target, args=args + (start, q)) for _ in range(k)]
    for p in procs:
        p.start()
    try:
        start.wait(timeout=900)
        t0 = time.perf_counter()
        lats = [q.get(timeout=900) for _ in procs]
        wall = time.perf_counter() - t0
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    lat = np.concatenate([np.array(x) for x in lats]) * 1e3
    return {"clients": k, "requests": int(lat.size), "requests_per_s": round(lat.size / wall, 1),
            "p50_ms": round(float(np.percentile(lat, 50)), 3), "p99_ms": round(float(np.percentile(lat, 99)), 3)}


def _context_memory(parts, q):
    """device memory one process's engine context takes beyond the CUDA context itself: free memory before sv_create, after
    it, and after its first commitment_signed with 483 HTLCs"""
    import torch
    import lightning_b200 as LB
    before = torch.cuda.mem_get_info(0)[0]  # cudaMemGetInfo; creates the CUDA context first, so it is not counted
    eng = LB.SigVerifier(0)
    created = torch.cuda.mem_get_info(0)[0]
    for part in parts:
        txs, blob, key, sigs = _records(part)
        keys = np.frombuffer(key * len(txs), np.uint8).reshape(len(txs), len(key))
        eng.check_tx_sigs(1, txs, blob, keys, sigs)
    used = torch.cuda.mem_get_info(0)[0]
    eng.close()
    q.put({"after_sv_create_mib": round((before - created) / 2**20, 1), "after_first_request_mib": round((before - used) / 2**20, 1)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", default="1,4,16,64")
    ap.add_argument("--htlcs", default="0,30,483")
    ap.add_argument("--requests", type=int, default=100, help="timed requests per client process")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_tx: no GPU")
    name, power = card()
    clients = [int(x) for x in a.clients.split(",")]
    htlcs = [int(x) for x in a.htlcs.split(",")]
    work = workload(sorted(set(htlcs) | {483}))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_context_memory, args=(work[483], q))
    p.start()
    try:
        mem = q.get(timeout=600)
    finally:
        p.join(timeout=60)
        if p.is_alive():
            p.kill()
            p.join()
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
            for h in htlcs:
                for k in clients:
                    rows.append(dict(mode="daemon", htlcs=h, **_run_clients(k, _client_daemon, (sock_path, work[h], a.requests))))
        finally:
            daemon.terminate()
            try:
                daemon.wait(timeout=30)
            except subprocess.TimeoutExpired:
                daemon.kill()
                daemon.wait(timeout=30)
    for h in htlcs:
        for k in clients:
            rows.append(dict(mode="in_process", htlcs=h, **_run_clients(k, _client_inprocess, (work[h], a.requests))))
    print(json.dumps({"metric": "sigverifyd_tx", "gpu": name, "power_limit": power, "context_memory": mem, "rows": rows}))


if __name__ == "__main__":
    main()
