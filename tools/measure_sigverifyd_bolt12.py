"""Time BOLT12 checks through the verifier subdaemon and the one-pass tagged call on the GPU; prints one JSON line.

(a) Requests per second and per-request latency (p50 / p99) for k = 1, 4 and 16 client processes, each sending one-stream
    sigverifyd_bolt12 requests to one cln_sigverifyd and waiting for each reply before sending the next (as a plugin's
    bolt12_check_signature does).  Against it: the same k processes each with an engine context of its own, calling
    sv_verify_bolt12_host on one stream per call (what every plugin does today when it links the drop-in).
(b) One pass mixing 2 or 5 tags at 64 and 8,192 streams: wall time of one sv_verify_bolt12_tagged_host call against one
    sv_verify_bolt12_host call per tag over the same streams (host clock around work that ends in a synchronise; median).

Streams: the fixture's signed invoice-sized streams (tools/measure_bolt12.py's workload).  The card's name and power limit
are read in the same run.  Fails if there is no GPU.

    python tools/measure_sigverifyd_bolt12.py [--clients 1,4,16] [--requests 400] [--sizes 64,8192]
"""
import argparse
import json
import multiprocessing as mp
import os
import socket
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_bolt12 import card, workload  # noqa: E402
from tests import bolt12  # noqa: E402

MADE_UP = [(b"offer", b"signature"), (b"invoice", b"payer_signature"), (b"invoice_request", b"payer_signature")]


def _stream(k):
    """the k-th workload stream (same bytes in every mode) and its key and signature"""
    fx = bolt12.load_fixture()
    blob, off, ln, xonly, sig, want = workload(fx, 64, np.random.default_rng(7))
    i = k % 64
    return blob[int(off[i]):int(off[i]) + int(ln[i])].tobytes(), xonly[i], sig[i], int(want[i])


def _client_daemon(sock_path, nreq, start, q):
    from lightning_b200 import sigverifyd_wire as W
    s, x, g, want = _stream(os.getpid())
    mn, fn = bolt12.NAMES[0]
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    frame = lambda rid: W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn,
                                 n=1, lens=[len(s)], bloblen=len(s), blob=s, xonly=x.tobytes(), sigs=g.tobytes(),
                                 want_sighash=0)
    for r in range(20):  # warm-up
        c.sendall(frame(r))
        W.read_msg(c)
    start.wait()
    lat = []
    for r in range(nreq):
        t0 = time.perf_counter()
        c.sendall(frame(1000 + r))
        name, v = W.read_msg(c)
        lat.append(time.perf_counter() - t0)
        assert name == "sigverifyd_bolt12_reply" and v["req_id"] == 1000 + r
        st = v["status"][0]
        assert (-1 if st == 255 else st) == want
    c.close()
    q.put(lat)


def _client_inprocess(nreq, start, q):
    import lightning_b200 as LB
    s, x, g, want = _stream(os.getpid())
    mn, fn = bolt12.NAMES[0]
    eng = LB.SigVerifier(0)
    blob = np.frombuffer(s, np.uint8)
    off, ln = np.zeros(1, np.uint64), np.array([len(s)], np.uint32)
    for _ in range(20):
        eng.verify_bolt12_spans(mn, fn, blob, off, ln, x[None], g[None])
    start.wait()
    lat = []
    for _ in range(nreq):
        t0 = time.perf_counter()
        got = eng.verify_bolt12_spans(mn, fn, blob, off, ln, x[None], g[None])
        lat.append(time.perf_counter() - t0)
        assert got[0] == want
    eng.close()
    q.put(lat)


def _run_clients(k, target, args):
    ctx = mp.get_context("spawn")
    start, q = ctx.Barrier(k + 1), ctx.Queue()
    procs = [ctx.Process(target=target, args=args + (start, q)) for _ in range(k)]
    for p in procs:
        p.start()
    try:
        start.wait(timeout=600)
        t0 = time.perf_counter()
        lats = [q.get(timeout=600) for _ in procs]
        wall = time.perf_counter() - t0
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    lat = np.concatenate([np.array(x) for x in lats]) * 1e3
    return {"clients": k, "requests": int(lat.size), "requests_per_s": round(lat.size / wall, 1),
            "p50_ms": round(float(np.percentile(lat, 50)), 4), "p99_ms": round(float(np.percentile(lat, 99)), 4)}


def part_a(clients, nreq):
    from lightning_b200 import build
    rows = []
    with tempfile.TemporaryDirectory() as d:
        sock_path = os.path.join(d, "sv.sock")
        daemon = subprocess.Popen([build.DAEMON, sock_path, "0"], stderr=subprocess.DEVNULL)
        try:
            for _ in range(600):
                if os.path.exists(sock_path):
                    break
                time.sleep(0.1)
            for k in clients:
                rows.append(dict(mode="daemon", **_run_clients(k, _client_daemon, (sock_path, nreq))))
        finally:
            daemon.terminate()
            daemon.wait(timeout=30)
    for k in clients:
        rows.append(dict(mode="in_process", **_run_clients(k, _client_inprocess, (nreq,))))
    return rows


def part_b(sizes, reps):
    import lightning_b200 as LB
    eng = LB.SigVerifier(0)
    fx = bolt12.load_fixture()
    rows = []
    for ntags in (2, 5):
        tags = (list(bolt12.NAMES) + MADE_UP)[:ntags]
        for n in sizes:
            blob, off, ln, xonly, sig, _ = workload(fx, n, np.random.default_rng(7))
            tag_of = (np.arange(n) % ntags).astype(np.uint32)
            sel = [np.nonzero(tag_of == t)[0] for t in range(ntags)]
            one = lambda: eng.verify_bolt12_tagged(tags, tag_of, blob, off, ln, xonly, sig, want_sighash=True)
            per_tag = lambda: [eng.verify_bolt12_spans(*tags[t], blob, off[s], ln[s], xonly[s], sig[s], want_sighash=True)
                               for t, s in enumerate(sel)]
            st1, sh1 = one()
            parts = per_tag()
            for t, s in enumerate(sel):  # the same answers both ways
                assert np.array_equal(st1[s], parts[t][0]) and np.array_equal(sh1[s], parts[t][1])
            for _ in range(3):
                one()
                per_tag()
            t_one, t_per = [], []
            for _ in range(reps):  # alternate the two so both see the same machine state
                t0 = time.perf_counter()
                one()
                t_one.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                per_tag()
                t_per.append(time.perf_counter() - t0)
            rows.append({"tags": ntags, "n": n, "one_call_ms": round(statistics.median(t_one) * 1e3, 4),
                         "per_tag_calls_ms": round(statistics.median(t_per) * 1e3, 4)})
    eng.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", default="1,4,16")
    ap.add_argument("--requests", type=int, default=400, help="timed requests per client process")
    ap.add_argument("--sizes", default="64,8192")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_bolt12: no GPU")
    name, power = card()
    b = part_b([int(s) for s in a.sizes.split(",")], a.reps)
    rows = part_a([int(s) for s in a.clients.split(",")], a.requests)
    print(json.dumps({"metric": "sigverifyd_bolt12", "gpu": name, "power_limit": power, "clients": rows, "tagged": b}))


if __name__ == "__main__":
    main()
