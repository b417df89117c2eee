"""Time BOLT11 checks (bolt11_decode's signature step) through the verifier subdaemon; prints one JSON line.

Invoices: the fixture's invoices Core Lightning accepts (tests/golden/bolt11_vectors.npz), with and without an `n` field in
the fixture's own proportion, which the output states.  Every client takes them in turn, one invoice per request.
(a) Many processes: k = 1, 4 and 16 client processes, each sending one-invoice sigverifyd_bolt11 requests to one
    cln_sigverifyd and waiting for each reply before sending the next (as bolt11_check_signature does in a plugin or in
    lightningd).  Against it: the same k processes each with an engine context of its own, calling sv_verify_bolt11_host
    on one invoice per call (what every process does when it links the drop-in in process).
(b) One process with a window: one connection keeps w = 1, 4, 16 and 64 one-invoice requests in flight, sending a new one
    whenever one is answered (as an event loop does with bolt11_check_signature_start).
Reported: requests/s over the run and p50 / p99 latency per request.  Every status and receiver id is checked against the
fixture.  The card's name and power limit are read in the same run.  Fails if there is no GPU.

    python tools/measure_sigverifyd_bolt11.py [--clients 1,4,16] [--windows 1,4,16,64] [--requests 400]
"""
import argparse
import json
import multiprocessing as mp
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_bolt11 import card  # noqa: E402
from tests import bolt11  # noqa: E402


def has_n(inv):
    """whether the invoice carries a 53-word `n` field (its key is verified against; without one it is recovered)"""
    s = inv.split(b"\0", 1)[0].decode().lower()
    words = [bolt11.CHARSET.index(ch) for ch in s[s.rindex("1") + 1:-6]]
    at = 7  # the timestamp
    while at + 3 <= len(words) - 104:  # the signature's 104 words end the data part
        typ, ln = words[at], words[at + 1] * 32 + words[at + 2]
        if typ == bolt11.CHARSET.index("n") and ln == 53:
            return True
        at += 3 + ln
    return False


def invoices():
    """the accepted invoices [(bytes, receiver id 33 bytes)] and how many carry an `n` field"""
    fx = bolt11.load_fixture()
    good = np.nonzero((fx["expected"] == 1) & ((fx["ret"] & 1) == 1))[0]
    invs = bolt11.invoices(fx)
    return [(invs[i], fx["node"][i].tobytes()) for i in good], sum(has_n(invs[i]) for i in good)


def _frame(inv, rid):
    from lightning_b200 import sigverifyd_wire as W
    return W.encode("sigverifyd_bolt11", req_id=rid, n=1, lens=[len(inv)], bloblen=len(inv), blob=inv)


def _checked(v, rid, node):
    return v["req_id"] == rid and v["status"] == b"\x01" and v["node_ids"] == node


def _client_daemon(sock_path, nreq, start, q):
    from lightning_b200 import sigverifyd_wire as W
    invs, _ = invoices()
    first = os.getpid()
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    for r in range(20):  # warm-up
        c.sendall(_frame(invs[r % len(invs)][0], r))
        W.read_msg(c)
    start.wait()
    lat = []
    for r in range(nreq):
        inv, node = invs[(first + r) % len(invs)]
        t0 = time.perf_counter()
        c.sendall(_frame(inv, 1000 + r))
        name, v = W.read_msg(c)
        lat.append(time.perf_counter() - t0)
        assert name == "sigverifyd_bolt11_reply" and _checked(v, 1000 + r, node), (name, r)
    c.close()
    q.put(lat)


def _client_inprocess(nreq, start, q):
    import lightning_b200 as LB
    invs, _ = invoices()
    first = os.getpid()
    eng = LB.SigVerifier(0)
    off, ln = np.zeros(1, np.uint64), np.zeros(1, np.uint32)

    def one(inv):
        ln[0] = len(inv)
        return eng.verify_bolt11_spans(np.frombuffer(inv, np.uint8), off, ln)

    for r in range(20):
        one(invs[r % len(invs)][0])
    start.wait()
    lat = []
    for r in range(nreq):
        inv, node = invs[(first + r) % len(invs)]
        t0 = time.perf_counter()
        st, nd, _ = one(inv)
        lat.append(time.perf_counter() - t0)
        assert st[0] == 1 and nd[0].tobytes() == node
    eng.close()
    q.put(lat)


def _row(n, wall, lat):
    lat = np.asarray(lat) * 1e3
    return {"requests": int(n), "requests_per_s": round(n / wall, 1), "p50_ms": round(float(np.percentile(lat, 50)), 4),
            "p99_ms": round(float(np.percentile(lat, 99)), 4)}


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
    lat = np.concatenate([np.array(x) for x in lats])
    return dict(clients=k, **_row(lat.size, wall, lat))


def window_client(sock_path, w, nreq):
    """one connection keeping w one-invoice requests in flight; returns (wall seconds, per-request latencies)"""
    from lightning_b200 import sigverifyd_wire as W
    invs, _ = invoices()
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    rid, flight, lat = 0, [], []  # flight: (rid, send time, receiver id) in request order

    def run(n, record):
        nonlocal rid
        sent = done = 0
        while done < n:
            while sent < n and len(flight) < w:
                inv, node = invs[rid % len(invs)]
                rid += 1
                flight.append((rid, time.perf_counter(), node))
                c.sendall(_frame(inv, rid))
                sent += 1
            name, v = W.read_msg(c)
            r, t0, node = flight.pop(0)
            assert name == "sigverifyd_bolt11_reply" and _checked(v, r, node), (name, r)
            if record:
                lat.append(time.perf_counter() - t0)
            done += 1

    run(min(200, nreq), False)  # warm-up
    t0 = time.perf_counter()
    run(nreq, True)
    wall = time.perf_counter() - t0
    c.close()
    return wall, lat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clients", default="1,4,16")
    ap.add_argument("--windows", default="1,4,16,64")
    ap.add_argument("--requests", type=int, default=400, help="timed requests per blocking client process")
    ap.add_argument("--window-requests", type=int, default=2000, help="timed requests of the window client")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_bolt11: no GPU")
    name, power = card()
    invs, with_n = invoices()
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
                rows.append(dict(mode="daemon", **_run_clients(k, _client_daemon, (sock_path, a.requests))))
            for w in [int(x) for x in a.windows.split(",")]:
                rows.append(dict(mode="window", window=w, **_row(a.window_requests,
                                                                 *window_client(sock_path, w, a.window_requests))))
        finally:
            daemon.terminate()
            try:
                daemon.wait(timeout=30)
            except subprocess.TimeoutExpired:
                daemon.kill()
                daemon.wait(timeout=30)
    for k in clients:
        rows.append(dict(mode="in_process", **_run_clients(k, _client_inprocess, (a.requests,))))
    print(json.dumps({"metric": "sigverifyd_bolt11", "gpu": name, "power_limit": power, "invoices": len(invs),
                      "with_n": with_n, "without_n": len(invs) - with_n,
                      "chars_per_invoice": round(float(np.mean([len(s) for s, _ in invs])), 1), "rows": rows}))


if __name__ == "__main__":
    main()
