"""Time one client process that keeps a window of requests in flight to the verifier subdaemon against k blocking client
processes; prints one JSON line.

The drop-in's _start functions (cln_dropin.h) let one process keep many requests at the daemon, which serves everything it
has read in one engine call per type.  This tool sends the same frames those functions send:
  bolt12  one-stream sigverifyd_bolt12 requests (the fixture's signed invoice-sized streams, as
          tools/measure_sigverifyd_bolt12.py sends them: what bolt12_check_signature_start sends);
  tx      commitment_signed-shaped sigverifyd_tx requests with H HTLCs, H in {0, 30} (tools/measure_sigverifyd_tx.py's
          workload: the commitment transaction, then the H HTLC transactions as one request).
Modes, for each workload:
  window   ONE process on one connection keeps w units in flight, w in {1, 4, 16, 64}: it sends a new unit whenever one
           is answered, as an event loop that starts a ticket per check does;
  blocking k processes, k in {1, 4, 16}, each waiting for its unit's replies before sending the next (the blocking
           drop-in functions).
Reported: units/s over the run and p50 / p99 latency per unit (send of its first frame to its last reply).  Every verdict is
checked.  The card's name and power limit are read in the same run.  Fails if there is no GPU.

    python tools/measure_sigverifyd_async.py [--windows 1,4,16,64] [--clients 1,4,16] [--requests 2000]
"""
import argparse
import json
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

import measure_sigverifyd_bolt12 as MB  # noqa: E402
import measure_sigverifyd_tx as MT  # noqa: E402
from measure_bolt12 import card  # noqa: E402


def bolt12_units():
    """one unit: one sigverifyd_bolt12 frame; its check: the fixture's status"""
    from lightning_b200 import sigverifyd_wire as W
    from tests import bolt12
    units = []
    for k in range(64):
        s, x, g, want = MB._stream(k)
        mn, fn = bolt12.NAMES[0]
        f = W.encode("sigverifyd_bolt12", req_id=0, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn, n=1,
                     lens=[len(s)], bloblen=len(s), blob=s, xonly=x.tobytes(), sigs=g.tobytes(), want_sighash=0)
        units.append(([bytearray(f)], lambda v, want=want: (-1 if v["status"][0] == 255 else v["status"][0]) == want))
    return units


def tx_units(parts):
    """one unit: the frames of one commitment_signed; every verdict must be 1"""
    from tests import txsig
    frames = []
    for k, part in enumerate(parts):
        txs, blob, key, sigs = MT._records(part)
        frames.append(bytearray(txsig.request(k, 1, key, txs, blob, sigs)))
    return [(frames, lambda v: all(v["verdicts"]))]


def window_client(sock_path, units, w, nunits):
    """one connection keeping w units in flight; returns (wall seconds, per-unit latencies)"""
    from lightning_b200 import sigverifyd_wire as W
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    rid, flight, lat = 0, [], []  # flight: per unit in flight, [start time, checks of its outstanding replies]

    def send(u):
        nonlocal rid
        frames, check = units[u % len(units)]
        ids = []
        t0 = time.perf_counter()
        for f in frames:
            rid += 1
            f[6:14] = rid.to_bytes(8, "big")  # after the length prefix and the message type
            c.sendall(f)
            ids.append(rid)
        flight.append([t0, [(r, check) for r in ids]])

    def run(n, record):
        sent = done = 0
        while done < n:
            while sent < n and len(flight) < w:
                send(sent)
                sent += 1
            name, v = W.read_msg(c)
            r, check = flight[0][1].pop(0)
            assert name.endswith("_reply") and v["req_id"] == r and check(v), (name, r)
            if not flight[0][1]:
                if record:
                    lat.append(time.perf_counter() - flight[0][0])
                flight.pop(0)
                done += 1

    run(min(200, nunits), False)  # warm-up
    t0 = time.perf_counter()
    run(nunits, True)
    wall = time.perf_counter() - t0
    c.close()
    return wall, lat


def _row(n, wall, lat):
    lat = np.array(lat) * 1e3
    return {"requests": int(n), "requests_per_s": round(n / wall, 1), "p50_ms": round(float(np.percentile(lat, 50)), 3),
            "p99_ms": round(float(np.percentile(lat, 99)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", default="1,4,16,64")
    ap.add_argument("--clients", default="1,4,16")
    ap.add_argument("--htlcs", default="0,30")
    ap.add_argument("--requests", type=int, default=2000, help="timed units of the window client")
    ap.add_argument("--blocking-requests", type=int, default=200, help="timed units per blocking client process")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_async: no GPU")
    name, power = card()
    windows = [int(x) for x in a.windows.split(",")]
    clients = [int(x) for x in a.clients.split(",")]
    htlcs = [int(x) for x in a.htlcs.split(",")]
    work = MT.workload(htlcs)
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
            loads = [("bolt12", None, bolt12_units())] + [("tx", h, tx_units(work[h])) for h in htlcs]
            for load, h, units in loads:
                for w in windows:
                    rows.append(dict(load=load, htlcs=h, mode="window", window=w,
                                     **_row(a.requests, *window_client(sock_path, units, w, a.requests))))
                for k in clients:
                    if load == "bolt12":
                        r = MB._run_clients(k, MB._client_daemon, (sock_path, a.blocking_requests))
                    else:
                        r = MT._run_clients(k, MT._client_daemon, (sock_path, work[h], a.blocking_requests))
                    rows.append(dict(load=load, htlcs=h, mode="blocking", **r))
        finally:
            daemon.terminate()
            try:
                daemon.wait(timeout=30)
            except subprocess.TimeoutExpired:
                daemon.kill()
                daemon.wait(timeout=30)
    print(json.dumps({"metric": "sigverifyd_async", "gpu": name, "power_limit": power, "rows": rows}))


if __name__ == "__main__":
    main()
