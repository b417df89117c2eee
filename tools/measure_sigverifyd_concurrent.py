"""Time the verifier subdaemon with its two engine workers against the parent revision's single-threaded daemon, in one
run, alternating between the two for every row; prints one JSON line.

  (a) channeld's commitment_signed checks (tools/measure_sigverifyd_tx.py's client: H = 0 and 30, k = 1, 4, 16, 64
      processes) and plugins' one-stream BOLT12 checks (tools/measure_sigverifyd_bolt12.py's client: k = 1, 4, 16).
  (b) a gossipd-like process sends the committed gossip subset tiled 53 times as sigverifyd_gossip_burst requests back to
      back while k = 1, 4, 16 channeld-like processes (H = 30) run: their requests/s and p50 / p99 latency, and the bursts
      served in that time.
Also the device memory each daemon holds once it has served a request (free memory on the card before it starts, and
after), so the difference between the two is the second worker's context.  The card's name and power limit are read in
the same run.  Every verdict is checked.  Fails if there is no GPU.

The parent daemon is compiled from the parent revision's sigverifyd.c (--parent-source FILE, or --parent-rev REV read
with git) against this tree's headers and engine library, into a temporary directory.

    python tools/measure_sigverifyd_concurrent.py --parent-source FILE | --parent-rev REV [--requests 100] [--rounds 1]
"""
import argparse
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
from measure_sigverifyd_bolt12 import _client_daemon as bolt12_client  # noqa: E402
from measure_sigverifyd_tx import _client_daemon as tx_client  # noqa: E402
from measure_sigverifyd_tx import _run_clients, workload  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def build_parent(source, out):
    """the parent revision's daemon: its source compiled in lightning_b200/csrc (so its includes resolve there) and
    linked against the engine library built in this tree"""
    from lightning_b200 import build
    r = subprocess.run(["gcc"] + build.DAEMON_CFLAGS + ["-x", "c", "-", "-o", out, "-L" + os.path.dirname(build.LIB),
                        "-lcln_sigverify", "-Wl,-rpath," + os.path.dirname(build.LIB)], input=source, cwd=build.CSRC,
                       capture_output=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (parent sigverifyd.c) failed:\n" + r.stderr.decode())


class Daemon:
    """one cln_sigverifyd on a socket in a temporary directory, with the device memory it took"""

    def __init__(self, binary, d):
        import torch
        self.sock = os.path.join(d, "sv.sock")
        free0 = torch.cuda.mem_get_info(0)[0]
        self.p = subprocess.Popen([binary, self.sock, "0"], stderr=subprocess.DEVNULL)
        for _ in range(600):
            if os.path.exists(self.sock) or self.p.poll() is not None:
                break
            time.sleep(0.1)
        assert os.path.exists(self.sock), "daemon did not come up"
        _one_tx(self.sock)
        self.mib = round((free0 - torch.cuda.mem_get_info(0)[0]) / 2**20, 1)

    def close(self):
        self.p.terminate()
        try:
            self.p.wait(timeout=30)
        except subprocess.TimeoutExpired:
            self.p.kill()
            self.p.wait(timeout=30)


def _one_tx(sock_path):
    import socket
    from lightning_b200 import sigverifyd_wire as W
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    c.sendall(W.encode("sigverifyd_verify", req_id=1, kind=2, n=1, hashes=bytes(32), keylen=32, keys=bytes(32), sigs=bytes(64)))
    assert W.read_msg(c)[0] == "sigverifyd_verify_reply"
    c.close()


def _gossipd(sock_path, ready, stop, q):
    """x53 bursts back to back until stop is set: (bursts answered, their latencies)"""
    import socket
    from lightning_b200 import sigverifyd_wire as W
    from tests import gossip
    msgs = gossip.load_subset() * 53
    blob = b"".join(msgs)
    frame = bytearray(W.encode("sigverifyd_gossip_burst", req_id=0, chain_hash=TESTNET, n=len(msgs),
                               lens=[len(m) for m in msgs], signer_kind=bytes(len(msgs)), signers=bytes(33 * len(msgs)),
                               bloblen=len(blob), blob=blob))
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    ready.set()
    lat, rid = [], 0
    while not stop.is_set():
        rid += 1
        frame[6:14] = rid.to_bytes(8, "big")
        t0 = time.perf_counter()
        c.sendall(frame)
        name, v = W.read_msg(c)
        lat.append(time.perf_counter() - t0)
        assert name == "sigverifyd_gossip_burst_reply" and v["req_id"] == rid and not any(v["status"])
    c.close()
    q.put(lat)


def _with_bursts(sock_path, k, parts, nreq):
    ctx = mp.get_context("spawn")
    ready, stop, q = ctx.Event(), ctx.Event(), ctx.Queue()
    g = ctx.Process(target=_gossipd, args=(sock_path, ready, stop, q))
    g.start()
    try:
        assert ready.wait(timeout=600)
        time.sleep(0.5)  # the first burst is on its way
        t0 = time.perf_counter()
        row = _run_clients(k, tx_client, (sock_path, parts, nreq))
        wall = time.perf_counter() - t0
        stop.set()
        lat = np.array(q.get(timeout=600)) * 1e3
    finally:
        g.join(timeout=120)
        if g.is_alive():
            g.kill()
            g.join()
    row.update(bursts=int(lat.size), burst_p50_ms=round(float(np.percentile(lat, 50)), 2), clients_wall_s=round(wall, 2))
    return row


def main():
    ap = argparse.ArgumentParser()
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--parent-source", help="the parent revision's lightning_b200/csrc/sigverifyd.c")
    src.add_argument("--parent-rev", help="a git revision to read it from")
    ap.add_argument("--requests", type=int, default=100, help="timed requests per client process")
    ap.add_argument("--rounds", type=int, default=1, help="alternations of the two daemons per row")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_concurrent: no GPU")
    from lightning_b200 import build
    if a.parent_source:
        source = open(a.parent_source, "rb").read()
    else:
        source = subprocess.run(["git", "show", a.parent_rev + ":lightning_b200/csrc/sigverifyd.c"], cwd=ROOT,
                                capture_output=True, check=True).stdout
    name, power = card()
    torch.cuda.init()
    torch.cuda.mem_get_info(0)  # this process's own CUDA context exists before any daemon is measured
    work = workload([0, 30])
    rows, memory = [], {}
    with tempfile.TemporaryDirectory() as d:
        parent = os.path.join(d, "cln_sigverifyd_parent")
        build_parent(source, parent)
        daemons = {"parent": parent, "workers": build.DAEMON}

        def each(case, fn):
            for r in range(a.rounds):
                for which in (("parent", "workers") if r % 2 == 0 else ("workers", "parent")):
                    with tempfile.TemporaryDirectory(dir=d) as dd:
                        dm = Daemon(daemons[which], dd)
                        memory.setdefault(which, dm.mib)
                        try:
                            rows.append(dict(case, daemon=which, round=r, **fn(dm.sock)))
                        finally:
                            dm.close()

        for h in (0, 30):
            for k in (1, 4, 16, 64):
                each(dict(part="a", load="commitment_signed", htlcs=h, clients=k),
                     lambda s, k=k, h=h: _run_clients(k, tx_client, (s, work[h], a.requests)))
        for k in (1, 4, 16):
            each(dict(part="a", load="bolt12", clients=k), lambda s, k=k: _run_clients(k, bolt12_client, (s, a.requests)))
        for k in (1, 4, 16):
            each(dict(part="b", load="commitment_signed beside x53 bursts", htlcs=30, clients=k),
                 lambda s, k=k: _with_bursts(s, k, work[30], a.requests))
    print(json.dumps({"metric": "sigverifyd_concurrent", "gpu": name, "power_limit": power, "daemon_memory_mib": memory,
                      "rows": rows}))


if __name__ == "__main__":
    main()
