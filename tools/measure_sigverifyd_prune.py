"""Time pruning a gossip_store FILE in place (sv_prune_gossip_store_fd) the three ways gossipd could do it, and what a
prune running back to back does to channel checks; prints one JSON line.

Stores: the committed fixture (tests/golden/gossip_store_subset.bin, 4,600 records) and the fixture tiled 53 times with
1 % of its records corrupted (tests/test_gpu_gossip_store_prune.py corrupted_x53, 51.6 MB).  Before every timed call the
file is rewritten with the unpruned store and synced (not timed), so the prune's own fsync flushes only the flags it
wrote, as it would on a store gossipd has had on disk.  Per store, the median wall time of one prune:
  daemon         through cln_sigverifyd: from the sendmsg carrying the request and the file's descriptor to the reply
                 (the daemon has served one prune first);
  in_process     SigVerifier.prune_gossip_store_fd on a warm context (after 2 calls);
  host_call      for comparison, SigVerifier.prune_gossip_store on the bytes in memory (no file);
  fresh_process  in a new process: sv_create plus the one prune (what gossipd would pay if it linked the library itself),
                 and the process's whole wall time from its start (interpreter and import included).
Channel checks: k = 4 channeld-like processes send commitment_signed checks (tools/measure_sigverifyd_tx.py's client,
H = 30) to one daemon, without prunes and while a gossipd-like process prunes the x53 store back to back: requests/s and
p50 / p99 latency, and the prunes served meanwhile.  The card's name and power limit are read in the same run.  Every
prune's summary and every verdict is checked.  Fails if there is no GPU.

    python tools/measure_sigverifyd_prune.py [--reps 7] [--requests 100]
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_bolt12 import card  # noqa: E402
from measure_sigverifyd_tx import _client_daemon as tx_client  # noqa: E402
from measure_sigverifyd_tx import _run_clients, workload  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def stores():
    from tests.test_gossip_store_host import load_fixture
    from tests.test_gpu_gossip_store_prune import corrupted_x53
    return {"fixture": load_fixture(), "x53_corrupted_1pct": corrupted_x53()}


def rewrite(path, store):
    """the file holds the unpruned store again, on disk"""
    with open(path, "wb") as f:
        f.write(store)
        f.flush()
        os.fsync(f.fileno())


def _prune_frame(rid, length):
    from lightning_b200 import sigverifyd_wire as W
    return W.encode("sigverifyd_gossip_store_prune", req_id=rid, has_chain=1, chain_hash=TESTNET, len=length)


def daemon_prune(sock_path, path, store, rid):
    """one prune through the daemon on a fresh copy of store: (seconds, reply fields)"""
    from lightning_b200 import sigverifyd_wire as W
    rewrite(path, store)
    fd = os.open(path, os.O_RDWR)
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    try:
        t0 = time.perf_counter()
        socket.send_fds(c, [_prune_frame(rid, len(store))], [fd])
        name, m = W.read_msg(c)
        dt = time.perf_counter() - t0
    finally:
        c.close()
        os.close(fd)
    assert name == "sigverifyd_gossip_store_prune_reply" and m["req_id"] == rid and m["err"] == 0, (name, m)
    return dt, m


FRESH = r"""
import os, sys, time
t_start = float(sys.argv[3])
sys.path.insert(0, sys.argv[1])
import lightning_b200 as LB
path, n = sys.argv[2], int(sys.argv[4])
t0 = time.perf_counter()
eng = LB.SigVerifier(0)
fd = os.open(path, os.O_RDWR)
s = eng.prune_gossip_store_fd(fd, n, bytes.fromhex(sys.argv[5]))
t1 = time.perf_counter()
os.close(fd)
print(t1 - t0, time.time() - t_start, s["pruned"])
"""


def _gossipd(sock_path, path, store, want, ready, stop, q):
    """x53 prunes back to back until stop is set: the prunes' latencies"""
    lat, rid = [], 0
    ready.set()
    while not stop.is_set():
        rid += 1
        dt, m = daemon_prune(sock_path, path, store, rid)
        assert m["pruned"] == want
        lat.append(dt)
    q.put(lat)


def _with_prunes(sock_path, path, store, want, work, nreq):
    ctx = mp.get_context("spawn")
    ready, stop, q = ctx.Event(), ctx.Event(), ctx.Queue()
    g = ctx.Process(target=_gossipd, args=(sock_path, path, store, want, ready, stop, q))
    g.start()
    try:
        assert ready.wait(timeout=600)
        time.sleep(0.3)  # the first prune is on its way
        row = _run_clients(4, tx_client, (sock_path, work, nreq))
        stop.set()
        lat = [x * 1e3 for x in q.get(timeout=600)]
    finally:
        g.join(timeout=120)
        if g.is_alive():
            g.kill()
            g.join()
    row.update(prunes=len(lat), prune_p50_ms=round(statistics.median(lat), 2))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--requests", type=int, default=100, help="timed commitment_signed requests per channeld process")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_sigverifyd_prune: no GPU")
    import lightning_b200 as LB
    from lightning_b200 import build
    name, power = card()
    st = stores()
    eng = LB.SigVerifier(0)
    want = {k: eng.prune_gossip_store(v, TESTNET)[2] for k, v in st.items()}
    out = {"metric": "sigverifyd_prune", "gpu": name, "power_limit": power, "stores": {}, "channel_checks": []}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gossip_store")
        for k, store in st.items():
            row = {"bytes": len(store), "records": want[k]["records"], "pruned": want[k]["pruned"]}
            # in-process, warm context
            times = []
            for r in range(a.reps + 2):
                rewrite(path, store)
                fd = os.open(path, os.O_RDWR)
                t0 = time.perf_counter()
                s = eng.prune_gossip_store_fd(fd, len(store), TESTNET)
                dt = time.perf_counter() - t0
                os.close(fd)
                assert s == want[k]
                if r >= 2:
                    times.append(dt * 1e3)
            row["in_process_ms"] = round(statistics.median(times), 2)
            times = []
            for r in range(a.reps + 2):
                t0 = time.perf_counter()
                eng.prune_gossip_store(store, TESTNET)
                if r >= 2:
                    times.append((time.perf_counter() - t0) * 1e3)
            row["host_call_ms"] = round(statistics.median(times), 2)
            # a fresh process: sv_create and one prune
            fresh, whole = [], []
            for r in range(3):
                rewrite(path, store)
                t = subprocess.run([sys.executable, "-c", FRESH, ROOT, path, repr(time.time()), str(len(store)), TESTNET.hex()],
                                   capture_output=True, text=True, timeout=600, check=True)
                x, y, pruned = t.stdout.split()
                assert int(pruned) == want[k]["pruned"]
                fresh.append(float(x) * 1e3)
                whole.append(float(y) * 1e3)
            row["fresh_process_create_and_prune_ms"] = round(statistics.median(fresh), 1)
            row["fresh_process_wall_ms"] = round(statistics.median(whole), 1)
            out["stores"][k] = row
        eng.close()
        sock_path = os.path.join(d, "sv.sock")
        daemon = subprocess.Popen([build.DAEMON, sock_path, "0"], stderr=subprocess.DEVNULL)
        try:
            for _ in range(600):
                if os.path.exists(sock_path) or daemon.poll() is not None:
                    break
                time.sleep(0.1)
            assert os.path.exists(sock_path), "daemon did not come up"
            daemon_prune(sock_path, path, st["fixture"], 1)  # warm-up
            for k, store in st.items():
                times = []
                for r in range(a.reps):
                    dt, m = daemon_prune(sock_path, path, store, 10 + r)
                    assert m["pruned"] == want[k]["pruned"] and m["records"] == want[k]["records"]
                    times.append(dt * 1e3)
                out["stores"][k]["daemon_ms"] = round(statistics.median(times), 2)
            work = workload([30])[30]
            out["channel_checks"].append(dict(load="commitment_signed, H = 30", **_run_clients(4, tx_client, (sock_path, work, a.requests))))
            x53 = st["x53_corrupted_1pct"]
            out["channel_checks"].append(dict(load="commitment_signed, H = 30, beside x53 prunes back to back",
                                              **_with_prunes(sock_path, path, x53, want["x53_corrupted_1pct"]["pruned"], work,
                                                             a.requests)))
        finally:
            daemon.terminate()
            try:
                daemon.wait(timeout=30)
            except subprocess.TimeoutExpired:
                daemon.kill()
                daemon.wait(timeout=30)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
