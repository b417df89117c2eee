"""Time repairing a torn gossip_store FILE in place (sv_repair_gossip_store_fd) against pruning it in place
(sv_prune_gossip_store_fd), in-process and through cln_sigverifyd; prints one JSON line.

Stores: the committed fixture (4,600 records) and the fixture tiled 53 times with 1 % of its records corrupted
(tests/test_gpu_gossip_store_prune.py corrupted_x53), each followed by a new channel's channel_announcement,
channel_amount, channel_update and node_announcement (tests/test_gpu_gossip_store_repair.py last_four) and torn halfway
through the channel_update, as a crash during its append leaves it.  The repair cuts the torn update; the prune leaves it.
Before every timed call the file is rewritten with the torn store and synced (not timed).  The two calls alternate, so a
drift of the machine affects both alike.  Per store, the median wall time of one call:
  in_process   SigVerifier.prune_gossip_store_fd / repair_gossip_store_fd on a warm context (after 2 calls each);
  daemon       through cln_sigverifyd: from the sendmsg carrying the request and the file's descriptor to the reply (the
               daemon has served one call of each first).
The difference should be one ftruncate and one fsync.  The card's name and power limit are read in the same run.  Every
summary and new length is checked.  Fails if there is no GPU.

    python tools/measure_gossip_store_repair.py [--reps 9]
"""
import argparse
import json
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
from measure_sigverifyd_prune import rewrite  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def stores():
    """name -> (torn store, offset of the torn channel_update)"""
    from tests.test_gossip_store_host import load_fixture
    from tests.test_gpu_gossip_store_prune import corrupted_x53
    from tests.test_gpu_gossip_store_repair import last_four
    out = {}
    for name, head in (("fixture", load_fixture()), ("x53_corrupted_1pct", corrupted_x53())):
        ca, am, cu, _ = last_four()
        at = len(head) + len(ca) + len(am)
        out[name] = ((head + ca + am + cu[:len(cu) // 2]), at)
    return out


def daemon_call(sock_path, path, store, rid, repair):
    """one call through the daemon on a fresh copy of store: (seconds, reply fields)"""
    from lightning_b200 import sigverifyd_wire as W
    rewrite(path, store)
    msg = "sigverifyd_gossip_store_repair" if repair else "sigverifyd_gossip_store_prune"
    frame = W.encode(msg, req_id=rid, has_chain=1, chain_hash=TESTNET, len=len(store))
    fd = os.open(path, os.O_RDWR)
    c = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    c.connect(sock_path)
    try:
        t0 = time.perf_counter()
        socket.send_fds(c, [frame], [fd])
        name, m = W.read_msg(c)
        dt = time.perf_counter() - t0
    finally:
        c.close()
        os.close(fd)
    assert name == msg + "_reply" and m["req_id"] == rid and m["err"] == 0, (name, m)
    return dt, m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_gossip_store_repair: no GPU")
    import lightning_b200 as LB
    from lightning_b200 import build
    name, power = card()
    st = stores()
    eng = LB.SigVerifier(0)
    want = {k: eng.prune_gossip_store(v, TESTNET)[2] for k, (v, _) in st.items()}
    out = {"metric": "gossip_store_repair", "gpu": name, "power_limit": power, "stores": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gossip_store")
        for k, (store, cut) in st.items():
            row = {"bytes": len(store), "records": want[k]["records"], "pruned": want[k]["pruned"], "cut_bytes": len(store) - cut}
            times = {False: [], True: []}
            for r in range(a.reps + 2):
                for repair in (False, True):
                    rewrite(path, store)
                    fd = os.open(path, os.O_RDWR)
                    t0 = time.perf_counter()
                    if repair:
                        s, new_len = eng.repair_gossip_store_fd(fd, len(store), TESTNET)
                    else:
                        s, new_len = eng.prune_gossip_store_fd(fd, len(store), TESTNET), len(store)
                    dt = time.perf_counter() - t0
                    os.close(fd)
                    assert s == want[k] and new_len == (cut if repair else len(store)) == os.path.getsize(path)
                    if r >= 2:
                        times[repair].append(dt * 1e3)
            row["in_process_prune_ms"] = round(statistics.median(times[False]), 2)
            row["in_process_repair_ms"] = round(statistics.median(times[True]), 2)
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
            rid = 1
            for repair in (False, True):  # warm-up
                daemon_call(sock_path, path, st["fixture"][0], rid, repair)
                rid += 1
            for k, (store, cut) in st.items():
                times = {False: [], True: []}
                for r in range(a.reps):
                    for repair in (False, True):
                        dt, m = daemon_call(sock_path, path, store, rid, repair)
                        rid += 1
                        assert m["pruned"] == want[k]["pruned"] and (not repair or m["new_len"] == cut)
                        times[repair].append(dt * 1e3)
                out["stores"][k]["daemon_prune_ms"] = round(statistics.median(times[False]), 2)
                out["stores"][k]["daemon_repair_ms"] = round(statistics.median(times[True]), 2)
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
