#!/usr/bin/env python3
"""Whole gossip_stores: what sv_verify_gossip_store_host costs, and the same work on the host's cores with CLN's code.

Stores: the committed fixture (tests/golden/gossip_store_subset.bin: 4,600 records, 974,526 bytes, 9,100 signatures
counting each announcement's four) and the fixture's records tiled 53 times (243,800 records, 51.6 MB; the copies are
redundant announcements and updates that resolve to the first copy).

GPU: wall time per call after warm-up (median of --reps calls), split with the engine's profiling events into the host
header walk, the H2D copy of the store, the checksum kernel and the rest (slicing, channel table, hashing,
verification).  CPU, where oracle/_ref holds CLN's code: gossipd/sigcheck.c's sigcheck_* over the same messages with the
signers gossmap's channel table gives, on every core (one process per core).  The CPU side does not include the
checksums: CLN's crc32c is not part of oracle/_ref, and CRC-32C on a CPU runs at GB/s, far below the signature cost.
Also prints the card's name and power limit.

  python tools/measure_gossip_store.py [--reps 15] [--out result.json]
"""
import argparse
import ctypes
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import lightning_b200 as L  # noqa: E402
from tests import gossip_store as gs  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
CLN = os.path.join(ROOT, "oracle", "_ref", "libcln_ref.so")


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def time_gpu(eng, store, reps):
    for _ in range(3):
        eng.verify_gossip_store(store, TESTNET)
    wall, parts = [], []
    for _ in range(reps):
        t = time.perf_counter()
        _, _, st, _, s = eng.verify_gossip_store(store, TESTNET)
        wall.append((time.perf_counter() - t) * 1e3)
        parts.append(eng.last_gossip_store_timing())
    assert s["stop"] == gs.EOF and s["bad_signature"] == s["malformed"] == s["no_channel"] == 0
    med = [statistics.median(p[i] for p in parts) for i in range(4)]
    return dict(wall_ms=statistics.median(wall), walk_ms=med[0], h2d_ms=med[1], crc_ms=med[2], verify_ms=med[3],
                good=s["good"], records=s["records"])


def _cpu_chunk(args):
    items = args
    lib = ctypes.CDLL(CLN)
    lib.cln_sigcheck_channel_announcement.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    lib.cln_sigcheck_node_announcement.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
    lib.cln_sigcheck_channel_update.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p]
    bad = 0
    for t, m, signer in items:
        if t == 256:
            bad += lib.cln_sigcheck_channel_announcement(m, len(m)) != 0
        elif t == 257:
            bad += lib.cln_sigcheck_node_announcement(m, len(m)) != 0
        else:
            bad += lib.cln_sigcheck_channel_update(m, len(m), signer) != 0
    return bad


def cpu_items(store):
    out, _ = gs.audit(store)
    recs = {o: n for o, _, n, _ in gs.walk(store)[0]}
    items = []
    for o, t, _, h in out:
        if t not in (256, 257, 258):
            continue
        m = store[o + 12:o + 12 + recs[o]]
        signer = None
        if t == 258:
            a = store[h + 12:h + 12 + recs[h]]
            signer = gs.ann_fields(a)[2 + (m[111] & 1)]
        items.append((t, m, signer))
    return items


def time_cpu(store, procs):
    items = cpu_items(store)
    chunks = [items[k::procs] for k in range(procs)]
    with mp.Pool(procs) as pool:
        pool.map(_cpu_chunk, [c[:10] for c in chunks])  # load the library in every worker
        t = time.perf_counter()
        bad = sum(pool.map(_cpu_chunk, chunks))
        ms = (time.perf_counter() - t) * 1e3
    assert bad == 0
    return dict(sigcheck_ms=ms, processes=procs, messages=len(items))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out")
    a = ap.parse_args()
    fx = open(os.path.join(ROOT, "tests", "golden", "gossip_store_subset.bin"), "rb").read()
    stores = {"fixture": fx, "x53": fx[:1] + fx[1:] * 53}
    res = dict(gpu=gpu_info(), cpu_cores=os.cpu_count())
    print("GPU (name, power limit):", res["gpu"], "| host cores:", res["cpu_cores"])
    eng = L.SigVerifier(0)
    eng.set_profiling(True)
    for name, st in stores.items():
        r = time_gpu(eng, st, a.reps)
        r["bytes"] = len(st)
        res[name] = r
        print(f"{name}: {len(st)} bytes, {r['records']} records, {r['good']} messages good | GPU wall {r['wall_ms']:.2f} ms "
              f"(walk {r['walk_ms']:.2f}, H2D {r['h2d_ms']:.2f}, CRC {r['crc_ms']:.3f}, verify {r['verify_ms']:.2f} ms)")
    eng.close()
    if os.path.exists(CLN):
        for name, st in stores.items():
            c = time_cpu(st, os.cpu_count() or 1)
            res[name]["cpu"] = c
            print(f"{name}: CLN sigcheck on {c['processes']} processes: {c['sigcheck_ms']:.1f} ms for {c['messages']} messages")
    else:
        print("oracle/_ref/libcln_ref.so not present: no CPU comparison")
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
