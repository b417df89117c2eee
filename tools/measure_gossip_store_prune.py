#!/usr/bin/env python3
"""What pruning a gossip_store costs next to auditing it: one sv_prune_gossip_store_host call against one
sv_verify_gossip_store_host call on the same store.

Stores: the committed fixture (tests/golden/gossip_store_subset.bin, 4,600 records) and the fixture tiled 53 times
(243,800 records, 51.6 MB), each as it is (0 %) and with 1 % of its records corrupted (a flipped signature bit with the
checksum recomputed, a flipped message bit, or an unknown type; tests/test_gpu_gossip_store_prune.py corrupted_x53's
recipe).  Wall time per call after warm-up (median of --reps calls); for the prune, the engine's profiling events split
it into the host header walk, the first round (H2D of the store, checksums, the audit's kernels), the second round
(mark, second resolution, compaction, re-verification of the updates whose signer changed) and the flag write with the
copy back of the changed flag bytes.  Also prints the card's name and power limit.

  python tools/measure_gossip_store_prune.py [--reps 15] [--out result.json]
"""
import argparse
import json
import os
import statistics
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import lightning_b200 as L  # noqa: E402
from tests import gossip_store as gs  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def corrupt(store, rate, seed=53):
    store = bytearray(store)
    rng = np.random.default_rng(seed)
    for off, t, ln, _ in gs.walk(bytes(store))[0]:
        if rng.random() >= rate:
            continue
        k = int(rng.integers(0, 3))
        if k == 0 and t in (256, 257, 258):
            store[off + 12 + 2 + int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
        elif k == 1:
            store[off + 12 + int(rng.integers(2, ln))] ^= 1
            continue
        else:
            store[off + 12:off + 14] = struct.pack(">H", 4999)
        ts = struct.unpack(">I", store[off + 8:off + 12])[0]
        struct.pack_into(">I", store, off + 4, gs.crc32c(ts, bytes(store[off + 12:off + 12 + ln])))
    return bytes(store)


def median_ms(fn, reps):
    for _ in range(3):
        fn()
    wall, parts = [], []
    for _ in range(reps):
        t = time.perf_counter()
        r = fn()
        wall.append((time.perf_counter() - t) * 1e3)
        parts.append(r)
    return statistics.median(wall), parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out")
    a = ap.parse_args()
    fx = open(os.path.join(ROOT, "tests", "golden", "gossip_store_subset.bin"), "rb").read()
    x53 = fx[:1] + fx[1:] * 53
    res = dict(gpu=gpu_info())
    print("GPU (name, power limit):", res["gpu"])
    eng = L.SigVerifier(0)
    eng.set_profiling(True)
    for name, base in (("fixture", fx), ("x53", x53)):
        for rate in (0.0, 0.01):
            st = corrupt(base, rate) if rate else base
            audit_ms, _ = median_ms(lambda: eng.verify_gossip_store(st, TESTNET), a.reps)

            def prune():
                _, _, s = eng.prune_gossip_store(st, TESTNET)
                return s, eng.last_gossip_prune_timing()
            prune_ms, parts = median_ms(prune, a.reps)
            s = parts[-1][0]
            split = [statistics.median(p[1][i] for p in parts) for i in range(4)]
            key = f"{name}_{int(rate * 100)}pct"
            res[key] = dict(bytes=len(st), records=s["records"], pruned=s["pruned"], reverified=s["reverified"],
                            audit_ms=audit_ms, prune_ms=prune_ms, walk_ms=split[0], first_round_ms=split[1],
                            second_round_ms=split[2], flags_ms=split[3])
            print(f"{key}: {s['records']} records, {s['pruned']} deleted, {s['reverified']} re-verified | audit "
                  f"{audit_ms:.2f} ms, prune {prune_ms:.2f} ms (walk {split[0]:.2f}, first round {split[1]:.2f}, "
                  f"second round {split[2]:.3f}, flags {split[3]:.3f} ms)")
    eng.close()
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
