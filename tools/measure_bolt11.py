"""Time sv_verify_bolt11_host (BOLT11 invoice signatures, everything on the device) on the GPU; prints one JSON line.

Workload: the fixture's invoices that Core Lightning accepts (tests/golden/bolt11_vectors.npz: the BOLT #11 examples and
the signed invoices, with and without `n`, route hints included), tiled to n invoices laid out one after another in one
blob, with 10 % of them replaced by the fixture's corrupted-signature invoices (a signature word changed, checksum
recomputed: bolt11_decode refuses them in its signature step).  For each n: wall time per synchronous call (host clock
around the call, which ends in a stream synchronise) and invoices/s; then, in a separate profiling pass, the device time
of the parse + hash stage and of the verification + recovery stage (CUDA events, sv_get_last_bolt11_timing).  The card's
name and power limit are read in the same run.  CPU baseline: the reference's bolt11_decode (oracle/_ref/libcln_bolt11.so,
one process per core) on the same invoices, when that library is present.  Fails if there is no GPU.

    python tools/measure_bolt11.py [--sizes 1,64,8192,100000,1000000] [--cpu-n 100000]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import bolt11  # noqa: E402


def workload(fx, n, rng):
    good = np.nonzero((fx["expected"] == 1) & ((fx["ret"] & 1) == 1))[0]
    bad = np.nonzero((fx["expected"] == 0) & np.isin(fx["label_name"], ["flip", "high_s"]))[0]
    corrupt = rng.random(n) < 0.1
    pick = np.where(corrupt, bad[rng.integers(0, len(bad), n)], good[np.arange(n) % len(good)])
    ln = fx["len"][pick].astype(np.uint32)
    off = np.zeros(n, np.uint64)
    off[1:] = np.cumsum(ln[:-1], dtype=np.uint64)
    src = fx["blob"]
    blob = np.concatenate([src[fx["off"][i]:fx["off"][i] + fx["len"][i]] for i in pick]) if n else np.zeros(0, np.uint8)
    return blob, off, ln, np.where(corrupt, 0, 1).astype(np.int32)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().splitlines() or ["?,?"])[0].split(",")[:2]
    return name.strip(), power.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64,8192,100000,1000000")
    ap.add_argument("--cpu-n", type=int, default=100000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_bolt11: no GPU")
    import lightning_b200 as LB
    eng = LB.SigVerifier(0)
    fx = bolt11.load_fixture()
    rng = np.random.default_rng(7)
    name, power = card()
    rows = []
    for n in [int(s) for s in a.sizes.split(",")]:
        blob, off, ln, want = workload(fx, n, rng)
        for _ in range(3):  # warm-up: module load, scratch growth
            got = eng.verify_bolt11_spans(blob, off, ln)[0]
        assert np.array_equal(got, want), f"n={n}: statuses differ from the fixture's"
        reps = 200 if n <= 64 else (20 if n <= 8192 else (5 if n <= 100000 else 3))
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            eng.verify_bolt11_spans(blob, off, ln)
            ts.append(time.perf_counter() - t0)
        wall = statistics.median(ts)
        eng.set_profiling(True)
        pm, cm = [], []
        for _ in range(min(reps, 20)):
            eng.verify_bolt11_spans(blob, off, ln)
            p, c = eng.last_bolt11_timing()
            pm.append(p)
            cm.append(c)
        eng.set_profiling(False)
        rows.append({"n": n, "wall_ms": round(wall * 1e3, 4), "invoices_per_s": round(n / wall, 1),
                     "parse_hash_device_ms": round(statistics.median(pm), 4),
                     "curve_device_ms": round(statistics.median(cm), 4), "chars_per_invoice": round(float(ln.mean()), 1)})
    cpu = None
    if os.path.exists(bolt11.LIB):
        lib = ctypes.CDLL(bolt11.LIB)
        blob, off, ln, want = workload(fx, a.cpu_n, rng)
        ok = np.zeros(a.cpu_n, np.int32)
        procs = os.cpu_count() or 1
        t0 = time.perf_counter()
        rc = lib.cln_bolt11_decode_batch(blob.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p),
                                         ln.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(a.cpu_n),
                                         ok.ctypes.data_as(ctypes.c_void_p), procs)
        dt = time.perf_counter() - t0
        assert rc == 0 and np.array_equal(ok, want), "CPU baseline disagrees with the fixture"
        cpu = {"n": a.cpu_n, "processes": procs, "wall_s": round(dt, 3), "invoices_per_s": round(a.cpu_n / dt, 1)}
    print(json.dumps({"metric": "bolt11_verify", "gpu": name, "power_limit": power, "rows": rows, "cpu_baseline": cpu}))
    eng.close()


if __name__ == "__main__":
    main()
