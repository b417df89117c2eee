"""Time sv_verify_bolt12_host (BOLT12 signatures, Merkle root on the device) on the GPU; prints one JSON line.

Workload: the fixture's signed invoice-sized streams (tests/golden/bolt12_vectors.npz, label "signed", invoice tag, at
least 250 bytes), tiled to n
streams laid out one after another in one blob, with 10 % of the signatures corrupted (one flipped bit).  For each n:
wall time per synchronous call (host clock around the call, which ends in a stream synchronise) and streams/s; then, in a
separate profiling pass, the device time of the parse + Merkle + sighash kernels and of the verification kernels (CUDA
events, sv_get_last_bolt12_timing).  The card's name and power limit are read in the same run.  CPU baseline: the
reference's fromwire_tlv + merkle_tlv + sighash_from_merkle + check_schnorr_sig (oracle/_ref/libcln_bolt12.so, one
process per core) on the same streams, when that library is present.  Fails if there is no GPU.

    python tools/measure_bolt12.py [--sizes 1,64,8192,100000,1000000] [--cpu-n 20000]
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

from tests import bolt12  # noqa: E402
from tests.golden.make_bolt12 import L  # noqa: E402


def workload(fx, n, rng):
    # invoice-sized streams: most fuzz-corpus streams are a few fields long, a real invoice is several hundred bytes
    pool = np.nonzero((fx["label"] == L["signed"]) & (fx["names"] == 0) & (fx["len"] >= 250))[0]
    pb = [fx["blob"][fx["off"][i]:fx["off"][i] + fx["len"][i]] for i in pool]
    pool_blob = np.concatenate(pb)
    pool_off = np.concatenate([[0], np.cumsum([b.size for b in pb])[:-1]]).astype(np.uint64)
    reps = -(-n // len(pool))
    idx = np.tile(np.arange(len(pool)), reps)[:n]
    rep = np.repeat(np.arange(reps, dtype=np.uint64), len(pool))[:n]
    blob = np.tile(pool_blob, reps)  # every stream has bytes of its own
    off = pool_off[idx] + rep * np.uint64(pool_blob.size)
    ln = fx["len"][pool][idx].astype(np.uint32)
    xonly = fx["xonly"][pool][idx].copy()
    sig = fx["sig"][pool][idx].copy()
    bad = rng.random(n) < 0.1
    sig[np.nonzero(bad)[0], rng.integers(0, 64, size=int(bad.sum()))] ^= 1
    want = np.where(bad, 0, 1).astype(np.int32)
    return blob, off, ln, xonly, sig, want


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.strip().splitlines() or ["?,?"])[0].split(",")[:2]
    return name.strip(), power.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64,8192,100000,1000000")
    ap.add_argument("--cpu-n", type=int, default=20000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_bolt12: no GPU")
    import lightning_b200 as LB
    eng = LB.SigVerifier(0)
    fx = bolt12.load_fixture()
    rng = np.random.default_rng(7)
    name, power = card()
    mn, fn = bolt12.NAMES[0]
    rows = []
    for n in [int(s) for s in a.sizes.split(",")]:
        blob, off, ln, xonly, sig, want = workload(fx, n, rng)
        for _ in range(3):  # warm-up: module load, scratch growth
            got = eng.verify_bolt12_spans(mn, fn, blob, off, ln, xonly, sig)
        assert np.array_equal(got, want), f"n={n}: statuses differ from the fixture's"
        reps = 200 if n <= 64 else (20 if n <= 8192 else (5 if n <= 100000 else 3))
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            eng.verify_bolt12_spans(mn, fn, blob, off, ln, xonly, sig)
            ts.append(time.perf_counter() - t0)
        wall = statistics.median(ts)
        eng.set_profiling(True)
        mk, vf = [], []
        for _ in range(min(reps, 20)):
            eng.verify_bolt12_spans(mn, fn, blob, off, ln, xonly, sig)
            m, v = eng.last_bolt12_timing()
            mk.append(m)
            vf.append(v)
        eng.set_profiling(False)
        rows.append({"n": n, "wall_ms": round(wall * 1e3, 4), "streams_per_s": round(n / wall, 1),
                     "merkle_device_ms": round(statistics.median(mk), 4), "verify_device_ms": round(statistics.median(vf), 4),
                     "bytes_per_stream": round(float(ln.mean()), 1)})
    cpu = None
    if os.path.exists(bolt12.LIB):
        lib = ctypes.CDLL(bolt12.LIB)
        blob, off, ln, xonly, sig, want = workload(fx, a.cpu_n, rng)
        st = np.zeros(a.cpu_n, np.int32)
        procs = os.cpu_count() or 1
        t0 = time.perf_counter()
        rc = lib.cln_bolt12_check_batch(blob.ctypes.data_as(ctypes.c_void_p), off.ctypes.data_as(ctypes.c_void_p),
                                        ln.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(a.cpu_n), mn, fn,
                                        xonly.ctypes.data_as(ctypes.c_void_p), sig.ctypes.data_as(ctypes.c_void_p),
                                        st.ctypes.data_as(ctypes.c_void_p), procs)
        dt = time.perf_counter() - t0
        assert rc == 0 and np.array_equal(st, want), "CPU baseline disagrees with the fixture"
        cpu = {"n": a.cpu_n, "processes": procs, "wall_s": round(dt, 3), "streams_per_s": round(a.cpu_n / dt, 1)}
    print(json.dumps({"metric": "bolt12_verify", "gpu": name, "power_limit": power, "rows": rows, "cpu_baseline": cpu}))
    eng.close()


if __name__ == "__main__":
    main()
