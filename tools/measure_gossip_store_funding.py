#!/usr/bin/env python3
"""What checking a gossip_store's channels against lightningd's funding outputs costs: the audit against the audit with
a funding table (sv_verify_gossip_store_host / sv_verify_gossip_store_funding_host), and the prune against the prune with
a funding table (sv_prune_gossip_store_host / sv_prune_gossip_store_funding_host), on the same store.

Stores: the committed fixture (tests/golden/gossip_store_subset.bin, 4,600 records, 1,500 announcements) and the fixture
tiled 53 times (243,800 records, 79,500 announcements, all but 1,500 of them redundant).  Tables: the one that funds
every announcement as its amount record says (tests/gossip_store_funding.py table_of_store, 1,500 outputs), as it is
(0 %) and with 1 % of its entries wrong (corrupt_table: an output removed, with or without its block, a script byte
flipped, or the amount one sat more).  Wall time per call after warm-up (median of --reps calls); the four calls of a
store and table (audit, audit + funding, prune, prune + funding) run in turn, one of each per repetition, so that host
noise falls on all four alike.  The engine's profiling events give the device time of the funding step (table staging
and sort, k_store_funding).

CPU column: Core Lightning's own scriptpubkey_p2wsh(bitcoin_redeem_2of2()) plus a lookup by scid (bsearch) and a script
compare per announcement, on one core (oracle/_ref/libcln_funding.so cln_funding_check_batch; median of --cpu-reps).
Also prints the card's name and power limit.

  python tools/measure_gossip_store_funding.py [--reps 15] [--cpu-reps 5] [--out result.json]
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

import lightning_b200 as L  # noqa: E402
from lightning_b200.funding import FundingTable  # noqa: E402
from tests import gossip_store as gs  # noqa: E402
from tests import gossip_store_funding as gf  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
FUNDING_LIB = os.path.join(ROOT, "oracle", "_ref", "libcln_funding.so")


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


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


def interleaved_ms(fns, reps):
    """fns called in turn, reps rounds after 3 of warm-up -> per fn (median ms, its results)"""
    for _ in range(3):
        for f in fns:
            f()
    wall, parts = [[] for _ in fns], [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            t = time.perf_counter()
            r = f()
            wall[k].append((time.perf_counter() - t) * 1e3)
            parts[k].append(r)
    return [(statistics.median(w), p) for w, p in zip(wall, parts)]


def table(t):
    return FundingTable.from_arrays(np.array(t[0], np.uint64), np.array(t[1], np.uint64),
                                    np.frombuffer(b"".join(t[2]), np.uint8).reshape(-1, 34), np.array(t[3], np.uint32))


def cpu_ms(store, ft, reps):
    """the reference's per-announcement work on one core, or None without oracle/_ref"""
    if not os.path.exists(FUNDING_LIB):
        return None
    lib = ctypes.CDLL(FUNDING_LIB)
    keys, scids = [], []
    for off, typ, ln, st in gs.walk(store)[0]:
        if typ == 256 and st == 0:
            s, k1, k2 = gf.ann_keys(store, off + gs.HDR)
            keys.append(k1 + k2)
            scids.append(s)
    k = np.frombuffer(b"".join(keys), np.uint8).copy()
    sc = np.array(scids, np.uint64)
    order = np.argsort(ft.scid)
    srt, script = ft.scid[order].copy(), ft.script[order].copy()
    match = np.zeros(len(scids), np.uint8)
    vp = ctypes.c_void_p
    lib.cln_funding_check_batch.argtypes = [vp, vp, ctypes.c_size_t, vp, vp, ctypes.c_size_t, vp]
    lib.cln_funding_check_batch.restype = None
    run = lambda: lib.cln_funding_check_batch(k.ctypes.data, sc.ctypes.data, sc.size, srt.ctypes.data, script.ctypes.data,
                                              srt.size, match.ctypes.data)
    ms, _ = median_ms(run, reps)
    return ms, len(scids), int(match.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--cpu-reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    fx = open(os.path.join(ROOT, "tests", "golden", "gossip_store_subset.bin"), "rb").read()
    x53 = fx[:1] + fx[1:] * 53
    base = gf.table_of_store(fx)
    tables = {"0pct": table(base), "1pct": table(gf.corrupt_table(base, 0.01, 53))}
    res = dict(gpu=gpu_info(), reps=a.reps, cpu_reps=a.cpu_reps)
    print("GPU (name, power limit):", res["gpu"])
    eng = L.SigVerifier(0)
    eng.set_profiling(True)
    for name, st in (("fixture", fx), ("x53", x53)):
        for tname, ft in tables.items():
            def audit_f():
                r = eng.verify_gossip_store(st, TESTNET, funding=ft)
                return r[6], eng.last_gossip_funding_timing()

            def prune_f():
                r = eng.prune_gossip_store(st, TESTNET, funding=ft)
                return r[4], eng.last_gossip_funding_timing(), eng.last_gossip_prune_timing()

            def prune_p():
                eng.prune_gossip_store(st, TESTNET)
                return eng.last_gossip_prune_timing()
            (audit_ms, _), (af_ms, ap), (prune_ms, p0), (pf_ms, pp) = interleaved_ms(
                [lambda: eng.verify_gossip_store(st, TESTNET), audit_f, prune_p, prune_f], a.reps)
            fs = pp[-1][0]
            stage = statistics.median(p[1][0] for p in ap)
            kern = statistics.median(p[1][1] for p in ap)
            # the prune's own profiling split (header walk, first round, second round, flag write), without and with
            split = [round(statistics.median(p[i] for p in p0), 3) for i in range(4)]
            split_f = [round(statistics.median(p[2][i] for p in pp), 3) for i in range(4)]
            cpu = cpu_ms(st, ft, a.cpu_reps)
            key = f"{name}_table_{tname}"
            res[key] = dict(bytes=len(st), outputs=len(ft), checked=fs["checked"], funded=fs["funded"],
                            deleted=fs["deleted"], audit_ms=audit_ms, audit_funding_ms=af_ms, prune_ms=prune_ms,
                            prune_funding_ms=pf_ms, funding_stage_ms=stage, funding_kernel_ms=kern,
                            prune_split_ms=split, prune_funding_split_ms=split_f,
                            cpu_ms=None if cpu is None else cpu[0], cpu_announcements=None if cpu is None else cpu[1])
            print(f"{key}: {fs['checked']} announcements checked, {fs['funded']} funded, {fs['deleted']} deleted | audit "
                  f"{audit_ms:.2f} -> {af_ms:.2f} ms, prune {prune_ms:.2f} -> {pf_ms:.2f} ms | device: staging+sort "
                  f"{stage:.3f} ms, k_store_funding {kern:.3f} ms | CPU (CLN, one core): "
                  + ("n/a" if cpu is None else f"{cpu[0]:.2f} ms for {cpu[1]} announcements")
                  + f" | prune split {split} -> {split_f} ms")
    eng.close()
    if a.out:
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
