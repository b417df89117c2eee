#!/usr/bin/env python3
"""Gossip bursts: what finding each channel_update's signer on the device costs, against doing it on the host.

On the same messages, in the same process, alternating call by call:
  (a) one sv_verify_gossip_burst_host call: the scid table, the resolution and the verification all on the device;
  (b) the host-side join (numpy: each announcement's scid and node ids, each update's scid and direction bit, first
      announcement per scid) followed by one sv_verify_gossip_host call with the signers it found.
Sizes: the committed fixture (3,100 messages) and the fixture tiled 53 times (164,300 messages; the tiles share scids,
so every update resolves to tile 0's announcement).  Both give all statuses 0 there, which the script checks.

Also reported:
  - the repair round: the fixture x53 where 1 % of the announcements are corrupted and sent again, uncorrupted, right
    after (the updates of those channels resolve to the corrupted copy first and take the repair round), against the
    clean batch;
  - sv_verify_gossip_host itself against another build of the library (--parent-lib, e.g. built from the parent
    revision), alternating, to show whether the shared-kernel change costs it anything.

  python tools/measure_gossip_burst.py [--reps 15] [--parent-lib path/to/libcln_sigverify.so] [--out result.json]
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
from tests import gossip  # noqa: E402

TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def layout(msgs):
    lens = np.array([len(m) for m in msgs], np.uint32)
    offs = np.zeros(len(msgs), np.uint64)
    offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    return np.frombuffer(b"".join(msgs), np.uint8), offs, lens


def host_join(blob, offs, lens):
    """(b)'s host work: the signer of every channel_update from the first channel_announcement of its scid"""
    o = offs.astype(np.int64)
    typ = (blob[o].astype(np.int32) << 8) | blob[o + 1]
    ca, cu = np.nonzero(typ == 256)[0], np.nonzero(typ == 258)[0]
    co = o[ca]
    base = co + 260 + ((blob[co + 258].astype(np.int64) << 8) | blob[co + 259])
    ca_scid = blob[base[:, None] + 32 + np.arange(8)].copy().view(">u8").ravel()
    nodes = blob[base[:, None] + 40 + np.arange(66)]
    uo = o[cu]
    cu_scid = blob[uo[:, None] + 98 + np.arange(8)].copy().view(">u8").ravel()
    order = np.argsort(ca_scid, kind="stable")  # stable: the first announcement of each scid comes first
    s_sorted = ca_scid[order]
    pos = np.searchsorted(s_sorted, cu_scid)
    pos_c = np.minimum(pos, len(s_sorted) - 1)
    found = (pos < len(s_sorted)) & (s_sorted[pos_c] == cu_scid)
    j = order[pos_c]
    found &= ca[j] < cu  # the announcement must come before the update
    d = (blob[uo + 111] & 1).astype(np.int64)
    signers = np.zeros((len(offs), 33), np.uint8)
    sel = nodes[j[found]]
    dd = d[found]
    signers[cu[found]] = np.where(dd[:, None] == 0, sel[:, :33], sel[:, 33:])
    return signers


def gossip_call(lib, ctx, blob, offs, lens, signers):
    st = np.zeros(len(offs), np.int32)
    rc = lib.sv_verify_gossip_host(ctx, blob.ctypes.data, blob.size, offs.ctypes.data, lens.ctypes.data, len(offs),
                                   signers.ctypes.data, st.ctypes.data)
    assert rc == 0, rc
    return st


def burst_call(eng, blob, offs, lens):
    st = np.zeros(len(offs), np.int32)
    chain = np.frombuffer(TESTNET, np.uint8)
    rc = eng.lib.sv_verify_gossip_burst_host(eng._ctx, chain.ctypes.data, blob.ctypes.data, blob.size, offs.ctypes.data,
                                             lens.ctypes.data, len(offs), None, None, st.ctypes.data)
    assert rc == 0, rc
    return st


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t) * 1e3, r


def med(xs):
    return round(statistics.median(xs), 3)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def corrupted_resent(msgs, every=100):
    """1 % of the announcements corrupted (node_signature_1) and sent again, uncorrupted, right after"""
    out, k = [], 0
    for m in msgs:
        if m[:2] == b"\x01\x00":
            if k % every == 0:
                bad = bytearray(m)
                bad[40] ^= 1
                out.append(bytes(bad))
            k += 1
        out.append(m)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    eng = L.SigVerifier(0)
    lib = eng.lib
    res = dict(gpu=gpu_info(), reps=a.reps, sizes={})
    fixture = gossip.load_subset()
    for name, msgs in (("fixture", fixture), ("fixture_x53", fixture * 53)):
        blob, offs, lens = layout(msgs)
        # warm every shape the timed loop uses, and check both ways give the same statuses
        sa = burst_call(eng, blob, offs, lens)
        sb = gossip_call(lib, eng._ctx, blob, offs, lens, host_join(blob, offs, lens))
        assert np.array_equal(sa, sb) and not sa.any(), name
        ta, tb, tj = [], [], []
        for _ in range(a.reps):
            ta.append(timed(lambda: burst_call(eng, blob, offs, lens))[0])
            t0 = time.perf_counter()
            sg = host_join(blob, offs, lens)
            tj.append((time.perf_counter() - t0) * 1e3)
            tb.append(tj[-1] + timed(lambda: gossip_call(lib, eng._ctx, blob, offs, lens, sg))[0])
        res["sizes"][name] = dict(messages=len(msgs), burst_ms=med(ta), join_plus_gossip_ms=med(tb), host_join_ms=med(tj))
        print(name, res["sizes"][name], flush=True)
    # the repair round
    clean = fixture * 53
    rep = corrupted_resent(clean)
    bc, bo, bl = layout(clean)
    rc_, ro, rl = layout(rep)
    st = burst_call(eng, rc_, ro, rl)
    repairs = lib.sv_last_gossip_repairs(eng._ctx)
    assert repairs > 0 and (st == 1).sum() == len(rep) - len(clean) and (st[st != 1] == 0).all()
    tc, tr = [], []
    for _ in range(a.reps):
        tc.append(timed(lambda: burst_call(eng, bc, bo, bl))[0])
        tr.append(timed(lambda: burst_call(eng, rc_, ro, rl))[0])
    res["repair"] = dict(messages=len(rep), corrupted_announcements=len(rep) - len(clean), repaired_updates=int(repairs),
                         clean_ms=med(tc), with_repair_ms=med(tr))
    print("repair", res["repair"], flush=True)
    # sv_verify_gossip_host against another build
    if a.parent_lib:
        plib = ctypes.CDLL(os.path.abspath(a.parent_lib), mode=ctypes.RTLD_LOCAL)
        plib.sv_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
        plib.sv_destroy.argtypes = [ctypes.c_void_p]
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        plib.sv_verify_gossip_host.argtypes = [vp, vp, sz, vp, vp, sz, vp, vp]
        pctx = ctypes.c_void_p()
        assert plib.sv_create(ctypes.byref(pctx), 0) == 0
        res["gossip_host_vs_parent"] = {}
        for name, msgs in (("fixture", fixture), ("fixture_x53", clean)):
            blob, offs, lens = layout(msgs)
            sg = host_join(blob, offs, lens)
            assert np.array_equal(gossip_call(lib, eng._ctx, blob, offs, lens, sg), gossip_call(plib, pctx, blob, offs, lens, sg))
            tn, tp = [], []
            for _ in range(a.reps):
                tn.append(timed(lambda: gossip_call(lib, eng._ctx, blob, offs, lens, sg))[0])
                tp.append(timed(lambda: gossip_call(plib, pctx, blob, offs, lens, sg))[0])
            res["gossip_host_vs_parent"][name] = dict(this_ms=med(tn), parent_ms=med(tp), this_min_ms=round(min(tn), 3),
                                                      parent_min_ms=round(min(tp), 3))
            print("gossip_host", name, res["gossip_host_vs_parent"][name], flush=True)
        plib.sv_destroy(pctx)
    eng.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
