"""Time salvaging a gossip_store past damaged headers (sv_salvage_gossip_store_host, sv_salvage_gossip_store_fd) against
repairing it (sv_repair_gossip_store_fd); prints one JSON line.

Stores: the committed fixture (4,600 records) and the fixture tiled 53 times, each with a gossip_store_uuid record first
(tests/test_gossip_store_salvage_host.py with_uuid), clean and with one break (bit 0 of the length's high byte flipped a
third of the way in).  Per store, medians over --reps runs after 2 warm-up runs:
  filter_ms, crc_ms   the device's two filter passes with the scan, and the checksum kernel (CUDA events around the
                      kernels only, profiling mode)
  walk_ms             the host walk over the sorted sound offsets
  in_memory_ms        SigVerifier.salvage_gossip_store, whole call (the store's copy to the device included)
  salvage_fd_ms       SigVerifier.salvage_gossip_store_fd: salvage, header writes, fsync, then the repair
  repair_fd_ms        SigVerifier.repair_gossip_store_fd alone, alternating with the call above
  cpu_scan_ms         one core: a plain scan of the same rule over every byte offset, each candidate's checksum in one
                      slice-by-8 pass (tests/host_emul libemul.so emul_gs_salvage_sound_plain, g++ -O2)
Before every file call the file is rewritten with the store and synced (not timed).  The card's name and power limit are
read in the same run.  The salvage's result is checked against the model's sound offsets on the fixture.  Fails if there
is no GPU.

    python tools/measure_gossip_store_salvage.py [--reps 9]
"""
import argparse
import ctypes
import json
import os
import statistics
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
    from tests import gossip_store as gs
    from tests.test_gossip_store_host import load_fixture
    from tests.test_gossip_store_salvage_host import with_uuid, x53
    out = {}
    for name, s in (("fixture", with_uuid(load_fixture())), ("x53", with_uuid(x53()))):
        recs = gs.walk(s)[0]
        d = bytearray(s)
        d[recs[len(recs) // 3][0] + 2] ^= 1
        out[name + "_clean"] = s
        out[name + "_one_break"] = bytes(d)
    return out


def med(xs):
    return round(statistics.median(xs), 3)


def file_call(path, store, fn):
    rewrite(path, store)
    fd = os.open(path, os.O_RDWR)
    try:
        t0 = time.perf_counter()
        r = fn(fd, len(store), TESTNET)
        return (time.perf_counter() - t0) * 1e3, r
    finally:
        os.close(fd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("measure_gossip_store_salvage: no GPU")
    import lightning_b200 as LB
    from tests import gossip_store_salvage as sv
    from tests import util
    name, power = card()
    emul = util.load_emul()
    emul.emul_gs_salvage_sound_plain.restype = ctypes.c_uint64
    emul.emul_gs_salvage_sound_plain.argtypes = [ctypes.c_char_p, ctypes.c_uint64]
    eng = LB.SigVerifier(0)
    out = {"metric": "gossip_store_salvage", "gpu": name, "power_limit": power, "stores": {}}
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gossip_store")
        for k, store in stores().items():
            _, acts, s = eng.salvage_gossip_store(store)
            if k.startswith("fixture"):
                assert s["sound"] == len(sv.sound_offsets(store))
            row = {"bytes": len(store), "sound": s["sound"], "breaks": s["breaks"], "restored": s["restored"]}
            t = {x: [] for x in ("filter", "crc", "walk", "mem", "sfd", "rfd", "cpu")}
            for r in range(a.reps + 2):
                eng.set_profiling(True)
                eng.salvage_gossip_store(store)
                f, c, w = eng.last_gossip_salvage_timing()
                eng.set_profiling(False)
                t0 = time.perf_counter()
                eng.salvage_gossip_store(store)
                mem = (time.perf_counter() - t0) * 1e3
                sfd, (ps, vs, n1) = file_call(path, store, eng.salvage_gossip_store_fd)
                rfd, (pr, n2) = file_call(path, store, eng.repair_gossip_store_fd)
                assert vs == s
                if r < 2:
                    continue
                for key, v in (("filter", f), ("crc", c), ("walk", w), ("mem", mem), ("sfd", sfd), ("rfd", rfd)):
                    t[key].append(v)
            for r in range(3):
                t0 = time.perf_counter()
                n = emul.emul_gs_salvage_sound_plain(store, len(store))
                t["cpu"].append((time.perf_counter() - t0) * 1e3)
                assert n == s["sound"]
            row.update(filter_ms=med(t["filter"]), crc_ms=med(t["crc"]), walk_ms=med(t["walk"]), in_memory_ms=med(t["mem"]),
                       salvage_fd_ms=med(t["sfd"]), repair_fd_ms=med(t["rfd"]), cpu_scan_ms=med(t["cpu"]),
                       new_len_salvage=n1, new_len_repair=n2)
            out["stores"][k] = row
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
