"""The verifier subdaemon and the drop-in on the fake engine (tests/host_emul/fake_engine*.c), for the CPU tests: the
fake's answers restated in Python, request builders with the replies the fake dictates, the builds, the fake's call log
and trace, and the client process of the drop-in's gossip_store calls."""
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

from lightning_b200 import build
from lightning_b200 import sigverifyd_wire as W
from lightning_b200.engine import SvGossipPruneSummary
from tests import txsig
from tests.gossip_store import EOF, INCOMPLETE, NO_AMOUNT, PARTIAL, ST_ENDED
from tests.gossip_store_prune import REASONS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HE = os.path.join(ROOT, "tests", "host_emul")
FAKE = os.path.join(HE, "fake_engine.c")
FAKE_GRIND = os.path.join(HE, "fake_engine_grind.c")
FAKE_BOLT11 = os.path.join(HE, "fake_engine_bolt11.c")
FAKE_PRUNE = os.path.join(HE, "fake_engine_prune.c")
STORE_FD = os.path.join(build.CSRC, "gossip_store_fd.c")
SALVAGE_FD = os.path.join(build.CSRC, "gossip_salvage_fd.c")
KS = {0: 33, 1: 64, 2: 32}
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")
TAGS = [(b"invoice", b"signature"), (b"invoice_request", b"signature"), (b"offer", b"signature")]
PRUNE = "sv_prune_gossip_store_host"
FIELDS = [f for f, _ in SvGossipPruneSummary._fields_]
MAX_PRUNE_STORE = 4 << 30  # sigverifyd_proto.h


# ---- the fake engine's functions (fake_engine.h) ---------------------------------------------------------------------
def fnv(data, h=0xcbf29ce484222325):
    for b in data:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def fill(h, n):
    return bytes(fnv(bytes([k]), h) & 0xFF for k in range(n))


def wire(status):
    return bytes(s & 0xFF for s in status)


def le(v, n):
    return int(v).to_bytes(n, "little")


def rev(b):
    """libsecp256k1's opaque structs hold two 32-byte numbers as little-endian limbs"""
    return b[31::-1] + b[:31:-1]


def tx_hash(kind, key, sig, f, spans):
    """f: version, locktime, sequence, sighash_type, prev_txid, prev_index, flags, input_amount, output_amount"""
    return fnv(bytes([kind]) + key + sig + b"".join(le(f[k], 4) for k in ("version", "locktime", "sequence", "sighash_type")) +
               f["prev_txid"] + le(f["prev_index"], 4) + le(f["flags"], 4) + le(f["input_amount"], 8) +
               le(f["output_amount"], 8) + b"".join(le(len(s), 4) + s for s in spans))


# ---- requests and the replies the fake dictates ---------------------------------------------------------------------
def rand(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def verify_req(rng, rid, kind, n):
    h, k, s = rand(rng, 32 * n), rand(rng, KS[kind] * n), rand(rng, 64 * n)
    ks = KS[kind]
    v = bytes(fnv(bytes([kind]) + h[32 * i:32 * i + 32] + k[ks * i:ks * i + ks] + s[64 * i:64 * i + 64]) % 3 for i in range(n))
    return (W.encode("sigverifyd_verify", req_id=rid, kind=kind, n=n, hashes=h, keylen=ks * n, keys=k, sigs=s),
            ("sigverifyd_verify_reply", dict(req_id=rid, n=n, verdicts=v)))


def bolt12_req(rng, rid, mn, fn, sizes, want):
    n = len(sizes)
    streams = [rand(rng, x) for x in sizes]
    xo, sg = rand(rng, 32 * n), rand(rng, 64 * n)
    hs = [fnv(mn + b"\0" + fn + b"\0" + streams[i] + xo[32 * i:32 * i + 32] + sg[64 * i:64 * i + 64]) for i in range(n)]
    blob = b"".join(streams)
    frame = W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn, n=n,
                     lens=sizes, bloblen=len(blob), blob=blob, xonly=xo, sigs=sg, want_sighash=want)
    return frame, ("sigverifyd_bolt12_reply", dict(req_id=rid, n=n, status=wire(h % 3 - 1 for h in hs),
                                                   nsighash=n if want else 0,
                                                   sighashes=b"".join(fill(h, 32) for h in hs) if want else b""))


def tx_req(rng, rid, kind, spans, want):
    """spans: per transaction the lengths of (script, outputs, outpoints, sequences)"""
    n = len(spans)
    key, sigs = rand(rng, KS[kind]), rand(rng, 64 * n)
    recs, data, hs = [], [], []
    for i, sp in enumerate(spans):
        f = dict(version=int(rng.integers(1, 3)), locktime=int(rng.integers(0, 2**32)), sequence=int(rng.integers(0, 2**32)),
                 sighash_type=int(rng.choice([1, 3, 0x83])), prev_txid=rand(rng, 32), prev_index=int(rng.integers(0, 9)),
                 flags=1 | (2 if sp[2] or sp[3] else 0), input_amount=int(rng.integers(0, 2**62)),
                 output_amount=int(rng.integers(0, 2**62)))
        b = [rand(rng, x) for x in sp]
        recs.append(f)
        data += b
        hs.append(tx_hash(kind, key, sigs[64 * i:64 * i + 64], f, b))
    kw = {k: [r[k] for r in recs] for k in txsig.U32_FIELDS}
    blob = b"".join(data)
    frame = W.encode("sigverifyd_tx", req_id=rid, kind=kind, keylen=len(key), key=key, n=n,
                     prev_txid=b"".join(r["prev_txid"] for r in recs), input_amount=[r["input_amount"] for r in recs],
                     output_amount=[r["output_amount"] for r in recs], script_len=[s[0] for s in spans],
                     outputs_len=[s[1] for s in spans], prevouts_len=[s[2] for s in spans],
                     sequences_len=[s[3] for s in spans], bloblen=len(blob), blob=blob, sigs=sigs, want_sighash=want, **kw)
    return frame, ("sigverifyd_tx_reply", dict(req_id=rid, n=n, verdicts=bytes(h % 3 for h in hs), nsighash=n if want else 0,
                                               sighashes=b"".join(fill(h, 32) for h in hs) if want else b""))


def sha_req(rng, rid, sizes):
    bufs = [rand(rng, x) for x in sizes]
    blob = b"".join(bufs)
    return (W.encode("sigverifyd_sha256d", req_id=rid, n=len(bufs), lens=sizes, bloblen=len(blob), blob=blob),
            ("sigverifyd_sha256d_reply", dict(req_id=rid, n=len(bufs), hashes=b"".join(fill(fnv(b), 32) for b in bufs))))


def key_req(rng, rid, n):
    keys = rand(rng, 33 * n)
    hs = [fnv(keys[33 * i:33 * i + 33]) for i in range(n)]
    return (W.encode("sigverifyd_pubkey", req_id=rid, n=n, keys=keys),
            ("sigverifyd_pubkey_reply", dict(req_id=rid, n=n, ok=bytes(h % 3 for h in hs),
                                             xy=b"".join(fill(h, 64) for h in hs))))


def gossip_req(rng, rid, n):
    msgs = [rand(rng, int(rng.integers(2, 300))) for _ in range(n)]
    sg = rand(rng, 33 * n)
    st = [fnv(m + sg[33 * i:33 * i + 33]) % 6 - 1 for i, m in enumerate(msgs)]
    blob = b"".join(msgs)
    return (W.encode("sigverifyd_gossip", req_id=rid, n=n, lens=[len(m) for m in msgs], signers=sg, bloblen=len(blob),
                     blob=blob), ("sigverifyd_gossip_reply", dict(req_id=rid, n=n, status=wire(st))))


def burst_req(rng, rid, n):
    msgs = [rand(rng, int(rng.integers(2, 300))) for _ in range(n)]
    kinds, sg = bytes(int(x) for x in rng.integers(0, 3, size=n)), rand(rng, 33 * n)
    st = [fnv(TESTNET + m + kinds[i:i + 1] + sg[33 * i:33 * i + 33]) % 10 - 4 for i, m in enumerate(msgs)]
    blob = b"".join(msgs)
    return (W.encode("sigverifyd_gossip_burst", req_id=rid, chain_hash=TESTNET, n=n, lens=[len(m) for m in msgs],
                     signer_kind=kinds, signers=sg, bloblen=len(blob), blob=blob),
            ("sigverifyd_gossip_burst_reply", dict(req_id=rid, n=n, status=wire(st))))


def prune_frame(rid, length, chain=TESTNET):
    return W.encode("sigverifyd_gossip_store_prune", req_id=rid, has_chain=1 if chain else 0, chain_hash=chain or bytes(32),
                    len=length)


def patched(frame, at, value):
    """frame with the bytes at offset `at` of its message replaced"""
    body = bytearray(frame[4:])
    body[at:at + len(value)] = value
    return len(body).to_bytes(4, "big") + bytes(body)


def short(frame):
    """frame one byte short of its fields"""
    body = frame[4:-1]
    return len(body).to_bytes(4, "big") + body


def roundtrip(c, reqs):
    """sends the frames in one write, reads one reply per frame and checks each against what the fake dictates"""
    c.sendall(b"".join(f for f, _ in reqs))
    for frame, want in reqs:
        got = W.read_msg(c)
        if want is None:  # a stats request: its counters are checked elsewhere
            assert got[0] == "sigverifyd_stats_reply" and got[1]["req_id"] == W.decode(frame[4:])[1]["req_id"]
        else:
            assert got == want, (got[0], got[1].get("req_id"), want[0], want[1]["req_id"])


# ---- stores and what the fake prune makes of them (fake_engine_prune.c) ----------------------------------------------
def make_store(rng, n, version=0x0C, tail=0):
    """a version byte, n records of random messages (some already deleted), then `tail` bytes of a record cut short"""
    out = bytearray([version])
    for _ in range(n):
        flags = (0x8000 if rng.random() < 0.15 else 0) | 0x2000
        msg = rng.integers(0, 256, size=int(rng.integers(2, 300)), dtype=np.uint8).tobytes()
        out += flags.to_bytes(2, "big") + len(msg).to_bytes(2, "big") + rng.integers(0, 2**32, size=2, dtype=np.uint64).astype(
            ">u4").tobytes() + msg
    if tail:
        out += (0x2000).to_bytes(2, "big") + (tail + 100).to_bytes(2, "big") + bytes(8) + bytes(tail)
    return bytes(out)


def fake_prune(store):
    """(the pruned store, the summary dict) the fake engine gives"""
    out, s = bytearray(store), dict.fromkeys(FIELDS, 0)
    off, r = 1, 0
    s["version"], s["stop"] = store[0], EOF
    while off + 12 < len(store):
        flags, mlen = struct.unpack(">HH", store[off:off + 4])
        typ = struct.unpack(">H", store[off + 12:off + 14])[0] if off + 14 <= len(store) else 0
        if not flags & 0x2000:
            s["stop"] = INCOMPLETE
            break
        if not flags & 0x8000:
            stop = PARTIAL if off + 12 + mlen > len(store) else ST_ENDED if typ == 4105 else \
                NO_AMOUNT if typ == 256 and off + 12 + mlen + 22 > len(store) else None
            if stop:
                s["stop"] = stop
                break
        if r % 3 == 1 and not store[off] & 0x80:
            why = 1 + (r // 3) % 8
            out[off] |= 0x80
            s["pruned"] += 1
            s[REASONS[why - 1]] += 1
            s["reverified"] += why == 6
        r += 1
        off += 12 + mlen
    s["end_offset"], s["records"] = off, r
    return bytes(out), s


def tail_rule(stop, end_offset, length):
    """where a repair ends a store of `length` bytes whose prune stopped at `stop` / `end_offset`, from the summary alone
    (the first three rules of sv_repair_gossip_store_fd in include/cln_sigverify.h)"""
    if stop in (INCOMPLETE, PARTIAL, NO_AMOUNT):
        return min(end_offset, length)
    if stop == EOF and end_offset < length:
        return end_offset
    return length


def room_back_off(pruned, cut):
    """the last rule: while the first live channel_announcement of pruned[:cut] has fewer than 22 bytes after it before
    cut (no room for its amount record), the store ends at it"""
    while True:
        off, at = 1, cut
        while off + 14 <= cut:
            flags, mlen = struct.unpack(">HH", pruned[off:off + 4])
            typ = struct.unpack(">H", pruned[off + 12:off + 14])[0]
            if off + 12 + mlen > cut:
                break
            if not flags & 0x8000 and typ == 256 and off + 12 + mlen + 22 > cut:
                at = off
                break
            off += 12 + mlen
        if at == cut:
            return cut
        cut = at


def cut_rule(pruned, s):
    """sv_gossip_prune_cut: the tail rule, then the back-off when it cuts"""
    cut = tail_rule(s["stop"], s["end_offset"], len(pruned))
    return room_back_off(pruned, cut) if cut < len(pruned) else cut


# ---- builds ----------------------------------------------------------------------------------------------------------
def gcc(args, cc="gcc"):
    r = subprocess.run([cc] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def daemon(path, *sources, limits=None):
    """cln_sigverifyd on the fake engine and the optional parts in `sources`, with the per-call `limits` overridden"""
    gcc(build.DAEMON_CFLAGS + ["-D%s=%d" % kv for kv in (limits or {}).items()] +
        [os.path.join(build.CSRC, "sigverifyd.c"), FAKE, *sources, "-o", str(path)])
    return str(path)


def dropin(path, *sources, client=True):
    """the drop-in library on the fake engine and `sources`: in client mode (its sv_create aborts) or in-process"""
    gcc(build.DROPIN_CFLAGS + ["-shared"] + (["-DFAKE_ENGINE_NO_CONTEXT"] if client else []) +
        [os.path.join(build.CSRC, "cln_dropin.c"), FAKE, *sources, "-o", str(path)])
    return str(path)


def fake_salvage_o(d):
    """the CPU salvage (fake_engine_salvage.cpp), compiled"""
    o = str(d / "fake_engine_salvage.o")
    gcc(["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-c", os.path.join(HE, "fake_engine_salvage.cpp"),
         "-o", o], cc="g++")
    return o


def store_bins(d, salvage=False):
    """the daemon, the in-process and the client-mode drop-in with the fake prune and the fd layer, and with the CPU
    salvage when asked"""
    parts = [FAKE_PRUNE, STORE_FD] + ([SALVAGE_FD, fake_salvage_o(d), "-lstdc++"] if salvage else [])
    return dict(daemon=daemon(d / "cln_sigverifyd", *parts), inproc=dropin(d / "libdropin_inproc.so", *parts, client=False),
                client=dropin(d / "libdropin_client.so", *parts))


# ---- the fake's log and trace ----------------------------------------------------------------------------------------
def env(tmp_path, delays=None):
    """the fake's variables: its log in tmp_path/engine.log, its trace in tmp_path/trace, `delays` {function: ms}"""
    return dict(os.environ, FAKE_ENGINE_LOG=str(tmp_path / "engine.log"), FAKE_ENGINE_TRACE=str(tmp_path / "trace"),
                FAKE_ENGINE_DELAY=",".join("%s=%d" % kv for kv in (delays or {}).items()))


def calls(log):
    """the fake's log: (function, kind, n, blob bytes) per call"""
    if not log.exists():
        return []
    return [(f, int(k), int(n), int(b)) for f, k, n, b in (line.split() for line in log.read_text().splitlines())]


def trace(tmp_path):
    """the fake's trace: (event, function, context) per line"""
    p = tmp_path / "trace"
    return [tuple(line.split()) for line in p.read_text().splitlines()] if p.exists() else []


def wait_trace(tmp_path, pred, timeout=30):
    """the trace once pred(trace) holds"""
    end = time.time() + timeout
    while time.time() < end:
        t = trace(tmp_path)
        if pred(t):
            return t
        time.sleep(0.01)
    raise AssertionError("trace condition not reached: %r" % (trace(tmp_path),))


def begun(fn, count=1):
    return lambda t: sum(1 for e in t if e[:2] == ("begin", fn)) >= count


def nfds(proc):
    return len(os.listdir("/proc/%d/fd" % proc.pid))


def back_to(proc, base, timeout=10):
    """the daemon's descriptor count, once it is back at base (or the timeout passed)"""
    end = time.time() + timeout
    while nfds(proc) != base and time.time() < end:
        time.sleep(0.02)
    return nfds(proc)


# ---- the drop-in's gossip_store calls in a process of their own ------------------------------------------------------
CLIENT = r"""
import ctypes, json, os, sys
from lightning_b200.engine import SvGossipPruneSummary, SvGossipSalvageSummary
lib = ctypes.CDLL(sys.argv[1], use_errno=True)
S, V, U64 = ctypes.POINTER(SvGossipPruneSummary), ctypes.POINTER(SvGossipSalvageSummary), ctypes.POINTER(ctypes.c_uint64)
for fn, outs in ((lib.gossip_store_prune, [S]), (lib.gossip_store_repair, [S, U64]), (lib.gossip_store_salvage, [S, V, U64])):
    fn.restype = ctypes.c_bool
    fn.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_void_p] + outs
lib.cln_sigverify_connect.argtypes = [ctypes.c_char_p]
mode = sys.argv[2]
if mode.startswith("sock:"):
    assert lib.cln_sigverify_connect(mode[5:].encode()) == 0
elif mode.startswith("fd:"):
    assert lib.cln_sigverify_connect_fd(int(mode[3:])) == 0
out = []
for c in json.load(open(sys.argv[3])):
    if c["kind"] == "pipe":
        fd, w = os.pipe()
        os.write(w, bytes(64))
    elif c["kind"] == "closed":
        fd = os.open(os.devnull, os.O_RDONLY)
        os.close(fd)
    else:
        fd = os.open(c["path"], os.O_RDWR if c["kind"] == "rw" else os.O_RDONLY)
    s, v, n = SvGossipPruneSummary(), SvGossipSalvageSummary(), ctypes.c_uint64(12345)
    chain = bytes.fromhex(c["chain"]) if c["chain"] else None
    fn, outs = {"prune": (lib.gossip_store_prune, [s]), "repair": (lib.gossip_store_repair, [s, n]),
                "salvage": (lib.gossip_store_salvage, [s, v, n])}[c["op"]]
    ok = fn(fd, c["len"], chain, *map(ctypes.byref, outs))
    e = ctypes.get_errno()
    if c["kind"] != "closed":
        os.close(fd)
    if c["kind"] == "pipe":
        os.close(w)
    row = [ok, 0 if ok else e, {f: getattr(s, f) for f, _ in s._fields_} if ok else None]
    if c["op"] == "salvage":
        row.append({f: getattr(v, f) for f, _ in v._fields_} if ok else None)
    out.append(row + [n.value if ok and c["op"] != "prune" else None])
print(json.dumps(out))
"""


def run_client(tmp_path, lib, mode, cases, pass_fds=(), check=True):
    """each case's [ok, errno, summary, new_len (a repair's or salvage's, else None)] from a process of its own, a
    salvage's with its salvage summary before new_len; mode "inproc", "sock:<path>" or "fd:<n>" """
    path = tmp_path / ("cases%d.json" % time.monotonic_ns())
    path.write_text(json.dumps(cases))
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", CLIENT, lib, mode, str(path)], env=env, capture_output=True, text=True,
                       timeout=300, pass_fds=pass_fds)
    if check:
        assert r.returncode == 0, r.stderr[-3000:]
        return json.loads(r.stdout)
    return r


def case(path, length=None, chain=TESTNET, kind="rw", op="prune"):
    """a gossip_store_prune, _repair or _salvage call (op) on the file at path, or on a pipe or a closed descriptor (kind
    "pipe", "closed")"""
    return dict(kind=kind, path=str(path), len=os.path.getsize(path) if length is None else length,
                chain=chain.hex() if chain else None, op=op)


def salvage_case(path, length=None, chain=TESTNET, kind="rw"):
    return case(path, length, chain, kind, op="salvage")
