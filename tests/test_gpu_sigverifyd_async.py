"""GPU: the drop-in's non-blocking client mode against the real verifier subdaemon and engine.  One client process keeps a
window of 64 tickets in flight (bolt12_check_signature_start, check_tx_sig_start, sigcheck_gossip_batch_start) and every
answer must equal the blocking drop-in's, in client mode (no visible GPU: opening a context would abort) and in process,
and the answers CLN gave: the reference's status per BOLT12 stream recorded in tests/golden/bolt12_vectors.npz, BOLT #3's
own HTLC signatures over libwally's sighashes (tests/golden/bolt3_htlc_txs.json), and gossipd's decisions on the
bit-flipped gossip fixture replayed from the CLN tape test_gpu_gossip_burst.py recorded.  The daemon's stats must show
requests of the one client coalesced into shared launches."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import lightning_b200 as L
from tests import bolt12, gossip, oracle_replay, txsig
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)
from tests.sigverifyd_daemon import stats as _stats
from tests.test_gpu_gossip_burst import TESTNET, burst_model, flipped_fixture

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SK = bytes([0x31]) * 32

DRIVER = r"""
import ctypes, json, select, sys
from tests import bolt12
from tests.txsig import WallyIn, WallyOut, WallyTx, BitcoinTx
lib = ctypes.CDLL(sys.argv[1])
sc = json.load(open(sys.argv[2]))
vp, sz, b_ = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_bool
DONE = ctypes.CFUNCTYPE(None, vp)
for f in ("check_tx_sig", "bolt12_check_signature"):
    getattr(lib, f).restype = b_
    getattr(lib, f + "_start").restype = ctypes.c_uint64
lib.sigcheck_gossip_batch_start.restype = ctypes.c_uint64
lib.check_tx_sig.argtypes = [vp, sz, vp, vp, vp, vp]
lib.check_tx_sig_start.argtypes = [vp, sz, vp, vp, vp, vp, vp, DONE, vp]
lib.bolt12_check_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp]
lib.bolt12_check_signature_start.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp, vp, DONE, vp]
lib.sigcheck_gossip_batch.argtypes = [vp, vp, vp, sz, vp, vp, vp]
lib.sigcheck_gossip_batch_start.argtypes = [vp, vp, vp, sz, vp, vp, vp, DONE, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
lib.cln_sigverify_events.restype = ctypes.c_short
lib.cln_sigverify_process.restype = sz
keep, sizes = [], {}
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: sizes[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
H = bytes.fromhex
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return ctypes.addressof(x)
def opaque(xy):  # secp256k1_pubkey / _ecdsa_signature: two 32-byte numbers as little-endian limbs
    return xy[31::-1] + xy[:31:-1]
done = []
cb = DONE(lambda arg: done.append(arg))

def run(checks):
    # checks: (start, blocking, answer) per check; a window of 64 tickets, then the same checks blocking
    tickets = []
    for start, _, _ in checks:
        while lib.cln_sigverify_process() >= 64:
            p = select.poll()
            p.register(lib.cln_sigverify_fd(), lib.cln_sigverify_events())
            p.poll()
        tickets.append(start(len(tickets) + 1))
    lib.cln_sigverify_drain()
    live = [i + 1 for i, t in enumerate(tickets) if t]
    assert done == live, "callbacks out of ticket order, or not exactly once"
    del done[:]
    return [answer() for _, _, answer in checks], [blocking() for _, blocking, _ in checks], sum(t > 0 for t in tickets)

out = {}
# BOLT12: the fixture's streams as tlv_field arrays
calls = []
for i, stream, xonly, sig, mn, fn in sc["bolt12"]:
    fields = bolt12.parse_fields(H(stream))
    arr = (ctypes.c_uint64 * max(4 * len(fields), 1))()
    for j, (t, _vo, v) in enumerate(fields):
        arr[4 * j + 1], arr[4 * j + 2], arr[4 * j + 3] = t, len(v), buf(v) if v else 0
    keep.append(arr)
    sizes[ctypes.addressof(arr)] = 4 * 8 * len(fields)
    a = (ctypes.addressof(arr), mn.encode(), fn.encode(), buf(opaque(H(xonly))), buf(H(sig)))
    ok = b_(False)
    keep.append(ok)
    calls.append((lambda arg, a=a, ok=ok: lib.bolt12_check_signature_start(*a, ctypes.addressof(ok), cb, arg),
                  lambda a=a: bool(lib.bolt12_check_signature(*a)), lambda ok=ok: bool(ok.value)))
out["bolt12"] = run(calls)
# check_tx_sig on one-input one-output transactions
calls = []
for c in sc["tx"]:
    ins = (WallyIn * 1)()
    ins[0].txhash[:] = list(H(c["prev_txid"])); ins[0].index = c["prev_index"]; ins[0].sequence = c["sequence"]
    outs = (WallyOut * 1)()
    o = H(c["out_script"])
    outs[0].satoshi = c["output_amount"]; outs[0].script = buf(o); outs[0].script_len = len(o)
    w = WallyTx(c["version"], c["locktime"], ctypes.addressof(ins), 1, 1, ctypes.addressof(outs), 1, 1)
    tx = BitcoinTx(ctypes.pointer(w), None, None)
    keep.extend([ins, outs, w, tx])
    sizes[ctypes.addressof(tx)] = c["input_amount"]
    ws = buf(H(c["wscript"]))
    sizes[ws] = len(H(c["wscript"]))
    a = (ctypes.addressof(tx), 0, None, ws, buf(opaque(H(c["xy"]))), buf(opaque(H(c["sig64"])) + c["type"].to_bytes(4, "little")))
    ok = b_(False)
    keep.append(ok)
    calls.append((lambda arg, a=a, ok=ok: lib.check_tx_sig_start(*a, ctypes.addressof(ok), cb, arg),
                  lambda a=a: bool(lib.check_tx_sig(*a)), lambda ok=ok: bool(ok.value)))
out["tx"] = run(calls)
# gossip bursts
calls = []
for b in sc["bursts"]:
    msgs = [H(m) for m in b["msgs"]]
    n = len(msgs)
    ptrs = buf(b"".join(buf(m).to_bytes(8, "little") for m in msgs))
    lens = buf(b"".join(len(m).to_bytes(8, "little") for m in msgs))
    a = (buf(H(sc["chain"])), ptrs, lens, n, buf(H(b["kinds"])) if b["kinds"] else None, buf(H(b["signers"])) if b["signers"] else None)
    st = (ctypes.c_int * n)()
    keep.append(st)
    def blocking(a=a, n=n):
        s = (ctypes.c_int * n)()
        lib.sigcheck_gossip_batch(*a, s)
        return list(s)
    calls.append((lambda arg, a=a, st=st: lib.sigcheck_gossip_batch_start(*a, ctypes.addressof(st), cb, arg), blocking,
                  lambda st=st: list(st)))
out["gossip"] = run(calls)
print(json.dumps(out))
"""


def _scenario(engine, tmp_path):
    """what the driver checks, with the answers CLN gave"""
    rng = np.random.default_rng(9)
    sc, want = dict(chain=TESTNET.hex()), {}
    # BOLT12: every 3rd stream of the fixture CLN parsed, every 4th signature with a flipped bit (then CLN's answer is 0)
    fx = bolt12.load_fixture()
    streams = bolt12.streams(fx)
    sc["bolt12"], want["bolt12"] = [], []
    for i in range(0, len(streams), 3):
        conv = txsig.ecc.pubkey_convert(b"\x02" + fx["xonly"][i].tobytes())
        if fx["status"][i] < 0 or conv is None:
            continue
        sig = bytearray(fx["sig"][i].tobytes())
        bad = len(sc["bolt12"]) % 4 == 1
        if bad:
            sig[int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
        mn, fn = bolt12.NAMES[fx["names"][i]]
        sc["bolt12"].append((i, streams[i].hex(), conv[1].hex(), bytes(sig).hex(), mn.decode(), fn.decode()))
        want["bolt12"].append(bool(fx["status"][i] == 1) and not bad)
    # BOLT #3's HTLC transactions: both parties' signatures under SIGHASH_ALL (valid), corrupted, under
    # SIGHASH_SINGLE|ANYONECANPAY (signed for ALL: invalid), and signatures made here under SINGLE|ANYONECANPAY
    recs = json.load(open(os.path.join(GOLD, "bolt3_htlc_txs.json")))
    sc["tx"], want["tx"] = [], []
    pub33, myxy = txsig.ecc.pubkey_create(SK)
    for r in recs:
        base = {k: r[k] for k in ("version", "locktime", "sequence", "prev_txid", "prev_index", "wscript", "out_script",
                                  "input_amount", "output_amount")}
        for who in (0, 1):
            xy = txsig.ecc.pubkey_convert(bytes.fromhex(r["sigs"][who]["pub33"]))[1].hex()
            sig = bytes.fromhex(r["sigs"][who]["sig64"])
            bad = bytes([sig[0]]) + bytes([sig[1] ^ 4]) + sig[2:]
            for s, t, ok in ((sig, 1, True), (bad, 1, False), (sig, 0x83, False)):
                sc["tx"].append(dict(base, xy=xy, sig64=s.hex(), type=t))
                want["tx"].append(ok)
        t = (L.SvTx * 1)()
        x = t[0]
        x.version, x.locktime, x.sequence, x.sighash_type = r["version"], r["locktime"], r["sequence"], 0x83
        x.prev_txid[:] = list(bytes.fromhex(r["prev_txid"]))
        x.prev_index, x.input_amount, x.output_amount = r["prev_index"], r["input_amount"], r["output_amount"]
        ws, os_ = bytes.fromhex(r["wscript"]), bytes.fromhex(r["out_script"])
        x.script_len, x.out_script_off, x.out_script_len = len(ws), len(ws), len(os_)
        _, sig = txsig.sign(engine, 1, SK, t, ws + os_)
        sig = sig[0].tobytes()
        for s, ok in ((sig, True), (sig[:63] + bytes([sig[63] ^ 1]), False)):
            sc["tx"].append(dict(base, xy=myxy.hex(), sig64=s.hex(), type=0x83))
            want["tx"].append(ok)
    # gossip: the bit-flipped fixture as one burst (its CLN answers come from the tape), and slices of the fixture
    batch, kinds, signers = flipped_fixture()
    sc["bursts"] = [dict(msgs=[m.hex() for m in batch], kinds=kinds.tobytes().hex(), signers=signers.tobytes().hex())]
    msgs = gossip.load_subset()
    for s in range(0, len(msgs), 73):
        sc["bursts"].append(dict(msgs=[m.hex() for m in msgs[s:s + 73]], kinds=None, signers=None))
    want["gossip_whole"] = (batch, kinds, signers)
    path = tmp_path / "scenario.json"
    path.write_text(json.dumps(sc))
    return str(path), want


def _gossipd(cln, batch, kinds, signers):
    """gossipd's decisions on the bit-flipped fixture, replayed from the tape test_gpu_gossip_burst.py recorded for these
    same inputs (every recorded call must be asked for)"""
    here = (oracle_replay._CURRENT[0], oracle_replay._CURRENT[1])
    oracle_replay.begin_test("test_gpu_gossip_burst", "test_burst_vs_gossipd")
    try:
        got = burst_model(cln, batch, TESTNET, kinds, signers)
        tape = cln.tape()
        assert tape is not None and tape.pos == len(tape.meta)
    finally:
        oracle_replay.begin_test(*here)
    return got


def _run(lib, path, tmp_path, env):
    r = subprocess.run([sys.executable, "-c", DRIVER, lib, path], env=env, cwd=str(tmp_path), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def test_window_of_tickets(engine, cln, daemon, tmp_path):
    from lightning_b200 import build
    path, want = _scenario(engine, tmp_path)
    base = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base.pop("CLN_SIGVERIFYD_SOCKET", None)
    remote = _run(build.LIB, path, tmp_path, dict(base, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES=""))
    local = _run(build.LIB, path, tmp_path, base)
    n = {k: len(remote[k][0]) for k in ("bolt12", "tx", "gossip")}
    for k in n:
        tickets, blocking, started = remote[k]
        assert tickets == blocking, k
        assert started == n[k], k  # nothing here is gated: every check was a ticket
        assert local[k][0] == local[k][1] == blocking and local[k][2] == 0, k  # in process: answered at once
    assert remote["bolt12"][0] == want["bolt12"] and 50 < sum(want["bolt12"]) < n["bolt12"]
    assert remote["tx"][0] == want["tx"] and n["tx"] == 40
    whole = remote["gossip"][0][0]
    assert whole == _gossipd(cln, *want["gossip_whole"])
    msgs = gossip.load_subset()
    assert remote["gossip"][0][1:] == [engine.verify_gossip_burst(msgs[s:s + 73], TESTNET).tolist()
                                       for s in range(0, len(msgs), 73)]
    st = _stats(daemon)
    assert st["requests"] == 2 * sum(n.values()), st
    assert st["max_coalesced"] > 1, st  # one client's tickets shared launches
