"""CPU: the sigverifyd_fee_grind message (onchaind's HTLC fee grind through the verifier subdaemon).  The Python codec
reads both messages back; the daemon, built against the fake engine (tests/host_emul/fake_engine.c), routes each grind to
one sv_grind_tx_fee_host call with the request's own bytes, answers in request order among other traffic, and refuses
malformed requests; the drop-in's check_tx_sig_grind_fee in client mode sends the record check_tx_sig builds.  The fake's
grind is tests/host_emul/fake_engine_grind.c, linked beside the fake engine; a daemon linked without it refuses grinds."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.sigverifyd_fake import FAKE_GRIND, KS, calls, fnv, le, patched, rand, rev, roundtrip, short, tx_req, verify_req

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    """the daemon and the client-mode drop-in library on the fake engine with its grind, and a daemon without the grind"""
    d = tmp_path_factory.mktemp("fake_grind")
    return dict(daemon=sf.daemon(d / "cln_sigverifyd", FAKE_GRIND), lib=sf.dropin(d / "libcln_dropin_fake.so", FAKE_GRIND),
                bare=sf.daemon(d / "cln_sigverifyd_bare"))


@pytest.fixture
def fake(tmp_path, bins):
    """a daemon on the fake engine with its grind, and the engine's call log"""
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        yield sock, tmp_path / "engine.log"


def grind_answer(kind, key, sig, f, script, out_script, weight, lo, hi):
    """what the fake engine returns: (found, feerate, fee)"""
    h = fnv(bytes([kind]) + key + sig + b"".join(le(f[k], 4) for k in ("version", "locktime", "sequence", "sighash_type")) +
            f["prev_txid"] + le(f["prev_index"], 4) + le(f["input_amount"], 8) + le(len(script), 4) + script +
            le(len(out_script), 4) + out_script + le(weight, 8) + le(lo, 4) + le(hi, 4))
    if lo > hi or h % 3 == 0:
        return 0, 0, 0
    rate = lo + (h >> 8) % (hi - lo + 1)
    return 1, rate, rate * weight // 1000


def grind_req(rng, rid, kind, script_len=140, out_len=34, weight=663, lo=253, hi=125000):
    f = dict(version=2, locktime=int(rng.integers(0, 2**31)), sequence=int(rng.integers(0, 2)),
             sighash_type=int(rng.choice([1, 0x83])), prev_index=int(rng.integers(0, 600)), prev_txid=rand(rng, 32),
             input_amount=int(rng.integers(0, 2**40)))
    key, sig, script, out_script = rand(rng, KS[kind]), rand(rng, 64), rand(rng, script_len), rand(rng, out_len)
    frame = W.encode("sigverifyd_fee_grind", req_id=rid, kind=kind, keylen=len(key), key=key, script_len=len(script),
                     script=script, out_script_len=len(out_script), out_script=out_script, sig=sig, weight=weight,
                     min_feerate=lo, max_feerate=hi, **f)
    found, rate, fee = grind_answer(kind, key, sig, f, script, out_script, weight, lo, hi)
    return frame, ("sigverifyd_fee_grind_reply", dict(req_id=rid, found=found, feerate=rate, fee=fee))


def test_codec_round_trip():
    """Python encode -> decode gives the fields back, for both replies (found and not found)"""
    rng = np.random.default_rng(1)
    frame, _ = grind_req(rng, 77, 1, script_len=0, out_len=300)
    name, m = W.decode(frame[4:])
    assert name == "sigverifyd_fee_grind" and m["req_id"] == 77 and m["kind"] == 1 and m["script_len"] == 0
    assert len(m["out_script"]) == 300 and len(m["sig"]) == 64 and m["min_feerate"] == 253
    for found, rate, fee in ((1, 0xFFFFFFFF, 2**64 - 1), (0, 0, 0)):
        r = W.encode("sigverifyd_fee_grind_reply", req_id=5, found=found, feerate=rate, fee=fee)
        assert W.decode(r[4:]) == ("sigverifyd_fee_grind_reply", dict(req_id=5, found=found, feerate=rate, fee=fee))


def test_daemon_routes_each_grind_to_one_engine_call(fake):
    """grinds of both key kinds written at once with tx and verify requests: every reply is the fake's for that
    request, in order, and each grind is one sv_grind_tx_fee_host call with its own kind and spans"""
    sock, log = fake
    rng = np.random.default_rng(2)
    reqs = [grind_req(rng, 1, 0), tx_req(rng, 2, 1, [(10, 20, 0, 0)], 0), grind_req(rng, 3, 1, 71, 22, 703, 0, 0xFFFFFFFF),
            verify_req(rng, 4, 0, 2), grind_req(rng, 5, 0, 0, 0, 0, 9, 8), grind_req(rng, 6, 1, 300, 34, 1, 10, 10)]
    c = sigverifyd_daemon.connect(sock)
    roundtrip(c, reqs)
    c.close()
    grinds = [x for x in calls(log) if x[0] == "sv_grind_tx_fee_host"]
    assert grinds == [("sv_grind_tx_fee_host", 0, 1, 174), ("sv_grind_tx_fee_host", 0, 1, 0),
                     ("sv_grind_tx_fee_host", 1, 1, 93), ("sv_grind_tx_fee_host", 1, 1, 334)]
    assert sum(r[1][1]["found"] for r in reqs[0::2] if r[1][0] == "sigverifyd_fee_grind_reply") >= 1


def test_malformed_grinds_are_refused(fake):
    """a short frame, a Schnorr or unknown kind, a key of the wrong size, a weight of 2^32 or more: error 1, and the
    connection keeps serving"""
    sock, log = fake
    rng = np.random.default_rng(3)
    c = sigverifyd_daemon.connect(sock)
    frame, want = grind_req(rng, 9, 0)
    weight_at = len(frame[4:]) - 16  # weight u64, then the two u32 feerates
    bad = [short(frame), patched(frame, 10, b"\x02"), patched(frame, 10, b"\x07"), patched(frame, 11, le(64, 4)[::-1]),
           patched(frame, weight_at, (1 << 32).to_bytes(8, "big"))]
    for b in bad:
        c.sendall(b)
        got = W.read_msg(c)
        assert got[0] == "sigverifyd_error" and got[1]["code"] == 1 and got[1]["req_id"] in (9, 0), got
    roundtrip(c, [(frame, want)])
    c.close()
    assert [x[0] for x in calls(log)] == ["sv_grind_tx_fee_host"]


def test_engine_without_grind_refuses_grinds(tmp_path, bins):
    """a daemon linked against an engine without sv_grind_tx_fee_host answers a grind with error 1 and keeps serving"""
    rng = np.random.default_rng(5)
    log = tmp_path / "engine.log"
    with sigverifyd_daemon.running(tmp_path, bins["bare"], sf.env(tmp_path)) as sock:
        c = sigverifyd_daemon.connect(sock)
        frame, _ = grind_req(rng, 11, 1)
        c.sendall(frame)
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=11, code=1))
        roundtrip(c, [verify_req(rng, 12, 0, 2)])
        c.close()
    assert [x[0] for x in calls(log)] == ["sv_verify_host"]


CLIENT = r"""
import ctypes, json, sys
from tests.txsig import WallyIn as In, WallyOut as Out, WallyTx as WTx, BitcoinTx as BTx
lib = ctypes.CDLL(sys.argv[2])
vp, sz = ctypes.c_void_p, ctypes.c_size_t
lib.check_tx_sig_grind_fee.restype = ctypes.c_bool
lib.check_tx_sig_grind_fee.argtypes = [vp, vp, vp, vp, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, vp, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
sizes, keep = {}, []
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: sizes[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return ctypes.addressof(x)
H = bytes.fromhex
out = []
for c in json.load(open(sys.argv[1])):
    ins = (In * 1)()
    ins[0].txhash[:] = list(H(c["txid"])); ins[0].index = c["index"]; ins[0].sequence = c["sequence"]
    outs = (Out * 1)()
    outs[0].satoshi = c["out_amount"]; outs[0].script = buf(H(c["out_script"])) if c["out_script"] else None
    outs[0].script_len = len(H(c["out_script"]))
    w = WTx(2, c["locktime"], ctypes.addressof(ins), 1, 1, ctypes.addressof(outs), 1, 1)
    tx = BTx(ctypes.pointer(w), None, None)
    keep.extend([ins, outs, w, tx])
    sizes[ctypes.addressof(tx)] = c["amount"]
    ws = buf(H(c["wscript"]))
    sizes[ws] = len(H(c["wscript"]))
    fee, rate = ctypes.c_uint64(), ctypes.c_uint32()
    ok = lib.check_tx_sig_grind_fee(ctypes.addressof(tx), ws, buf(H(c["key"])), buf(H(c["sig"])), c["weight"], c["lo"],
                                    c["hi"], ctypes.byref(fee), ctypes.byref(rate))
    out.append([rate.value, fee.value] if ok else None)
print(json.dumps(out))
"""


def test_dropin_client_mode(tmp_path, bins):
    """check_tx_sig_grind_fee in client mode: the sighash-type gate, then one request with the fields check_tx_sig reads
    (output 0's script alone, its amount ignored); the answer is the fake's, no context is opened"""
    rng = np.random.default_rng(4)
    cases, want = [], []
    for i in range(16):
        sht = int(rng.choice([1, 0x83, 2, 3, 0x81]))
        c = dict(txid=rand(rng, 32).hex(), index=int(rng.integers(0, 9)), sequence=int(rng.integers(0, 2)),
                 locktime=int(rng.integers(0, 2**31)), out_amount=int(rng.integers(0, 2**40)),
                 out_script=rand(rng, int(rng.choice([0, 22, 34]))).hex(), amount=int(rng.integers(0, 2**40)),
                 wscript=rand(rng, int(rng.choice([1, 140]))).hex(), key=rand(rng, 64).hex(),
                 sig=(rand(rng, 64) + le(sht, 4)).hex(), weight=int(rng.choice([0, 663, 703])),
                 lo=int(rng.integers(0, 1000)), hi=int(rng.integers(0, 200000)))
        cases.append(c)
        if sht not in (1, 0x83):
            want.append(None)
            continue
        f = dict(version=2, locktime=c["locktime"], sequence=c["sequence"], sighash_type=sht, prev_txid=bytes.fromhex(c["txid"]),
                 prev_index=c["index"], input_amount=c["amount"])
        found, rate, fee = grind_answer(1, rev(bytes.fromhex(c["key"])), rev(bytes.fromhex(c["sig"])[:64]), f,
                                        bytes.fromhex(c["wscript"]), bytes.fromhex(c["out_script"]), c["weight"], c["lo"], c["hi"])
        want.append([rate, fee] if found else None)
    path = tmp_path / "grind.json"
    path.write_text(json.dumps(cases))
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CLN_SIGVERIFYD_SOCKET=sock)
        r = subprocess.run([sys.executable, "-c", CLIENT, str(path), bins["lib"]], env=env, cwd=str(tmp_path),
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
        assert json.loads(r.stdout) == want
        sent = sigverifyd_daemon.stats(sock)["requests"]
    assert sent == sum(1 for c in cases if int.from_bytes(bytes.fromhex(c["sig"])[64:], "little") in (1, 0x83))
    assert any(want) and None in want
