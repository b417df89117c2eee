"""onchaind's HTLC fee grind on the device (sv_grind_tx_fee_host, SigVerifier.grind_tx_fee, the drop-in's
check_tx_sig_grind_fee in process and through cln_sigverifyd).  Transactions of the BOLT #3 HTLC shape
(tests/golden/bolt3_htlc_txs.json) are signed with tests/ecc.py at known feerates over the device's sighash.  Every answer
is checked against the model of the reference loop (tests/feegrind.py), whose per-candidate predicate is the verdict
sv_verify_tx_host gives for that transaction (itself checked against Core Lightning's check_tx_sig by
tests/test_gpu_vectors.py); tests/test_fee_grind_host.py checks the candidate check against Core Lightning directly."""
import ctypes
import json
import os
import resource
import subprocess
import sys
import threading

import numpy as np
import pytest

import lightning_b200 as L
from lightning_b200 import SvTx
from lightning_b200 import sigverifyd_wire as W
from tests import ecc, feegrind, sigverifyd_daemon, txsig, util
from tests.sigverifyd_daemon import daemon  # noqa: F401

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VECTORS = json.load(open(os.path.join(ROOT, "tests", "golden", "bolt3_htlc_txs.json")))
CHUNK = 1 << 20
INPUT = 5_000_000


def _sk(i):
    return (0x1234567 + 7919 * i).to_bytes(32, "big")


def signed(engine, kind, vec, sht, weight, feerate, sk, input_amount=INPUT):
    """(tx, blob, key, sig): vector `vec` as an HTLC transaction spending input_amount, signed by sk at feerate's fee"""
    t, blob = feegrind.htlc_tx(VECTORS[vec], sht, input_amount)
    t.output_amount = input_amount - feegrind.fee(feerate, weight)
    txs = (SvTx * 1)(t)
    key, sigs = txsig.sign(engine, kind, sk, txs, blob)
    return t, blob, key, bytes(sigs[0])


def tx_verdicts(engine, kind, t, blob, key, sig, amounts):
    """sv_verify_tx_host's verdict for t with each output amount"""
    n = len(amounts)
    txs = (SvTx * n)()
    for i, a in enumerate(amounts):
        txs[i] = t
        txs[i].output_amount = a
    keys = np.frombuffer(bytes(key) * n, np.uint8).reshape(n, len(key))
    sigs = np.frombuffer(bytes(sig) * n, np.uint8).reshape(n, 64)
    return engine.check_tx_sigs(kind, txs, blob, keys, sigs)


@pytest.mark.parametrize("kind", [0, 1])
def test_signed_feerates_found_from_253(engine, kind):
    """signed at each feerate, ground from 253: the answer is the first feerate with the signed fee; the transaction
    verifies at that fee and not at the previous distinct fee"""
    for i, fs in enumerate((253, 648, 2070, 2195, 3703, 4915, 9651, 15000, 100000)):
        vec = i % len(VECTORS)
        weight = feegrind.HTLC_SUCCESS_WEIGHT if "success" in VECTORS[vec]["name"] else feegrind.HTLC_TIMEOUT_WEIGHT
        t, blob, key, sig = signed(engine, kind, vec, (1, 0x83)[i % 2], weight, fs, _sk(i))
        want_fee = feegrind.fee(fs, weight)
        want = feegrind.grind(253, 125000, weight, INPUT, lambda f, x: x == want_fee)
        assert want[0] <= fs and engine.grind_tx_fee(kind, t, blob, key, sig, weight, 253, 125000) == want, fs
        prev = [x for _, x in feegrind.walk(253, want[0], weight, INPUT)]
        amounts = [INPUT - want_fee] + ([INPUT - prev[-2]] if len(prev) > 1 else [])
        assert list(tx_verdicts(engine, kind, t, blob, key, sig, amounts)) == [1] + [0] * (len(amounts) - 1)


def test_ranges_against_every_candidate(engine):
    """ranges of up to 2,000 candidates: the grind equals the reference loop run over sv_verify_tx_host's verdict for every
    candidate transaction (signed fee inside, at the edges of and outside the range)"""
    rng = np.random.default_rng(5)
    for it in range(12):
        kind, vec, sht = it % 2, it % len(VECTORS), (1, 0x83)[(it // 2) % 2]
        weight = int(rng.choice([663, 703, 666, 706, 1000, 1, 2500]))
        lo = int(rng.integers(0, 30000))
        hi = lo + int(rng.integers(0, 2000 * 1000 // max(weight, 1) + 1))
        fs = [lo, hi, (lo + hi) // 2, hi + 50][it % 4]
        input_amount = int(rng.choice([INPUT, feegrind.fee(hi, weight) + int(rng.integers(0, 3)), 10**9]))
        if feegrind.fee(fs, weight) > input_amount:
            input_amount = feegrind.fee(fs, weight)
        t, blob, key, sig = signed(engine, kind, vec, sht, weight, fs, _sk(100 + it), input_amount)
        cands = list(feegrind.walk(lo, hi, weight, input_amount))
        assert len(cands) <= 2001
        v = tx_verdicts(engine, kind, t, blob, key, sig, [input_amount - x for _, x in cands]) if cands else []
        ok = {f: int(x) for (f, _), x in zip(cands, v)}
        want = feegrind.grind(lo, hi, weight, input_amount, lambda f, x: ok[f] == 1)
        assert engine.grind_tx_fee(kind, t, blob, key, sig, weight, lo, hi) == want, (it, lo, hi, fs, weight)


def test_not_found(engine):
    """wrong key, high S, r or s >= n, a flipped bit, a sighash type sv_verify_tx_host refuses, an input too small for
    the signed fee: none found"""
    w, fs = 663, 4915
    t, blob, key, sig = signed(engine, 0, 1, 1, w, fs, _sk(7))
    assert engine.grind_tx_fee(0, t, blob, key, sig, w, 253, 20000) == (feegrind.grind(
        253, 20000, w, INPUT, lambda f, x: x == feegrind.fee(fs, w)))
    r, s = int.from_bytes(sig[:32], "big"), int.from_bytes(sig[32:], "big")
    bad = {"high_s": sig[:32] + (util.N_ORDER - s).to_bytes(32, "big"),
           "s_ge_n": sig[:32] + (s + util.N_ORDER).to_bytes(32, "big") if s + util.N_ORDER < 2**256 else sig[:32] + bytes([255]) * 32,
           "r_ge_n": (r + util.N_ORDER).to_bytes(32, "big") + sig[32:] if r + util.N_ORDER < 2**256 else bytes([255]) * 32 + sig[32:],
           "flip": sig[:40] + bytes([sig[40] ^ 1]) + sig[41:]}
    for name, b in bad.items():
        assert engine.grind_tx_fee(0, t, blob, key, b, w, 253, 20000) == (None, 0), name
    assert engine.grind_tx_fee(0, t, blob, ecc.pubkey_create(_sk(8))[0], sig, w, 253, 20000) == (None, 0)
    t2 = SvTx.from_buffer_copy(t)
    t2.sighash_type = 0x101
    assert engine.grind_tx_fee(0, t2, blob, key, sig, w, 253, 20000) == (None, 0)
    t3 = SvTx.from_buffer_copy(t)
    t3.input_amount = feegrind.fee(fs, w) - 1
    assert engine.grind_tx_fee(0, t3, blob, key, sig, w, 253, 20000) == (None, 0)


@pytest.mark.parametrize("offset", [CHUNK - 1, CHUNK, 3 * CHUNK + 17, 20_000_005])
def test_chunks_and_early_stop(engine, offset):
    """matches on both sides of a chunk boundary and past 2*10^7 candidates: found exactly, with one launch per chunk up
    to the matching one (the walk stops there)"""
    lo, w = 253, 1000
    fs = lo + offset
    t, blob, key, sig = signed(engine, 1, 2, 1, w, fs, _sk(9), 10**9)
    before = engine.info()["launches"]
    assert engine.grind_tx_fee(1, t, blob, key, sig, w, lo, 0xFFFFFFFF) == (fs, fs)
    assert engine.info()["launches"] - before == 1 + offset // CHUNK + 1


def test_no_match_walks_to_the_input_and_edges(engine):
    """no match: the walk stops where the fee passes the input (no launch past it); min > max and a fee above the input
    at min_feerate launch nothing; weight 0 is one candidate, fee 0; bad arguments are SV_ERR_ARG"""
    t, blob, key, sig = signed(engine, 0, 3, 1, 1000, 77, _sk(10), 3 * CHUNK)
    before = engine.info()["launches"]
    assert engine.grind_tx_fee(0, t, blob, key, sig, 1000, 100, 0xFFFFFFFF) == (None, 0)
    assert engine.info()["launches"] - before == 1 + (3 * CHUNK - 100) // CHUNK + 1
    before = engine.info()["launches"]
    assert engine.grind_tx_fee(0, t, blob, key, sig, 1000, 5, 4) == (None, 0)
    assert engine.grind_tx_fee(0, t, blob, key, sig, 1000, 3 * CHUNK + 1, 0xFFFFFFFF) == (None, 0)
    assert engine.info()["launches"] == before
    t0, blob0, key0, sig0 = signed(engine, 0, 3, 1, 0, 0, _sk(11))
    assert engine.grind_tx_fee(0, t0, blob0, key0, sig0, 0, 1000, 0xFFFFFFFF) == (1000, 0)
    tf = SvTx.from_buffer_copy(t)
    tf.flags = 1
    for args in ((tf, blob, key, sig, 1000), (t, blob, key, sig, 1 << 32), (t, blob[:-1], key, sig, 1000)):
        with pytest.raises(L.EngineError):
            engine.grind_tx_fee(0, *args[:4], args[4], 253, 300)


# ---- the drop-in: in process, and in client mode through a daemon with no GPU visible to the client -----------------
CLIENT = r"""
import ctypes, json, sys
from lightning_b200 import engine
from tests.txsig import WallyIn as In, WallyOut as Out, WallyTx as WTx, BitcoinTx as BTx
lib = ctypes.CDLL(engine.LIB_PATH)
vp, sz = ctypes.c_void_p, ctypes.c_size_t
lib.check_tx_sig_grind_fee.restype = ctypes.c_bool
lib.check_tx_sig_grind_fee.argtypes = [vp, vp, vp, vp, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, vp, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
sizes, amounts, keep = {}, {}, []
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: amounts[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return x
out = []
for c in json.load(open(sys.argv[1])):
    H = bytes.fromhex
    ins = (In * 1)()
    ins[0].txhash[:] = list(H(c["txid"])); ins[0].index = c["index"]; ins[0].sequence = c["sequence"]
    outs = (Out * 1)()
    os_ = buf(H(c["out_script"]))
    outs[0].satoshi = 12345; outs[0].script = ctypes.addressof(os_); outs[0].script_len = len(H(c["out_script"]))
    w = WTx(c["version"], c["locktime"], ctypes.addressof(ins), 1, 1, ctypes.addressof(outs), 1, 1)
    tx = BTx(ctypes.pointer(w), None, None)
    keep += [ins, outs, w, tx]
    amounts[ctypes.addressof(tx)] = c["amount"]
    ws = buf(H(c["wscript"]))
    sizes[ctypes.addressof(ws)] = len(H(c["wscript"]))
    xy, sig = H(c["xy"]), H(c["sig"])
    pub = buf(xy[31::-1] + xy[:31:-1])
    bsig = buf(sig[31::-1] + sig[:31:-1] + int(c["sht"]).to_bytes(4, "little"))
    fee, rate = ctypes.c_uint64(), ctypes.c_uint32()
    ok = lib.check_tx_sig_grind_fee(ctypes.addressof(tx), ctypes.addressof(ws), ctypes.addressof(pub), ctypes.addressof(bsig),
                                    c["weight"], c["lo"], c["hi"], ctypes.byref(fee), ctypes.byref(rate))
    out.append([rate.value, fee.value] if ok else None)
print(json.dumps(out))
"""


def _no_core():
    resource.setrlimit(resource.RLIMIT_CORE, (0, 0))


def _scenario(engine, tmp_path):
    """grinds through the drop-in and the answers SigVerifier.grind_tx_fee gives (None where the sighash-type gate
    refuses before anything is sent)"""
    cases, want = [], []
    for i, (sht, fs) in enumerate([(1, 2070), (0x83, 15000), (1, 9651), (2, 3703), (0x83, 648), (1, 100000)]):
        vec = i % len(VECTORS)
        w = feegrind.HTLC_SUCCESS_WEIGHT if "success" in VECTORS[vec]["name"] else feegrind.HTLC_TIMEOUT_WEIGHT
        t, blob, xy, sig = signed(engine, 1, vec, sht, w, fs, _sk(200 + i))
        lo, hi = 253, (125000 if i != 5 else 50000)  # the last one's feerate lies outside the range
        v = VECTORS[vec]
        cases.append(dict(txid=v["prev_txid"], index=v["prev_index"], sequence=v["sequence"], version=v["version"],
                          locktime=v["locktime"], out_script=v["out_script"], wscript=v["wscript"], amount=INPUT,
                          xy=xy.hex(), sig=sig.hex(), sht=sht, weight=w, lo=lo, hi=hi))
        got = engine.grind_tx_fee(1, t, blob, xy, sig, w, lo, hi)
        want.append(list(got) if got[0] is not None and sht in (1, 0x83) else None)
    path = tmp_path / "grind.json"
    path.write_text(json.dumps(cases))
    return str(path), want


def _run_client(path, tmp_path, env):
    r = subprocess.run([sys.executable, "-c", CLIENT, path], env=env, cwd=str(tmp_path), capture_output=True, text=True,
                       timeout=900, preexec_fn=_no_core)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def test_dropin_in_process_and_client_mode(engine, daemon, tmp_path):  # noqa: F811
    path, want = _scenario(engine, tmp_path)
    assert sum(x is not None for x in want) == 4
    base = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base.pop("CLN_SIGVERIFYD_SOCKET", None)
    assert _run_client(path, tmp_path, base) == want
    assert _run_client(path, tmp_path, dict(base, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES="")) == want
    assert sigverifyd_daemon.stats(daemon)["requests"] == 5  # the SIGHASH_NONE one is refused before it is sent


def grind_frame(rid, kind, t, blob, key, sig, weight, lo, hi):
    return W.encode("sigverifyd_fee_grind", req_id=rid, kind=kind, keylen=len(key), key=bytes(key), version=t.version,
                    locktime=t.locktime, sequence=t.sequence, sighash_type=t.sighash_type, prev_index=t.prev_index,
                    prev_txid=bytes(t.prev_txid), input_amount=t.input_amount, script_len=t.script_len,
                    script=blob[t.script_off:t.script_off + t.script_len], out_script_len=t.out_script_len,
                    out_script=blob[t.out_script_off:t.out_script_off + t.out_script_len], sig=bytes(sig), weight=weight,
                    min_feerate=lo, max_feerate=hi)


def test_daemon_interleaves_grinds_with_other_traffic(engine, daemon):  # noqa: F811
    """four clients each write grind, sigverifyd_tx and sigverifyd_verify requests at once: every reply is the in-process
    answer, in request order"""
    rng = np.random.default_rng(17)
    plans = []
    for ci in range(4):
        reqs = []
        for j in range(3):
            kind, vec, fs = (ci + j) % 2, (ci + j) % len(VECTORS), int(rng.integers(253, 30000))
            w = 663 if j % 2 else 703
            t, blob, key, sig = signed(engine, kind, vec, 1, w, fs, _sk(300 + 10 * ci + j))
            lo = 253 if j != 2 else fs + 5
            f, fee = engine.grind_tx_fee(kind, t, blob, key, sig, w, lo, 125000)
            rid = 1000 * ci + 10 * j
            reqs.append((grind_frame(rid, kind, t, blob, key, sig, w, lo, 125000),
                         ("sigverifyd_fee_grind_reply", dict(req_id=rid, found=int(f is not None), feerate=f or 0, fee=fee))))
            txs, tblob = txsig.make_multi_txs(rng, 3)
            tkey, tsigs = txsig.sign(engine, 1, _sk(400 + ci), txs, tblob)
            v, sh = txsig.expected(engine, 1, tkey, txs, tblob, tsigs)
            reqs.append((txsig.request(rid + 1, 1, tkey, txs, tblob, tsigs, 1),
                         ("sigverifyd_tx_reply", dict(req_id=rid + 1, n=3, verdicts=bytes(v), nsighash=3, sighashes=sh.tobytes()))))
            m = rng.integers(0, 256, size=(2, 32), dtype=np.uint8)
            pk, _ = ecc.pubkey_create(_sk(500 + ci))
            sg = np.frombuffer(ecc.ecdsa_sign(_sk(500 + ci), bytes(m[0])) * 2, np.uint8).reshape(2, 64)
            vv = engine.verify(0, m, np.frombuffer(pk * 2, np.uint8).reshape(2, 33), sg)
            reqs.append((W.encode("sigverifyd_verify", req_id=rid + 2, kind=0, n=2, hashes=m.tobytes(), keylen=66, keys=pk * 2,
                                  sigs=sg.tobytes()),
                         ("sigverifyd_verify_reply", dict(req_id=rid + 2, n=2, verdicts=bytes(vv)))))
        plans.append(reqs)
    errors = []

    def client(reqs):
        try:
            c = sigverifyd_daemon.connect(daemon)
            c.sendall(b"".join(f for f, _ in reqs))
            for _, want in reqs:
                got = W.read_msg(c)
                assert got == want, (got, want)
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append(repr(ex))

    th = [threading.Thread(target=client, args=(p,)) for p in plans]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=600)
    assert not errors, errors
    assert any(r[1][1]["found"] for p in plans for r in p[0::3]) and not all(r[1][1]["found"] for p in plans for r in p[0::3])
