"""GPU: the verifier subdaemon's two engine workers under a gossip burst.  One client sends the committed gossip subset
tiled 53 times as one sigverifyd_gossip_burst; right after, 8 channeld-like clients send sigverifyd_tx requests (BOLT #3
Appendix C's HTLC transactions under SIGHASH_ALL, and anchor-style HTLC transactions under
SIGHASH_SINGLE|SIGHASH_ANYONECANPAY, part of them corrupted) and BOLT12 requests.  Every answer must equal the
in-process engine's and the recorded answers (BOLT #3's libwally sighashes, the BOLT12 fixture's statuses), the channel
checks must not wait for the burst, and the stats must count every request."""
import json
import os
import threading
import time

import numpy as np
import pytest

import lightning_b200 as L
from lightning_b200 import sigverifyd_wire as W
from tests import bolt12, gossip, txsig
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)
from tests.sigverifyd_daemon import stats as _stats
from tests.test_gpu_gossip_burst import TESTNET, _burst_frame, _wire_status

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SK = bytes([0x42]) * 32


def _bolt3():
    """BOLT #3 Appendix C's HTLC transactions as records, and per side its key and signatures (SIGHASH_ALL)"""
    recs = json.load(open(os.path.join(GOLD, "bolt3_htlc_txs.json")))
    txs = (L.SvTx * len(recs))()
    blob = bytearray()
    for t, r in zip(txs, recs):
        t.version, t.locktime, t.sequence, t.sighash_type = r["version"], r["locktime"], r["sequence"], 1
        t.prev_txid[:] = list(bytes.fromhex(r["prev_txid"]))
        t.prev_index = r["prev_index"]
        ws, os_ = bytes.fromhex(r["wscript"]), bytes.fromhex(r["out_script"])
        t.script_off, t.script_len = len(blob), len(ws)
        blob += ws
        t.out_script_off, t.out_script_len = len(blob), len(os_)
        blob += os_
        t.input_amount, t.output_amount = r["input_amount"], r["output_amount"]
    sides = []
    for who in (0, 1):
        assert all(r["sigs"][who]["sighash_type"] == 1 and r["sigs"][who]["expected"] == 1 for r in recs)
        pub33 = bytes.fromhex(recs[0]["sigs"][who]["pub33"])
        sig = np.stack([np.frombuffer(bytes.fromhex(r["sigs"][who]["sig64"]), np.uint8) for r in recs])
        sides.append((pub33, sig))
    return txs, bytes(blob), sides, [bytes.fromhex(r["sighash"]) for r in recs]


def _plans(engine):
    """per client, its requests: (req_id, frame, reply name, want fields)"""
    txs, blob, sides, sighashes = _bolt3()
    (_, _), (htlc, hblob) = txsig.commitment_signed(np.random.default_rng(9), 24)  # anchors: 0x83 on every record
    assert all(t.sighash_type == 0x83 for t in htlc)
    hkey, hsig = txsig.sign(engine, 0, SK, htlc, hblob)
    fx = bolt12.load_fixture()
    streams = bolt12.streams(fx)
    plans = []
    for ci in range(8):
        rng = np.random.default_rng(900 + ci)
        plan = []
        for j in range(6):
            rid = 1000 * (ci + 1) + j
            if j == 0:  # BOLT #3: one side's signatures, one corrupted on odd clients
                key, sig = sides[ci % 2]
                sig = sig.copy()
                want = [1] * len(txs)
                if ci % 2:
                    sig[2, 40] ^= 1
                    want[2] = 0
                v, sh = txsig.expected(engine, 0, key, txs, blob, sig)
                assert v.tolist() == want and [bytes(h) for h in sh] == sighashes
                plan.append((rid, txsig.request(rid, 0, key, txs, blob, sig, 1), "sigverifyd_tx_reply",
                             dict(verdicts=bytes(want), sighashes=b"".join(sighashes))))
            elif j % 2 == 1:  # anchor HTLC transactions under SIGHASH_SINGLE|ANYONECANPAY, some signatures corrupted
                idx = rng.choice(len(htlc), size=int(rng.integers(1, 12)), replace=False)
                sub, sig = txsig.subset(htlc, idx), hsig[idx].copy()
                bad = rng.random(len(idx)) < 0.3
                sig[bad, 7] ^= 0x10
                v, sh = txsig.expected(engine, 0, hkey, sub, hblob, sig)
                assert v.tolist() == [int(not b) for b in bad]
                plan.append((rid, txsig.request(rid, 0, hkey, sub, hblob, sig, 1), "sigverifyd_tx_reply",
                             dict(verdicts=v.tobytes(), sighashes=sh.tobytes())))
            else:  # BOLT12: the fixture's invoices, with its recorded statuses
                items = np.nonzero(fx["names"] == 0)[0][rng.integers(0, 50, size=int(rng.integers(1, 10)))]
                mn, fn = bolt12.NAMES[0]
                b = b"".join(streams[i] for i in items)
                frame = W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn,
                                 n=len(items), lens=[len(streams[i]) for i in items], bloblen=len(b), blob=b,
                                 xonly=fx["xonly"][items].tobytes(), sigs=fx["sig"][items].tobytes(), want_sighash=0)
                st = fx["status"][items].astype(np.int32)
                plan.append((rid, frame, "sigverifyd_bolt12_reply", dict(status=bytes(_wire_status(st.tolist())))))
        plans.append(plan)
    return plans


def test_channel_checks_beside_a_burst(engine, daemon):
    msgs = gossip.load_subset() * 53
    burst_want = engine.verify_gossip_burst(msgs, TESTNET)
    assert not burst_want.any()  # test_gpu_gossip_burst.py pins the fixture's statuses
    burst_frame = _burst_frame(1, msgs)
    plans = _plans(engine)
    arrived, errors = {}, []
    g = _connect(daemon)
    conns = [_connect(daemon) for _ in plans]

    def channeld(ci):
        try:
            c = conns[ci]
            c.sendall(b"".join(f for _, f, _, _ in plans[ci]))
            for rid, _, name, want in plans[ci]:
                got = W.read_msg(c)
                arrived[rid] = time.monotonic()
                assert got[0] == name and got[1]["req_id"] == rid, (got[0], got[1].get("req_id"), rid)
                for k, v in want.items():
                    assert got[1][k] == v, (rid, k)
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    g.sendall(burst_frame)
    th = [threading.Thread(target=channeld, args=(ci,)) for ci in range(len(plans))]
    for t in th:
        t.start()
    name, rep = W.read_msg(g)
    burst_at = time.monotonic()
    for t in th:
        t.join(timeout=300)
    assert not errors, errors
    assert name == "sigverifyd_gossip_burst_reply" and rep["req_id"] == 1 and rep["n"] == len(msgs)
    assert np.array_equal(np.frombuffer(rep["status"], np.uint8), np.array(_wire_status(burst_want.tolist()), np.uint8))
    assert len(arrived) == sum(len(p) for p in plans)
    assert min(arrived.values()) < burst_at, "every channel check waited for the burst"
    st = _stats(daemon)
    assert st["requests"] == 1 + len(arrived), st
    g.close()
    for c in conns:
        c.close()
