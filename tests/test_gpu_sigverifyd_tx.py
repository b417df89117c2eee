"""check_tx_sig through the verifier subdaemon (cln_sigverifyd): sigverifyd_tx requests of many clients coalesced into
shared launches, BOLT #3's HTLC transactions, malformed requests, many concurrent clients, and the drop-in library's
client mode for check_tx_sig and check_tx_sigs_bip143_batch, which must never open a CUDA context of its own.  Expected
answers come from the in-process engine on the same records (sv_verify_tx_host, pinned against libwally and CLN's own
check_tx_sig by tests/test_gpu_vectors.py); signatures are made with tests/ecc.py over the device's sighashes."""
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
from lightning_b200 import sigverifyd_wire as W
from tests import bolt12, txsig
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)
from tests.sigverifyd_daemon import stats as _stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SKS = [bytes([0x11 + s]) * 32 for s in range(2)]


@pytest.fixture(scope="module")
def pool(engine):
    """per signer: HTLC-shaped and multi-input / multi-output records in one blob, signed for both key kinds"""
    out = []
    for s, sk in enumerate(SKS):
        rng = np.random.default_rng(40 + s)
        a, ablob = txsig.util.make_htlc_txs(rng, 48)
        b, bblob = txsig.make_multi_txs(rng, 24)
        txs = (L.SvTx * (len(a) + len(b)))()
        for i in range(len(a)):
            txs[i] = a[i]
        for i in range(len(b)):
            t = b[i]
            for f in ("script_off", "out_script_off", "prevouts_off", "sequences_off"):
                setattr(t, f, getattr(t, f) + len(ablob))
            txs[len(a) + i] = t
        blob = ablob + bblob
        key0, sig0 = txsig.sign(engine, 0, sk, txs, blob)
        key1, sig1 = txsig.sign(engine, 1, sk, txs, blob)
        out.append(dict(txs=txs, blob=blob, keys=(key0, key1), sigs=(sig0, sig1)))
    return out


def _corrupted(rng, p, kind, k):
    """k records of the pool with corruptions: a flipped signature bit, a changed amount, SV_TX_OUTPUTS_ZERO, a sighash
    type above the low byte"""
    idx = rng.integers(0, len(p["txs"]), size=k)
    txs = txsig.subset(p["txs"], idx)
    sigs = p["sigs"][kind][idx].copy()
    for j in range(k):
        c = int(rng.integers(0, 9))
        if c == 0:
            sigs[j, int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
        elif c == 1:
            txs[j].input_amount += 1
        elif c == 2:
            txs[j].flags |= txsig.SV_TX_OUTPUTS_ZERO
        elif c == 3:
            txs[j].sighash_type |= 0x100
    return txs, sigs


def test_coalesced_tx_requests(engine, pool, daemon):
    """8 clients x 24 requests in flight: tx requests of 1..40 records under both key kinds (some asking for the
    sighashes), mixed with sigverifyd_verify and sigverifyd_bolt12 requests; every reply equals the in-process engine,
    each client's replies arrive in request order, and the requests shared launches"""
    fx = bolt12.load_fixture()
    streams = bolt12.streams(fx)
    parsed = np.nonzero(fx["status"] >= 0)[0]
    plans = []
    for ci in range(8):
        rng = np.random.default_rng(500 + ci)
        plan = []
        for j in range(24):
            rid = ci * 1000 + j
            if j % 6 == 5:  # a pre-hashed BIP-340 verify request
                items = rng.choice(parsed, size=int(rng.integers(1, 20)))
                frame = W.encode("sigverifyd_verify", req_id=rid, kind=2, n=len(items), hashes=fx["sighash"][items].tobytes(),
                                 keylen=32 * len(items), keys=fx["xonly"][items].tobytes(), sigs=fx["sig"][items].tobytes())
                plan.append((rid, frame, "sigverifyd_verify_reply", (fx["status"][items] == 1).astype(np.uint8), None))
            elif j % 6 == 2:  # a BOLT12 request
                items = np.nonzero(fx["names"] == 0)[0][rng.integers(0, 50, size=int(rng.integers(1, 10)))]
                mn, fn = bolt12.NAMES[0]
                blob = b"".join(streams[i] for i in items)
                frame = W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn,
                                 n=len(items), lens=[len(streams[i]) for i in items], bloblen=len(blob), blob=blob,
                                 xonly=fx["xonly"][items].tobytes(), sigs=fx["sig"][items].tobytes(), want_sighash=0)
                st = fx["status"][items].astype(np.int32)
                plan.append((rid, frame, "sigverifyd_bolt12_reply", np.where(st < 0, 255, st).astype(np.uint8), None))
            else:
                p = pool[int(rng.integers(0, 2))]
                kind = int(rng.integers(0, 2))
                txs, sigs = _corrupted(rng, p, kind, int(rng.integers(1, 41)))
                want = int(j % 3 == 0)
                v, sh = txsig.expected(engine, kind, p["keys"][kind], txs, p["blob"], sigs)
                frame = txsig.request(rid, kind, p["keys"][kind], txs, p["blob"], sigs, want)
                plan.append((rid, frame, "sigverifyd_tx_reply", v.copy(), sh.tobytes() if want else b""))
        plans.append(plan)
    errors = []

    def client(ci):
        try:
            c = _connect(daemon)
            for _, frame, _, _, _ in plans[ci]:
                c.sendall(frame)
            for rid, _, want_name, verdicts, sh in plans[ci]:
                name, v = W.read_msg(c)
                assert v["req_id"] == rid, ("order", rid, v["req_id"])
                assert name == want_name, (rid, name)
                got = v["status"] if name == "sigverifyd_bolt12_reply" else v["verdicts"]
                assert np.array_equal(np.frombuffer(got, np.uint8), verdicts), rid
                if sh is not None:
                    assert v["nsighash"] == (len(verdicts) if sh else 0) and v["sighashes"] == sh, rid
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not errors, errors
    tx_verdicts = np.concatenate([x[3] for p in plans for x in p if x[2] == "sigverifyd_tx_reply"])
    assert 0.3 * tx_verdicts.size < tx_verdicts.sum() < 0.95 * tx_verdicts.size  # good and bad signatures both present
    st = _stats(daemon)
    assert st["requests"] == 8 * 24, st
    assert st["launches"] < st["requests"] and st["max_coalesced"] >= 2, st


def test_bolt3_htlc_transactions(engine, daemon):
    """BOLT #3 Appendix C's five HTLC transactions verify through the daemon with both of their signatures, and do not with
    a corrupted signature; the sighashes are libwally's (recorded in the fixture)"""
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
    blob = bytes(blob)
    c = _connect(daemon)
    rid = 0
    for who in (0, 1):
        pub33 = bytes.fromhex(recs[0]["sigs"][who]["pub33"])
        assert all(bytes.fromhex(r["sigs"][who]["pub33"]) == pub33 for r in recs)  # one key per side
        sig = np.stack([np.frombuffer(bytes.fromhex(r["sigs"][who]["sig64"]), np.uint8) for r in recs])
        xy = txsig.ecc.pubkey_convert(pub33)[1]
        for kind, key in ((0, pub33), (1, xy)):
            for s in (sig, sig.copy()):
                if s is not sig:
                    s[2, 40] ^= 1
                rid += 1
                c.sendall(txsig.request(rid, kind, key, txs, blob, s, 1))
                name, v = W.read_msg(c)
                assert name == "sigverifyd_tx_reply" and v["req_id"] == rid
                assert [v["sighashes"][32 * i:32 * i + 32].hex() for i in range(len(recs))] == [r["sighash"] for r in recs]
                want = [1] * 5 if s is sig else [1, 1, 0, 1, 1]
                assert list(v["verdicts"]) == want, (who, kind)
                assert np.array_equal(txsig.expected(engine, kind, key, txs, blob, s)[0], want)
    c.close()


def test_malformed_tx_requests(pool, daemon):
    """each refusal rule gets sigverifyd_error code 1; the same connection then serves a good request"""
    p = pool[0]
    multi = [i for i in range(len(p["txs"])) if p["txs"][i].flags & txsig.SV_TX_INPUTS_SERIALIZED][:2]
    sel = [1] + multi  # an HTLC-shaped record and two multi-input / multi-output ones
    txs = txsig.subset(p["txs"], sel)
    key, sigs = p["keys"][1], p["sigs"][1][sel]
    c = _connect(daemon)

    def refused(rid, frame):
        c.sendall(frame)
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=rid, code=1)), rid

    def fields(rid, **over):
        body = W.decode(txsig.request(rid, 1, key, txs, p["blob"], sigs)[4:])[1]
        body.update(over)
        return W.encode("sigverifyd_tx", **body)

    def be32(vals):
        return b"".join(int(v).to_bytes(4, "big") for v in vals)

    n = 3
    too_many = W.encode("sigverifyd_tx", req_id=101, kind=1, keylen=64, key=key, n=(1 << 20) + 1,
                        **{f: b"\0" * 4 * ((1 << 20) + 1) for f in txsig.U32_FIELDS},
                        prev_txid=b"\0" * 32 * ((1 << 20) + 1), input_amount=b"\0" * 8 * ((1 << 20) + 1),
                        output_amount=b"\0" * 8 * ((1 << 20) + 1),
                        **{f: b"\0" * 4 * ((1 << 20) + 1) for f in ("script_len", "outputs_len", "prevouts_len",
                                                                     "sequences_len")},
                        bloblen=0, blob=b"", sigs=b"\0" * 64 * ((1 << 20) + 1), want_sighash=0)
    refused(101, too_many)
    refused(102, fields(102, kind=2, keylen=32, key=key[:32]))  # a BIP-340 kind
    refused(103, fields(103, kind=0))  # a 64-byte key for the 33-byte kind
    refused(104, fields(104, keylen=33, key=key[:33]))  # a 33-byte key for the 64-byte kind
    body = W.decode(txsig.request(0, 1, key, txs, p["blob"], sigs)[4:])[1]
    sl = [int.from_bytes(body["script_len"][4 * i:4 * i + 4], "big") for i in range(n)]
    refused(105, fields(105, script_len=be32([sl[0] + 1] + sl[1:])))  # spans longer than the blob
    refused(106, fields(106, script_len=be32([sl[0] - 1] + sl[1:])))  # and shorter
    flags = [int.from_bytes(body["flags"][4 * i:4 * i + 4], "big") for i in range(n)]
    refused(107, fields(107, flags=be32([flags[0] | 8] + flags[1:])))  # an unknown flag bit
    refused(108, fields(108, flags=be32([flags[0] | 0x80000000] + flags[1:])))
    # outpoints or sequences on a record without SV_TX_INPUTS_SERIALIZED: 36 / 4 bytes moved over from the script span
    ol = [int.from_bytes(body["prevouts_len"][4 * i:4 * i + 4], "big") for i in range(n)]
    ql = [int.from_bytes(body["sequences_len"][4 * i:4 * i + 4], "big") for i in range(n)]
    assert flags[0] == 0 and sl[0] > 40
    refused(109, fields(109, script_len=be32([sl[0] - 36] + sl[1:]), prevouts_len=be32([36] + ol[1:])))
    refused(110, fields(110, script_len=be32([sl[0] - 4] + sl[1:]), sequences_len=be32([4] + ql[1:])))
    cut = txsig.request(111, 1, key, txs, p["blob"], sigs)[4:-1]  # one byte short of its fields: does not parse
    refused(111, len(cut).to_bytes(4, "big") + cut)
    c.sendall(txsig.request(9, 1, key, txs, p["blob"], sigs, 1))
    name, v = W.read_msg(c)
    assert name == "sigverifyd_tx_reply" and v["req_id"] == 9 and list(v["verdicts"]) == [1, 1, 1] and v["nsighash"] == 3
    c.close()


def test_many_clients(pool, daemon):
    """200 concurrent connections (more than a fixed table of 64 would hold), one request each: all are answered"""
    p = pool[1]
    conns = [_connect(daemon) for _ in range(200)]
    try:
        for i, c in enumerate(conns):
            k = i % len(p["txs"])
            c.sendall(txsig.request(i, i % 2, p["keys"][i % 2], txsig.subset(p["txs"], [k]), p["blob"], p["sigs"][i % 2][[k]]))
        for i, c in enumerate(conns):
            name, v = W.read_msg(c)
            assert name == "sigverifyd_tx_reply" and v["req_id"] == i and list(v["verdicts"]) == [1], i
    finally:
        for c in conns:
            c.close()
    assert _stats(daemon)["requests"] == 200


# the drop-in library driven through its C ABI with stand-alone wally_tx structs (cln_dropin.h); prints its answers and
# the number of requests it expects to have sent.  Run once with a GPU and no daemon (in-process) and once in client mode.
CLIENT = r"""
import ctypes, json, sys
import numpy as np
from lightning_b200 import engine
from tests.txsig import WallyIn as In, WallyOut as Out, WallyTx as WTx, BitcoinTx as BTx
lib = ctypes.CDLL(engine.LIB_PATH)
vp, sz = ctypes.c_void_p, ctypes.c_size_t
lib.check_tx_sig.restype = ctypes.c_bool
lib.check_tx_sig.argtypes = [vp, sz, vp, vp, vp, vp]
lib.check_tx_sigs_bip143_batch.argtypes = [vp, vp, sz, vp, vp, sz, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
sizes, amounts, keep = {}, {}, []
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: amounts[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return x
def bsig(sig64, sht):  # struct bitcoin_signature: r and s as little-endian limbs, then the sighash type
    return buf(sig64[31::-1] + sig64[:31:-1] + int(sht).to_bytes(4, "little"))
sc = json.load(open(sys.argv[1]))
xy = bytes.fromhex(sc["xy"])
pub = buf(xy[31::-1] + xy[:31:-1])
out = {"single": [], "batch": [], "sent": 0}
for c in sc["single"]:
    ins = (In * len(c["ins"]))()
    for k, (txid, idx, seq) in enumerate(c["ins"]):
        ins[k].txhash[:] = list(bytes.fromhex(txid)); ins[k].index = idx; ins[k].sequence = seq
    outs = (Out * len(c["outs"]))()
    for k, (sat, script) in enumerate(c["outs"]):
        s = bytes.fromhex(script)
        outs[k].satoshi = sat; outs[k].script = ctypes.addressof(buf(s)) if s else None; outs[k].script_len = len(s)
    w = WTx(c["version"], c["locktime"], ctypes.addressof(ins), len(c["ins"]), len(c["ins"]), ctypes.addressof(outs),
            len(c["outs"]), len(c["outs"]))
    tx = BTx(ctypes.pointer(w), None, None)
    keep += [ins, outs, w, tx]
    amounts[ctypes.addressof(tx)] = c["amount"]
    script = buf(bytes.fromhex(c["script"]))
    sizes[ctypes.addressof(script)] = len(bytes.fromhex(c["script"]))
    args = (None, ctypes.addressof(script)) if c["witness"] else (ctypes.addressof(script), None)
    got = lib.check_tx_sig(ctypes.addressof(tx), c["input"], args[0], args[1], ctypes.addressof(pub),
                           ctypes.addressof(bsig(bytes.fromhex(c["sig"]), c["sighash_type"])))
    out["single"].append(bool(got))
    out["sent"] += c["sighash_type"] == 1 or (c["witness"] and c["sighash_type"] == 0x83)
txs = np.fromfile(sc["txs"], np.uint8)
blob = open(sc["blob"], "rb").read()
sigs = bytes.fromhex(sc["sigs"])
for n in sc["batches"]:
    rec = n * sc["rec_size"]
    stx = b"".join(bsig(sigs[64 * (i % sc["nsig"]):64 * (i % sc["nsig"]) + 64], sc["types"][i % sc["nsig"]]) for i in range(n))
    ok = (ctypes.c_bool * n)()
    lib.check_tx_sigs_bip143_batch(txs[:rec].ctypes.data, ctypes.addressof(buf(blob)), len(blob), ctypes.addressof(pub),
                                   ctypes.addressof(buf(stx)), n, ok)
    out["batch"].append([bool(x) for x in ok])
    out["sent"] += (n + 65535) // 65536
print(json.dumps(out))
"""


def _scenario(engine, tmp_path):
    """check_tx_sig calls on transactions of 1-3 inputs and 1-6 outputs (every sighash type, witness and redeem script
    argument, signatures over the device's sighash, some corrupted) and check_tx_sigs_bip143_batch calls on HTLC records,
    one of them over 65,536 records (two requests)"""
    rng = np.random.default_rng(77)
    sk = SKS[0]
    pub33, xy = txsig.ecc.pubkey_create(sk)
    single = []
    for it in range(60):
        nin, nout = int(rng.integers(1, 4)), int(rng.integers(1, 7))
        ins = [(bytes(rng.integers(0, 256, size=32, dtype=np.uint8)).hex(), int(rng.integers(0, 5)), int(rng.integers(0, 2**32)))
               for _ in range(nin)]
        outs = [(int(rng.integers(0, 2**40)), bytes(rng.integers(0, 256, size=int(rng.choice([0, 22, 34, 300])), dtype=np.uint8)).hex())
                for _ in range(nout)]
        inp = int(rng.integers(0, nin))
        script = bytes(rng.integers(0, 256, size=int(rng.choice([1, 71, 142, 253, 700])), dtype=np.uint8))
        sht = int(rng.choice([1, 1, 1, 0x83, 0x83, 2, 3, 0x81]))
        c = dict(version=2, locktime=int(rng.integers(0, 2**31)), ins=ins, outs=outs, input=inp, script=script.hex(),
                 witness=bool(rng.random() < 0.85), sighash_type=sht, amount=int(rng.integers(0, 2**45)))
        # the record check_tx_sig builds (cln_dropin.c), for the device's sighash to sign
        t = (L.SvTx * 1)()
        r = t[0]
        r.version, r.locktime, r.sequence, r.sighash_type = 2, c["locktime"], ins[inp][2], sht
        r.prev_txid[:] = list(bytes.fromhex(ins[inp][0]))
        r.prev_index, r.input_amount = ins[inp][1], c["amount"]
        ser = [sat.to_bytes(8, "little") + bytes([len(bytes.fromhex(s))]) + bytes.fromhex(s) if len(bytes.fromhex(s)) < 0xfd
               else sat.to_bytes(8, "little") + b"\xfd" + len(bytes.fromhex(s)).to_bytes(2, "little") + bytes.fromhex(s)
               for sat, s in outs]
        if sht & 0x1f == 3:
            o = ser[inp] if inp < nout else b""
            r.flags = txsig.SV_TX_OUTPUTS_SERIALIZED if inp < nout else txsig.SV_TX_OUTPUTS_ZERO
        else:
            o = b"".join(ser)
            r.flags = txsig.SV_TX_OUTPUTS_SERIALIZED
        pv = b"".join(bytes.fromhex(x) + i.to_bytes(4, "little") for x, i, _ in ins) if nin > 1 else b""
        sq = b"".join(s.to_bytes(4, "little") for _, _, s in ins) if nin > 1 else b""
        if nin > 1:
            r.flags |= txsig.SV_TX_INPUTS_SERIALIZED
        blob = script + o + pv + sq
        r.script_len, r.out_script_off, r.out_script_len = len(script), len(script), len(o)
        r.prevouts_off, r.prevouts_len = len(script) + len(o), len(pv)
        r.sequences_off, r.sequences_len = len(script) + len(o) + len(pv), len(sq)
        _, sig = txsig.sign(engine, 1, sk, t, blob)
        sig = sig[0]
        if it % 4 == 1:
            sig[int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
        elif it % 4 == 2:
            c["amount"] += 1  # signed for another amount
        c["sig"] = bytes(sig).hex()
        single.append(c)
    txs, blob = txsig.util.make_htlc_txs(rng, 64)
    _, sigs = txsig.sign(engine, 1, sk, txs, blob)
    sigs[5::7, 33] ^= 2
    big = 65536 + 300
    recs = (L.SvTx * big)()
    for i in range(big):
        recs[i] = txs[i % 64]
    path_txs, path_blob = tmp_path / "txs.bin", tmp_path / "blob.bin"
    open(path_txs, "wb").write(bytes(recs))
    open(path_blob, "wb").write(blob)
    sc = dict(xy=xy.hex(), single=single, txs=str(path_txs), blob=str(path_blob), sigs=sigs.tobytes().hex(), nsig=64,
              types=[t.sighash_type for t in txs], rec_size=ctypes.sizeof(L.SvTx), batches=[64, 7, big])
    path = tmp_path / "scenario.json"
    json.dump(sc, open(path, "w"))
    return str(path)


def _no_core():
    resource.setrlimit(resource.RLIMIT_CORE, (0, 0))


def _run_client(path, tmp_path, env):
    r = subprocess.run([sys.executable, "-c", CLIENT, path], env=env, cwd=str(tmp_path), capture_output=True, text=True,
                       timeout=900, preexec_fn=_no_core)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def test_dropin_client_mode_tx(engine, daemon, tmp_path):
    """check_tx_sig and check_tx_sigs_bip143_batch in client mode (no visible GPU: creating a context would abort) give
    exactly the in-process answers, and every call that passed the sighash-type gate went through the daemon"""
    path = _scenario(engine, tmp_path)
    base = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base.pop("CLN_SIGVERIFYD_SOCKET", None)
    local = _run_client(path, tmp_path, base)
    remote = _run_client(path, tmp_path, dict(base, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES=""))
    assert remote["single"] == local["single"] and remote["batch"] == local["batch"]
    assert 10 < sum(local["single"]) < 50
    types = [t in (1, 0x83) for t in json.load(open(path))["types"]]
    assert 20 < sum(local["batch"][0]) < 64 and local["batch"][0] == [ok and ty for ok, ty in zip(local["batch"][0], types)]
    assert local["batch"][2] == [local["batch"][0][i % 64] for i in range(len(local["batch"][2]))]
    assert _stats(daemon)["requests"] == remote["sent"]
