"""GPU: gossip bursts (sv_verify_gossip_burst_host), where a channel_update's signer is found among the batch's own
channel_announcements on the device.  The committed fixture as one burst, the fixture bit-flipped against CLN's own
gossipd/sigcheck.c with gossipd's gates and pending-map rule applied in Python, crafted messages for every resolution
rule (the repair round included), and the verifier subdaemon's sigverifyd_gossip_burst message and the drop-in
sigcheck_gossip_batch in client mode."""
import ctypes
import hashlib
import json
import os
import struct
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import ecc, gossip
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))  # noqa: E731
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")  # every fixture message's chain
OTHER = bytes(31) + b"\x01"


def _sha256d(b):
    return hashlib.sha256(hashlib.sha256(b).digest()).digest()


def _typ(m):
    return struct.unpack(">H", m[:2])[0] if len(m) >= 2 else 0


def _ca_fields(m):
    """(chain_hash, scid, node_id_1, node_id_2) of a channel_announcement"""
    p = 260 + struct.unpack(">H", m[258:260])[0]
    return m[p:p + 32], m[p + 32:p + 40], m[p + 40:p + 73], m[p + 73:p + 106]


def burst_model(cln, msgs, chain, kinds, signers):
    """gossipd's decisions in message order: CLN's sigcheck for the signatures, its gates (gossmap_manage.c:659-670,
    :1048-1051) and its pending map (an announcement enters it only with status 0; an update finds the first one)"""
    out, pending = [], {}
    zero = np.zeros(33, np.uint8)
    for m, b in enumerate(msgs):
        L = ctypes.c_size_t(len(b))
        t = _typ(b)
        if t == 256:
            s = cln.cln_sigcheck_channel_announcement(b, L)
            if s != -1:
                ch, scid, n1, n2 = _ca_fields(b)
                s = -4 if n1 >= n2 else (-3 if ch != chain else s)
                if s == 0:
                    pending.setdefault(scid, b)
        elif t == 257:
            s = cln.cln_sigcheck_node_announcement(b, L)
        elif t == 258 and len(b) >= 138:
            k, key, peer = kinds[m], None, False
            if k == 1:
                key = signers[m]
            elif b[98:106] in pending:
                ann = pending[b[98:106]]
                key = _ca_fields(ann)[2 + (b[111] & 1)]
            elif k == 2:
                key, peer = signers[m], True
            kk = zero if key is None else np.frombuffer(bytes(key), np.uint8).copy()
            s = cln.cln_sigcheck_channel_update(b, L, P(kk))
            if s != -1:
                if b[66:98] != chain:
                    s = -3
                elif key is None:
                    s = -2
                elif peer:
                    s = 5 if s == 0 else -2
        else:
            s = -1
        out.append(s)
    return out


def test_whole_fixture_as_one_burst(engine):
    """every update's announcement comes earlier in the fixture and no scid repeats: all 3,100 statuses 0, equal to
    sv_verify_gossip_host fed with the signers the host-side join (tests/gossip.py:items_of) finds"""
    msgs = gossip.load_subset()
    cas = [m for m in msgs if _typ(m) == 256]
    assert len({_ca_fields(m)[1] for m in cas}) == len(cas)
    got = engine.verify_gossip_burst(msgs, TESTNET)
    assert got.tolist() == [0] * len(msgs)
    assert engine.last_gossip_repairs() == 0
    _, _, _, key, _, owner, _ = gossip.items_of(msgs)
    signers = np.zeros((len(msgs), 33), np.uint8)
    cu = [i for i, o in enumerate(owner) if _typ(msgs[o]) == 258]
    assert len(cu) == 1200
    signers[owner[cu]] = key[cu]
    assert np.array_equal(engine.verify_gossip(msgs, signers), got)
    assert np.array_equal(engine.verify_gossip_burst(msgs, TESTNET, np.zeros(len(msgs), np.uint8), signers), got)


def flipped_fixture():
    """the fixture with ~15 % of messages bit-flipped, the flips aimed at scids, chain hashes, node ids and
    channel_flags as often as anywhere else (never at the length fields); signer kinds 0, 1 and 2 mixed"""
    msgs = gossip.load_subset()
    rng = np.random.default_rng(2026)
    chans = {}
    for m in msgs:
        if _typ(m) == 256:
            ch, scid, n1, n2 = _ca_fields(m)
            chans[scid] = (n1, n2)
    batch = []
    for m in msgs:
        b = bytearray(m)
        if rng.random() < 0.15:
            t = _typ(m)
            r = rng.random()
            if t == 256:
                base = 260 + struct.unpack(">H", m[258:260])[0]
                region = [(base, base + 32), (base + 32, base + 40), (base + 40, base + 106), (2, 258)][int(r * 4)]
            elif t == 258:
                region = [(66, 98), (98, 106), (111, 112), (2, len(m))][int(r * 4)]
            else:
                region = (2, len(m))
            while True:
                pos = int(rng.integers(*region))
                if pos not in (66, 67, 258, 259):
                    break
            b[pos] ^= 1 << int(rng.integers(0, 8))
        batch.append(bytes(b))
    n = len(batch)
    kinds = np.zeros(n, np.uint8)
    signers = np.zeros((n, 33), np.uint8)
    for i, m in enumerate(msgs):
        if _typ(m) != 258:
            continue
        kinds[i] = int(rng.choice([0, 0, 0, 1, 2]))
        if kinds[i] and m[98:106] in chans:
            # kind 1: the gossmap's node for the direction; kind 2: a peer that is right half of the time
            signers[i] = np.frombuffer(chans[m[98:106]][(m[111] & 1) ^ (kinds[i] == 2 and rng.random() < 0.5)], np.uint8)
    return batch, kinds, signers


def test_burst_vs_gossipd(engine, cln):
    """every status of the bit-flipped fixture equals gossipd's decision (CLN's own sigcheck, replayed)"""
    batch, kinds, signers = flipped_fixture()
    want = burst_model(cln, batch, TESTNET, kinds, signers)
    got = engine.verify_gossip_burst(batch, TESTNET, kinds, signers)
    assert got.tolist() == want
    for code in (0, 1, -1, -2, -3, -4):
        assert code in want, code
    assert want.count(0) > 2000


# ---- crafted messages ----------------------------------------------------------------------------------------------
SK = {name: hashlib.sha256(name.encode()).digest() for name in ("a", "b", "ba", "bb", "x", "y", "z")}
PUB = {name: ecc.pubkey_create(sk)[0] for name, sk in SK.items()}


def _ordered(u, v):
    return (u, v) if PUB[u] < PUB[v] else (v, u)


def make_ca(scid, n1, n2, b1="ba", b2="bb", chain=TESTNET, bad=None, swap=False):
    """a signed channel_announcement; bad = index of a signature to corrupt; swap puts node_id_2 first"""
    ids = (PUB[n2], PUB[n1]) if swap else (PUB[n1], PUB[n2])
    tail = b"\x00\x00" + chain + scid + ids[0] + ids[1] + PUB[b1] + PUB[b2]
    h = _sha256d(tail)
    sks = [SK[n2], SK[n1]] if swap else [SK[n1], SK[n2]]
    sigs = [bytearray(ecc.ecdsa_sign(k, h)) for k in sks + [SK[b1], SK[b2]]]
    if bad is not None:
        sigs[bad][40] ^= 1
    return b"\x01\x00" + b"".join(bytes(s) for s in sigs) + tail


def make_cu(scid, signer, direction, chain=TESTNET, ts=1):
    tail = chain + scid + ts.to_bytes(4, "big") + b"\x01" + bytes([direction]) + (6).to_bytes(2, "big") + bytes(8) + \
        (1000).to_bytes(4, "big") + (1).to_bytes(4, "big") + (10 ** 9).to_bytes(8, "big")
    return b"\x01\x02" + ecc.ecdsa_sign(SK[signer], _sha256d(tail)) + tail


def _kinds(msgs, spec):
    """spec: {index: (kind, signer name)}"""
    kinds = np.zeros(len(msgs), np.uint8)
    signers = np.zeros((len(msgs), 33), np.uint8)
    for i, (k, who) in spec.items():
        kinds[i] = k
        signers[i] = np.frombuffer(PUB[who], np.uint8)
    return kinds, signers


def test_crafted_resolution_rules(engine):
    a, b = _ordered("a", "b")
    A, B, C = b"\x00\x00\x01\x00\x00\x02\x00\x01", b"\x00\x00\x01\x00\x00\x03\x00\x01", b"\x00\x00\x01\x00\x00\x04\x00\x01"
    ca = make_ca(A, a, b)
    # an update before its announcement: -2; kind 2 with the right peer: 5, with a wrong peer: -2
    msgs = [make_cu(A, a, 0), make_cu(A, a, 0), make_cu(A, a, 0), ca, make_cu(A, a, 0)]
    kinds, sg = _kinds(msgs, {1: (2, a), 2: (2, "x")})
    assert engine.verify_gossip_burst(msgs, TESTNET, kinds, sg).tolist() == [-2, 5, -2, 0, 0]
    # the direction bit selects node_id_2; a wrong one gives 1
    msgs = [ca, make_cu(A, b, 1), make_cu(A, a, 1), make_cu(A, b, 0)]
    assert engine.verify_gossip_burst(msgs, TESTNET).tolist() == [0, 0, 1, 1]
    # kind 1 overrides the batch's announcement
    msgs = [ca, make_cu(A, "x", 0), make_cu(A, a, 0)]
    kinds, sg = _kinds(msgs, {1: (1, "x"), 2: (1, "y")})
    assert engine.verify_gossip_burst(msgs, TESTNET, kinds, sg).tolist() == [0, 0, 1]
    # wrong chain: -3 for an announcement and for an update; an update of the wrong-chain announcement's scid finds none
    msgs = [make_ca(B, a, b, chain=OTHER), make_cu(B, a, 0), make_cu(A, a, 0, chain=OTHER), ca, make_cu(A, a, 0)]
    assert engine.verify_gossip_burst(msgs, TESTNET).tolist() == [-3, -2, -3, 0, 0]
    # node ids out of order: -4, and updates do not resolve to it (kind 2 falls back to the peer)
    msgs = [make_ca(C, a, b, swap=True), make_cu(C, a, 0), make_cu(C, b, 0)]
    kinds, sg = _kinds(msgs, {2: (2, b)})
    assert engine.verify_gossip_burst(msgs, TESTNET, kinds, sg).tolist() == [-4, -2, 5]
    assert engine.last_gossip_repairs() == 0
    # a node_announcement in the mix keeps its own status, a foreign type is -1
    na_tail = b"\x00\x00" + (7).to_bytes(4, "big") + PUB["z"] + b"\x01\x02\x03" + bytes(32) + b"\x00\x00"
    na = b"\x01\x01" + ecc.ecdsa_sign(SK["z"], _sha256d(na_tail)) + na_tail
    assert engine.verify_gossip_burst([na, b"\x01\x03" + bytes(200), ca], TESTNET).tolist() == [0, -1, 0]


@pytest.mark.parametrize("first", ["bad_bitcoin_signature_2", "malformed"])
def test_crafted_duplicate_announcements_repair_round(engine, first):
    """two announcements of one scid, the first failing (status 4, or -1 for a signature with r >= n): updates between
    them find no channel, updates after both resolve to the second; both took the repair round"""
    a, b = _ordered("a", "b")
    A = b"\x00\x00\x01\x00\x00\x05\x00\x01"
    if first == "malformed":
        ca1 = bytearray(make_ca(A, a, b))
        ca1[2:34] = b"\xff" * 32  # node_signature_1's r >= n: the wire parser refuses the message
        ca1, want1 = bytes(ca1), -1
    else:
        ca1, want1 = make_ca(A, a, b, bad=3), 4
    ca2 = make_ca(A, a, b, b1="x", b2="y")
    msgs = [ca1, make_cu(A, a, 0), make_cu(A, b, 1, ts=2), ca2, make_cu(A, a, 0, ts=3), make_cu(A, b, 1, ts=4),
            make_cu(A, a, 1, ts=5)]
    kinds, sg = _kinds(msgs, {2: (2, b)})  # between the two, kind 2: the peer's check
    assert engine.verify_gossip_burst(msgs, TESTNET, kinds, sg).tolist() == [want1, -2, 5, 0, 0, 0, 1]
    assert engine.last_gossip_repairs() == 5
    # the same burst beyond the small-batch limit: de-duplicated verification in both rounds
    big = msgs * 1200
    kinds_big = np.tile(kinds, 1200)
    sg_big = np.tile(sg, (1200, 1))
    got = engine.verify_gossip_burst(big, TESTNET, kinds_big, sg_big)
    # later copies: the first status-0 announcement of the scid (ca2 of copy 0) is before every later update
    want = [want1, -2, 5, 0, 0, 0, 1] + [want1, 0, 0, 0, 0, 0, 1] * 1199
    assert got.tolist() == want


def test_fixture_x53_dedup_on_and_off(engine):
    """164,300 messages (the fixture tiled 53 times: the tiles share scids, so every update resolves to tile 0): the
    same statuses with key de-duplication on and off, all 0"""
    msgs = gossip.load_subset() * 53
    engine.set_dedup(True)
    on = engine.verify_gossip_burst(msgs, TESTNET)
    assert engine.last_distinct_keys() > 0
    engine.set_dedup(False)
    try:
        off = engine.verify_gossip_burst(msgs, TESTNET)
    finally:
        engine.set_dedup(True)
    assert np.array_equal(on, off) and not on.any()


def test_argument_errors(engine):
    ca = make_ca(b"\x00" * 8, *_ordered("a", "b"))
    with pytest.raises(Exception, match="sv_verify_gossip_burst_host"):
        engine.verify_gossip_burst([ca], TESTNET, np.array([3], np.uint8), np.zeros((1, 33), np.uint8))
    with pytest.raises(Exception, match="sv_verify_gossip_burst_host"):  # kind 1 without signers
        engine.verify_gossip_burst([make_cu(b"\x00" * 8, "a", 0)], TESTNET, np.array([1], np.uint8))
    assert engine.verify_gossip_burst([], TESTNET).tolist() == []


# ---- the verifier subdaemon ----------------------------------------------------------------------------------------
def _burst_frame(rid, msgs, kinds=None, signers=None, chain=TESTNET):
    n = len(msgs)
    kinds = np.zeros(n, np.uint8) if kinds is None else kinds
    signers = np.zeros((n, 33), np.uint8) if signers is None else signers
    blob = b"".join(msgs)
    return W.encode("sigverifyd_gossip_burst", req_id=rid, chain_hash=chain, n=n, lens=[len(m) for m in msgs],
                    signer_kind=kinds.tobytes(), signers=signers.tobytes(), bloblen=len(blob), blob=blob)


def _wire_status(st):
    return [s if s >= 0 else 256 + s for s in st]


def test_daemon_bursts_from_8_clients(engine, daemon):
    """8 clients pipeline bursts (slices of the fixture, crafted duplicates), gossip requests and verify requests; every
    reply equals the in-process call, and bursts count in the stats like gossip requests"""
    fixture = gossip.load_subset()
    a, b = _ordered("a", "b")
    A = b"\x00\x00\x01\x00\x00\x06\x00\x01"
    dup = [make_ca(A, a, b, bad=1), make_cu(A, a, 0), make_ca(A, a, b), make_cu(A, b, 1), make_cu(A, a, 1)]
    plans = []
    for ci in range(8):
        rng = np.random.default_rng(80 + ci)
        plan = []
        for j in range(9):
            rid = ci * 100 + j
            if j % 3 == 0:
                lo = int(rng.integers(0, 2000))
                msgs = fixture[lo:lo + int(rng.integers(1, 1100))] + dup
                plan.append((rid, _burst_frame(rid, msgs), "sigverifyd_gossip_burst_reply",
                             _wire_status(engine.verify_gossip_burst(msgs, TESTNET).tolist())))
            elif j % 3 == 1:
                msgs = [m for m in fixture[:400] if _typ(m) != 258][:int(rng.integers(1, 60))]
                frame = W.encode("sigverifyd_gossip", req_id=rid, n=len(msgs), lens=[len(m) for m in msgs],
                                 signers=bytes(33 * len(msgs)), bloblen=sum(map(len, msgs)), blob=b"".join(msgs))
                plan.append((rid, frame, "sigverifyd_gossip_reply", _wire_status(engine.verify_gossip(msgs).tolist())))
            else:
                k = int(rng.integers(1, 5))
                h = [bytes(rng.integers(0, 256, size=32, dtype=np.uint8)) for _ in range(k)]
                sig = [ecc.ecdsa_sign(SK["x"], x) for x in h]
                if k > 1:
                    h[0] = bytes(32)
                frame = W.encode("sigverifyd_verify", req_id=rid, kind=0, n=k, hashes=b"".join(h), keylen=33 * k,
                                 keys=PUB["x"] * k, sigs=b"".join(sig))
                plan.append((rid, frame, "sigverifyd_verify_reply", [0 if (k > 1 and i == 0) else 1 for i in range(k)]))
        plans.append(plan)
    errors = []

    def client(ci):
        try:
            c = _connect(daemon)
            for _, frame, _, _ in plans[ci]:
                c.sendall(frame)
            for rid, _, want_name, want in plans[ci]:
                name, v = W.read_msg(c)
                assert (name, v["req_id"]) == (want_name, rid)
                got = v["verdicts"] if name == "sigverifyd_verify_reply" else v["status"]
                assert list(got) == want, rid
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not errors, errors
    c = _connect(daemon)
    c.sendall(W.encode("sigverifyd_stats", req_id=1))
    name, st = W.read_msg(c)
    c.close()
    assert st["requests"] == 8 * 9


def test_daemon_no_resolution_across_clients(daemon):
    """client A's announcement never signs for client B's update, even when both are pending together"""
    a, b = _ordered("a", "b")
    A = b"\x00\x00\x01\x00\x00\x07\x00\x01"
    ca, cu = make_ca(A, a, b), make_cu(A, a, 0)
    ca_client, cu_client = _connect(daemon), _connect(daemon)
    ca_client.sendall(_burst_frame(1, [ca]))
    cu_client.sendall(_burst_frame(2, [cu]))
    assert W.read_msg(ca_client) == ("sigverifyd_gossip_burst_reply", dict(req_id=1, n=1, status=b"\x00"))
    assert W.read_msg(cu_client) == ("sigverifyd_gossip_burst_reply", dict(req_id=2, n=1, status=b"\xfe"))
    cu_client.sendall(_burst_frame(3, [ca, cu]))
    assert W.read_msg(cu_client) == ("sigverifyd_gossip_burst_reply", dict(req_id=3, n=2, status=b"\x00\x00"))
    ca_client.close()
    cu_client.close()


def test_daemon_refusals(daemon):
    """each refusal rule gets sigverifyd_error code 1 and the connection keeps serving"""
    c = _connect(daemon)
    a, b = _ordered("a", "b")
    ca = make_ca(b"\x00\x00\x01\x00\x00\x08\x00\x01", a, b)

    def refused(rid, frame):
        c.sendall(frame)
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=rid, code=1)), rid

    too_many = (1 << 20) + 1
    refused(11, W.encode("sigverifyd_gossip_burst", req_id=11, chain_hash=TESTNET, n=too_many, lens=bytes(4 * too_many),
                         signer_kind=bytes(too_many), signers=bytes(33 * too_many), bloblen=0, blob=b""))
    body = _burst_frame(12, [ca, ca])[4:]
    lens_at = 2 + 8 + 32 + 4
    for rid, lens in ((12, [len(ca), len(ca) + 1]), (13, [len(ca), len(ca) - 1]), (14, [0xFFFFFFFF, 2 * len(ca) + 1])):  # 14: the 32-bit sum wraps to bloblen
        lb = b"".join(x.to_bytes(4, "big") for x in lens)
        bad = body[:2] + rid.to_bytes(8, "big") + body[10:lens_at] + lb + body[lens_at + 8:]
        refused(rid, len(bad).to_bytes(4, "big") + bad)
    refused(15, _burst_frame(15, [ca, ca], kinds=np.array([0, 3], np.uint8)))
    short = _burst_frame(16, [ca])[4:-1]
    refused(16, len(short).to_bytes(4, "big") + short)
    c.sendall(_burst_frame(17, [ca]))
    assert W.read_msg(c) == ("sigverifyd_gossip_burst_reply", dict(req_id=17, n=1, status=b"\x00"))
    c.close()


CLIENT = r"""
import ctypes, json, sys
from lightning_b200 import engine
lib = ctypes.CDLL(engine.LIB_PATH)
vp, sz = ctypes.c_void_p, ctypes.c_size_t
lib.sigcheck_gossip_batch.argtypes = [vp, vp, vp, sz, vp, vp, vp]
sc = json.load(open(sys.argv[1]))
out = []
for b in sc["bursts"]:
    msgs = [bytes.fromhex(m) for m in b["msgs"]]
    n = len(msgs)
    bufs = [ctypes.create_string_buffer(m, len(m)) for m in msgs]
    ptrs = (ctypes.c_void_p * n)(*[ctypes.addressof(x) for x in bufs])
    lens = (ctypes.c_size_t * n)(*[len(m) for m in msgs])
    kinds = (ctypes.c_uint8 * n)(*b["kinds"]) if b["kinds"] is not None else None
    sg = ctypes.create_string_buffer(bytes.fromhex(b["signers"]), 33 * n) if b["signers"] else None
    chain = ctypes.create_string_buffer(bytes.fromhex(sc["chain"]), 32)
    st = (ctypes.c_int * n)()
    lib.sigcheck_gossip_batch(chain, ptrs, lens, n, kinds, sg, st)
    out.append(list(st))
print(json.dumps(out))
"""


def test_dropin_client_mode_gossip_batch(engine, daemon, tmp_path):
    """sigcheck_gossip_batch in client mode with no visible GPU (opening a context would abort): the statuses of the
    in-process run and of the engine, one request per call"""
    a, b = _ordered("a", "b")
    A = b"\x00\x00\x01\x00\x00\x09\x00\x01"
    fixture = gossip.load_subset()
    crafted = [make_cu(A, a, 0), make_ca(A, a, b, bad=2), make_cu(A, a, 0), make_ca(A, a, b), make_cu(A, b, 1),
               make_cu(A, a, 0, chain=OTHER)]
    kinds = [2, 0, 0, 0, 1, 0]
    signers = np.zeros((6, 33), np.uint8)
    signers[0] = np.frombuffer(PUB[a], np.uint8)
    signers[4] = np.frombuffer(PUB[b], np.uint8)
    bursts = [dict(msgs=[m.hex() for m in fixture[:900]], kinds=None, signers=None),
              dict(msgs=[m.hex() for m in crafted], kinds=kinds, signers=signers.tobytes().hex())]
    path = tmp_path / "bursts.json"
    json.dump(dict(chain=TESTNET.hex(), bursts=bursts), open(path, "w"))
    base = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base.pop("CLN_SIGVERIFYD_SOCKET", None)

    def run(env):
        r = subprocess.run([sys.executable, "-c", CLIENT, str(path)], env=env, cwd=str(tmp_path), capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        return json.loads(r.stdout)

    local = run(base)
    remote = run(dict(base, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES=""))
    assert remote == local
    assert local[0] == engine.verify_gossip_burst(fixture[:900], TESTNET).tolist()
    assert local[1] == [5, 3, -2, 0, 0, -3]
    c = _connect(daemon)
    c.sendall(W.encode("sigverifyd_stats", req_id=1))
    assert W.read_msg(c)[1]["requests"] == 2
    c.close()
