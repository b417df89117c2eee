"""sha256_double and pubkey_from_der through the verifier subdaemon (cln_sigverifyd): sigverifyd_sha256d and
sigverifyd_pubkey requests of many clients coalesced into shared launches, malformed requests, and the drop-in library's
client mode for both functions, which must never open a CUDA context of its own.  Hashes are checked against hashlib,
keys against the in-process engine (sv_pubkey_parse_host) and tests/golden/pubkey_parse.json (the reference's
run_ec_pubkey_parse_test tables)."""
import hashlib
import json
import os
import resource
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import ecc
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)
from tests.sigverifyd_daemon import stats as _stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
BOUNDARIES = [0, 1, 55, 56, 63, 64, 119, 120, 174]  # every SHA-256 padding boundary of one and two blocks


def _sha256d(b):
    return hashlib.sha256(hashlib.sha256(b).digest()).digest()


def _golden_keys():
    """the 33-byte encodings of the golden tables with their expected verdict and point"""
    return [v for v in json.load(open(os.path.join(GOLD, "pubkey_parse.json"))) if "pub33" in v]


def _sha_request(rid, bufs):
    blob = b"".join(bufs)
    return W.encode("sigverifyd_sha256d", req_id=rid, n=len(bufs), lens=[len(b) for b in bufs], bloblen=len(blob),
                    blob=blob)


def _key_request(rid, keys):
    return W.encode("sigverifyd_pubkey", req_id=rid, n=len(keys), keys=b"".join(keys))


def test_coalesced_hash_and_key_requests(engine, daemon):
    """8 clients x 24 requests in flight: sha256d requests (buffers on every padding boundary, some of 100 kB, some
    requests empty), pubkey requests (the golden tables and random valid keys) and ECDSA verify requests; every hash is
    SHA-256 twice, every key result is the in-process engine's and the golden table's, each client's replies arrive in
    request order, and the requests shared launches"""
    gold = _golden_keys()
    gold_keys = [bytes.fromhex(v["pub33"]) for v in gold]
    rng = np.random.default_rng(9)
    signers = []
    for s in range(16):
        sk = bytes(rng.integers(1, 256, size=32, dtype=np.uint8))
        signers.append((sk, ecc.pubkey_create(sk)[0]))
    plans = []
    for ci in range(8):
        rng = np.random.default_rng(600 + ci)
        plan = []
        for j in range(24):
            rid = ci * 1000 + j
            if j % 3 == 0:
                n = 0 if j == 21 else int(rng.integers(1, 12))
                sizes = [int(rng.choice(BOUNDARIES)) if rng.random() < 0.85 else 100_000 for _ in range(n)]
                bufs = [bytes(rng.integers(0, 256, size=s, dtype=np.uint8)) for s in sizes]
                plan.append((rid, _sha_request(rid, bufs), "sigverifyd_sha256d_reply", bufs))
            elif j % 3 == 1:
                keys = [gold_keys[int(k)] for k in rng.integers(0, len(gold_keys), size=int(rng.integers(0, 6)))]
                keys += [signers[int(k)][1] for k in rng.integers(0, len(signers), size=int(rng.integers(1, 6)))]
                keys = [keys[int(k)] for k in rng.permutation(len(keys))]
                plan.append((rid, _key_request(rid, keys), "sigverifyd_pubkey_reply", keys))
            else:
                n = int(rng.integers(1, 8))
                items = []
                for _ in range(n):
                    sk, pub33 = signers[int(rng.integers(0, len(signers)))]
                    msg = bytes(rng.integers(0, 256, size=32, dtype=np.uint8))
                    sig = bytearray(ecc.ecdsa_sign(sk, msg))
                    good = rng.random() < 0.7
                    if not good:
                        sig[int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
                    items.append((msg, pub33, bytes(sig)))
                frame = W.encode("sigverifyd_verify", req_id=rid, kind=0, n=n, hashes=b"".join(i[0] for i in items),
                                 keylen=33 * n, keys=b"".join(i[1] for i in items), sigs=b"".join(i[2] for i in items))
                plan.append((rid, frame, "sigverifyd_verify_reply", items))
        plans.append(plan)
    errors, got = [], [None] * 8

    def client(ci):
        try:
            c = _connect(daemon)
            for _, frame, _, _ in plans[ci]:
                c.sendall(frame)
            replies = []
            for rid, _, want_name, _ in plans[ci]:
                name, v = W.read_msg(c)
                assert v["req_id"] == rid, ("order", rid, v["req_id"])
                assert name == want_name, (rid, name)
                replies.append(v)
            c.close()
            got[ci] = replies
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not errors, errors
    all_keys, key_ok, key_xy = [], [], []
    verify_items, verdicts = [], []
    for ci in range(8):
        for (rid, _, name, what), v in zip(plans[ci], got[ci]):
            assert v["n"] == len(what), rid
            if name == "sigverifyd_sha256d_reply":
                assert v["hashes"] == b"".join(_sha256d(b) for b in what), rid
            elif name == "sigverifyd_pubkey_reply":
                all_keys += what
                key_ok.append(np.frombuffer(v["ok"], np.uint8))
                key_xy.append(np.frombuffer(v["xy"], np.uint8).reshape(-1, 64))
            else:
                verify_items += what
                verdicts.append(np.frombuffer(v["verdicts"], np.uint8))
    key_ok, key_xy = np.concatenate(key_ok), np.concatenate(key_xy)
    want_xy, want_ok = engine.pubkey_parse(np.frombuffer(b"".join(all_keys), np.uint8).reshape(-1, 33))
    assert np.array_equal(key_ok, want_ok) and np.array_equal(key_xy, want_xy)
    by_key = {bytes.fromhex(v["pub33"]): v for v in gold}
    seen_bad = 0
    for k, ok, xy in zip(all_keys, key_ok, key_xy):
        if k in by_key:
            assert ok == by_key[k]["expected"], k.hex()
            assert bytes(xy).hex() == (by_key[k]["xy"] if ok else "00" * 64), k.hex()
            seen_bad += not ok
        else:
            assert ok == 1 and bytes(xy) == ecc.pubkey_convert(k)[1], k.hex()
    assert seen_bad > 10  # invalid encodings were among them
    verdicts = np.concatenate(verdicts)
    msg = np.frombuffer(b"".join(i[0] for i in verify_items), np.uint8).reshape(-1, 32)
    pub = np.frombuffer(b"".join(i[1] for i in verify_items), np.uint8).reshape(-1, 33)
    sig = np.frombuffer(b"".join(i[2] for i in verify_items), np.uint8).reshape(-1, 64)
    assert np.array_equal(verdicts, engine.verify(0, msg, pub, sig))
    assert 0.4 * verdicts.size < verdicts.sum() < 0.95 * verdicts.size
    st = _stats(daemon)
    assert st["requests"] == 8 * 24, st
    assert st["signatures"] == verdicts.size, st  # hashes and keys are not signatures
    assert st["launches"] < st["requests"] and st["max_coalesced"] >= 2, st


def test_malformed_hash_and_key_requests(daemon):
    """each refusal rule gets sigverifyd_error code 1; the same connection then serves a good request of each kind"""
    c = _connect(daemon)

    def refused(rid, frame):
        c.sendall(frame)
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=rid, code=1)), rid

    too_many = (1 << 20) + 1
    refused(101, W.encode("sigverifyd_sha256d", req_id=101, n=too_many, lens=bytes(4 * too_many), bloblen=0, blob=b""))
    refused(102, W.encode("sigverifyd_pubkey", req_id=102, n=too_many, keys=bytes(33 * too_many)))
    blob = bytes(range(100))
    refused(103, W.encode("sigverifyd_sha256d", req_id=103, n=2, lens=[60, 41], bloblen=100, blob=blob))  # too long
    refused(104, W.encode("sigverifyd_sha256d", req_id=104, n=2, lens=[60, 39], bloblen=100, blob=blob))  # too short
    # lengths whose 32-bit sum wraps around to the blob's length
    refused(105, W.encode("sigverifyd_sha256d", req_id=105, n=2, lens=[0xFFFFFFFF, 101], bloblen=100, blob=blob))
    for rid, frame in ((106, _sha_request(106, [blob[:55], b""])), (107, _key_request(107, [bytes(33)] * 2))):
        body = frame[4:-1]  # one byte short of its fields: does not parse
        refused(rid, len(body).to_bytes(4, "big") + body)
    key = ecc.pubkey_create(bytes([7]) * 32)
    c.sendall(_sha_request(9, [blob[:55], b"", blob]))
    c.sendall(_key_request(10, [key[0], bytes(33)]))
    name, v = W.read_msg(c)
    assert name == "sigverifyd_sha256d_reply" and v["req_id"] == 9
    assert v["hashes"] == _sha256d(blob[:55]) + _sha256d(b"") + _sha256d(blob)
    name, v = W.read_msg(c)
    assert name == "sigverifyd_pubkey_reply" and v["req_id"] == 10
    assert v["ok"] == b"\1\0" and v["xy"] == key[1] + bytes(64)
    c.close()


# the drop-in library driven through its C ABI: pubkey_from_der, sha256_double, then check_signed_hash and
# check_signed_hash_nodeid on the parsed keys and computed hashes; prints its answers and the number of requests it
# expects to have sent.  Run once with a GPU and no daemon (in-process) and once in client mode without a visible GPU.
CLIENT = r"""
import ctypes, json, sys
from lightning_b200 import engine
lib = ctypes.CDLL(engine.LIB_PATH)
vp, sz = ctypes.c_void_p, ctypes.c_size_t
for f in ("pubkey_from_der", "check_signed_hash", "check_signed_hash_nodeid"):
    getattr(lib, f).restype = ctypes.c_bool
lib.pubkey_from_der.argtypes = [vp, sz, vp]
lib.sha256_double.argtypes = [vp, vp, sz]
lib.check_signed_hash.argtypes = [vp, vp, vp]
lib.check_signed_hash_nodeid.argtypes = [vp, vp, vp]
def buf(b):
    return (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
sc = json.load(open(sys.argv[1]))
out = {"keys": [], "hashes": [], "signed": [], "nodeid": [], "sent": 0}
pubs = {}
for k in sc["keys"]:
    der = bytes.fromhex(k)
    pk = (ctypes.c_uint8 * 64)()
    ok = lib.pubkey_from_der(buf(der), len(der), pk)
    out["keys"].append(bytes(pk).hex() if ok else None)
    out["sent"] += len(der) == 33
    if ok:
        pubs[k] = pk
hashes = []
for d in sc["data"]:
    data = bytes.fromhex(d)
    h = (ctypes.c_uint8 * 32)()
    lib.sha256_double(h, buf(data), len(data))
    hashes.append(h)
    out["hashes"].append(bytes(h).hex())
    out["sent"] += 1
for key, hi, sig in sc["sigs"]:
    rs = bytes.fromhex(sig)
    s = buf(rs[31::-1] + rs[:31:-1])  # secp256k1_ecdsa_signature: r and s as little-endian limbs
    out["signed"].append(bool(lib.check_signed_hash(hashes[hi], s, pubs[key])))
    out["nodeid"].append(bool(lib.check_signed_hash_nodeid(hashes[hi], s, buf(bytes.fromhex(key)))))
    out["sent"] += 2
print(json.dumps(out))
"""


def _scenario(tmp_path):
    """keys: the golden tables, signers' keys and lengths other than 33; buffers on every padding boundary and of
    100 kB; one signature per (signer, buffer) over the buffer's SHA-256d, every third corrupted"""
    rng = np.random.default_rng(31)
    signers = [ecc.pubkey_create(bytes([0x31 + s]) * 32)[0] for s in range(4)]
    keys = [bytes.fromhex(v["pub33"]) for v in _golden_keys()] + signers
    keys += [b"", signers[0][:32], signers[0] + b"\0", b"\4" + ecc.pubkey_create(bytes([0x31]) * 32)[1]]
    data = [bytes(rng.integers(0, 256, size=n, dtype=np.uint8)) for n in BOUNDARIES + [100_000, 100_001]]
    sigs = []
    for s, pub in enumerate(signers):
        for hi, d in enumerate(data):
            sig = bytearray(ecc.ecdsa_sign(bytes([0x31 + s]) * 32, _sha256d(d)))
            if (s + hi) % 3 == 1:
                sig[int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
            sigs.append([pub.hex(), hi, bytes(sig).hex()])
    sc = dict(keys=[k.hex() for k in keys], data=[d.hex() for d in data], sigs=sigs)
    path = tmp_path / "scenario.json"
    json.dump(sc, open(path, "w"))
    return str(path), sc


def _no_core():
    resource.setrlimit(resource.RLIMIT_CORE, (0, 0))


def _run_client(path, tmp_path, env):
    r = subprocess.run([sys.executable, "-c", CLIENT, path], env=env, cwd=str(tmp_path), capture_output=True, text=True,
                       timeout=600, preexec_fn=_no_core)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def test_dropin_client_mode_hash_and_key(daemon, tmp_path):
    """pubkey_from_der and sha256_double in client mode, with no visible GPU (creating a context would abort), followed by
    check_signed_hash / check_signed_hash_nodeid on what they returned: exactly the in-process answers, and every call
    except pubkey_from_der on a length other than 33 went through the daemon"""
    path, sc = _scenario(tmp_path)
    base = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base.pop("CLN_SIGVERIFYD_SOCKET", None)
    local = _run_client(path, tmp_path, base)
    remote = _run_client(path, tmp_path, dict(base, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES=""))
    assert remote == local
    gold = _golden_keys()
    for k, got in zip(sc["keys"], local["keys"]):
        der = bytes.fromhex(k)
        conv = ecc.pubkey_convert(der) if len(der) == 33 else None
        want = conv[1] if conv else None
        if got is not None:  # struct pubkey holds x and y as little-endian limbs
            got = bytes.fromhex(got)
            got = got[31::-1] + got[:31:-1]
        assert got == want, k
    assert sum(g is None for g in local["keys"]) > 10 + 4
    assert [local["keys"][i] is not None for i in range(len(gold))] == [bool(v["expected"]) for v in gold]
    assert local["hashes"] == [_sha256d(bytes.fromhex(d)).hex() for d in sc["data"]]
    want = [(s + hi) % 3 != 1 for s in range(4) for hi in range(len(sc["data"]))]
    assert local["signed"] == want and local["nodeid"] == want
    sent = sum(len(k) == 66 for k in sc["keys"]) + len(sc["data"]) + 2 * len(sc["sigs"])
    assert remote["sent"] == sent and _stats(daemon)["requests"] == sent
