"""BOLT12 checks through the verifier subdaemon (cln_sigverifyd): sigverifyd_bolt12 requests of many clients coalesced
into shared launches, malformed requests, and the drop-in library's client mode (CLN_SIGVERIFYD_SOCKET), which must never
open a CUDA context of its own.  Expected answers come from tests/golden/bolt12_vectors.npz (the reference's status and
sighash per item) and, for ECDSA, from signatures made with tests/ecc.py."""
import json
import os
import resource
import signal
import socket
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import bolt12, ecc
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx():
    return bolt12.load_fixture()


def _bolt12_request(fx, rid, ni, items, want):
    streams = bolt12.streams(fx)
    mn, fn = bolt12.NAMES[ni]
    blob = b"".join(streams[i] for i in items)
    return W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn,
                    n=len(items), lens=[len(streams[i]) for i in items], bloblen=len(blob), blob=blob,
                    xonly=fx["xonly"][items].tobytes(), sigs=fx["sig"][items].tobytes(), want_sighash=want)


def test_coalesced_bolt12_and_verify_requests(fx, daemon):
    """8 clients x 30 requests in flight: BOLT12 requests of 1..40 streams under both tags (some asking for the
    sighashes) mixed with BIP-340 sigverifyd_verify requests; every reply vs the fixture, replies in request order"""
    groups = [np.nonzero(fx["names"] == ni)[0] for ni in range(len(bolt12.NAMES))]
    parsed = np.nonzero(fx["status"] >= 0)[0]
    errors = []

    def client(ci):
        try:
            rng = np.random.default_rng(100 + ci)
            c = _connect(daemon)
            sent = []
            for j in range(30):
                rid = ci * 1000 + j
                k = int(rng.integers(1, 41))
                if j % 5 == 4:  # a pre-hashed BIP-340 request: the fixture's sighashes of streams that parse
                    items = rng.choice(parsed, size=k)
                    c.sendall(W.encode("sigverifyd_verify", req_id=rid, kind=2, n=k, hashes=fx["sighash"][items].tobytes(),
                                       keylen=32 * k, keys=fx["xonly"][items].tobytes(), sigs=fx["sig"][items].tobytes()))
                    sent.append((rid, "verify", items, False))
                else:
                    ni = int(rng.integers(0, 2))
                    items = rng.choice(groups[ni], size=k)
                    want = int(j % 3 == 0)
                    c.sendall(_bolt12_request(fx, rid, ni, items, want))
                    sent.append((rid, "bolt12", items, want))
            for rid, what, items, want in sent:
                name, v = W.read_msg(c)
                assert v["req_id"] == rid, ("order", rid, v["req_id"])
                if what == "verify":
                    assert name == "sigverifyd_verify_reply"
                    got = np.frombuffer(v["verdicts"], np.uint8)
                    assert np.array_equal(got, (fx["status"][items] == 1).astype(np.uint8)), rid
                else:
                    assert name == "sigverifyd_bolt12_reply" and v["n"] == len(items)
                    got = np.frombuffer(v["status"], np.uint8).astype(np.int32)
                    got[got == 255] = -1
                    assert np.array_equal(got, fx["status"][items].astype(np.int32)), rid
                    assert v["nsighash"] == (len(items) if want else 0)
                    if want:
                        assert v["sighashes"] == fx["sighash"][items].tobytes(), rid
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
    c.sendall(W.encode("sigverifyd_stats", req_id=5))
    name, st = W.read_msg(c)
    assert name == "sigverifyd_stats_reply" and st["requests"] == 240, st
    assert st["launches"] < st["requests"] and st["max_coalesced"] >= 2, st
    c.close()


def test_malformed_bolt12_request(fx, daemon):
    """a malformed request is answered with sigverifyd_error code 1; the same connection then serves a good one"""
    c = _connect(daemon)
    items = np.nonzero(fx["names"] == 0)[0][:3]
    good = _bolt12_request(fx, 9, 0, items, 1)
    body = good[4:]
    name_at = 2 + 8
    mnl = int.from_bytes(body[name_at:name_at + 2], "big")
    n_at = name_at + 2 + mnl + 2 + 9
    lens_at = n_at + 4

    def frame(b):
        return len(b).to_bytes(4, "big") + b

    bads = [
        body[:lens_at] + (int.from_bytes(body[lens_at:lens_at + 4], "big") + 1).to_bytes(4, "big") + body[lens_at + 4:],
        body[:name_at] + (0).to_bytes(2, "big") + body[name_at + 2 + mnl:],  # empty messagename
        body[:name_at + 2] + b"inv\0ice" + body[name_at + 2 + 7:],  # a NUL inside the messagename
        body[:-1],  # truncated: does not parse
    ]
    for k, b in enumerate(bads):
        b = b[:2] + (100 + k).to_bytes(8, "big") + b[10:]
        c.sendall(frame(b))
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=100 + k, code=1)), k
    c.sendall(good)
    name, v = W.read_msg(c)
    assert name == "sigverifyd_bolt12_reply" and v["req_id"] == 9
    assert list(np.frombuffer(v["status"], np.uint8).astype(np.int8)) == list(fx["status"][items])
    assert v["sighashes"] == fx["sighash"][items].tobytes()
    c.close()


# the client-mode subprocess: loads the library, never creates an engine context (there is no visible GPU), and prints
# its answers as JSON
CLIENT = r"""
import ctypes, json, sys
import numpy as np
from lightning_b200 import engine
from tests import bolt12, ecc
lib = ctypes.CDLL(engine.LIB_PATH)
vp = ctypes.c_void_p
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
for f in ("bolt12_check_signature", "check_schnorr_sig", "check_signed_hash_nodeid"):
    getattr(lib, f).restype = ctypes.c_bool
lib.bolt12_check_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp]
lib.check_schnorr_sig.argtypes = [vp, vp, vp]
lib.check_signed_hash_nodeid.argtypes = [vp, vp, vp]
class TlvField(ctypes.Structure):
    _fields_ = [("meta", vp), ("numtype", ctypes.c_uint64), ("length", ctypes.c_size_t), ("value", ctypes.POINTER(ctypes.c_uint8))]
sizes = {}
hook = ctypes.CFUNCTYPE(ctypes.c_size_t, vp)(lambda p: sizes[p])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(hook, vp), None)
fx = bolt12.load_fixture()
streams = bolt12.streams(fx)
out = {"bolt12": [], "schnorr": [], "nodeid": []}
def buf(b):
    return (ctypes.c_uint8 * len(b)).from_buffer_copy(b)
for i in range(0, len(streams), 7):
    if fx["status"][i] < 0:
        continue
    conv = ecc.pubkey_convert(b"\x02" + fx["xonly"][i].tobytes())
    if conv is None:
        continue
    xy = conv[1]
    pub = buf(xy[31::-1] + xy[:31:-1])
    sig = buf(fx["sig"][i].tobytes())
    fields = bolt12.parse_fields(streams[i])
    arr = (TlvField * max(len(fields), 1))()
    keep = []
    for k, (t, _vo, v) in enumerate(fields):
        b = buf(v + b"\0")
        keep.append(b)
        arr[k] = TlvField(None, t, len(v), ctypes.cast(b, ctypes.POINTER(ctypes.c_uint8)))
    sizes[ctypes.addressof(arr)] = len(fields) * ctypes.sizeof(TlvField)
    mn, fn = bolt12.NAMES[fx["names"][i]]
    got = lib.bolt12_check_signature(ctypes.addressof(arr), mn, fn, ctypes.addressof(pub), ctypes.addressof(sig))
    out["bolt12"].append([i, bool(got)])
    if len(out["schnorr"]) < 40:
        h = buf(fx["sighash"][i].tobytes())
        out["schnorr"].append([i, bool(lib.check_schnorr_sig(ctypes.addressof(h), ctypes.addressof(pub), ctypes.addressof(sig)))])
for j in range(6):
    sk = bytes([j + 1]) * 32
    pub33 = ecc.pubkey_create(sk)[0]
    msg = bytes([0xA0 + j]) * 32
    rs = ecc.ecdsa_sign(sk, msg)
    if j % 2:
        msg = bytes([msg[0] ^ 1]) + msg[1:]  # a known-bad triple: the signature is over another message
    s = buf(rs[31::-1] + rs[:31:-1])  # secp256k1_ecdsa_signature: r and s as little-endian limbs
    h, k = buf(msg), buf(pub33)
    out["nodeid"].append([j, bool(lib.check_signed_hash_nodeid(ctypes.addressof(h), ctypes.addressof(s), ctypes.addressof(k)))])
print(json.dumps(out))
"""


def _client_env(sock_path):
    env = dict(os.environ, CLN_SIGVERIFYD_SOCKET=sock_path, CUDA_VISIBLE_DEVICES="",
               PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return env


def _no_core():
    resource.setrlimit(resource.RLIMIT_CORE, (0, 0))


def test_dropin_client_mode(fx, daemon, tmp_path):
    r = subprocess.run([sys.executable, "-c", CLIENT], env=_client_env(daemon), cwd=str(tmp_path), capture_output=True,
                       text=True, timeout=600, preexec_fn=_no_core)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout)
    assert len(out["bolt12"]) > 100 and len(out["schnorr"]) == 40
    for i, got in out["bolt12"] + out["schnorr"]:
        assert got == (fx["status"][i] == 1), i
    assert [g for _, g in out["nodeid"]] == [True, False] * 3
    c = _connect(daemon)
    c.sendall(W.encode("sigverifyd_stats", req_id=1))
    _, st = W.read_msg(c)
    assert st["requests"] == len(out["bolt12"]) + 40 + 6, st  # every check went through the daemon
    c.close()


def test_dropin_client_mode_lost_daemon_aborts(tmp_path):
    """no daemon behind the socket: the library aborts (its rule for internal errors) rather than answer false"""
    path = str(tmp_path / "gone.sock")
    s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    s.bind(path)
    s.close()  # the socket file stays, nobody listens
    r = subprocess.run([sys.executable, "-c", CLIENT], env=_client_env(path), cwd=str(tmp_path), capture_output=True,
                       text=True, timeout=600, preexec_fn=_no_core)
    assert r.returncode == -signal.SIGABRT, (r.returncode, r.stderr[-2000:])
    assert "cannot connect" in r.stderr and r.stdout == ""
