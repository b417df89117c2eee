"""BOLT11 checks through the verifier subdaemon (cln_sigverifyd): sigverifyd_bolt11 requests of many clients coalesced
into shared sv_verify_bolt11_host launches beside BOLT12 and sigverifyd_verify requests, malformed requests, and the
drop-in's bolt11_check_signature in client mode (CLN_SIGVERIFYD_SOCKET, no visible GPU) and in process.  Every answer must
be byte-identical to one in-process SigVerifier.verify_bolt11 call over the whole fixture (tests/golden/bolt11_vectors.npz),
and equal to Core Lightning's recorded answer wherever the fixture checks one."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import bolt11, bolt12
from tests.sigverifyd_daemon import connect as _connect
from tests.sigverifyd_daemon import daemon  # noqa: F401  (fixture)
from tests.sigverifyd_daemon import stats as _stats

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ITEMS = 1 << 20


@pytest.fixture(scope="module")
def fx():
    return bolt11.load_fixture()


@pytest.fixture(scope="module")
def fx12():
    return bolt12.load_fixture()


@pytest.fixture(scope="module")
def ref(engine, fx):
    """status (n,), receiver ids (n, 33): one in-process call over the whole fixture, checked against CLN's answers"""
    status, node, _ = engine.verify_bolt11(bolt11.invoices(fx))
    e = fx["expected"]
    m = e != bolt11.UNCHECKED
    assert np.array_equal(status[m], e[m])
    np.testing.assert_array_equal(node[e == 1], fx["node"][e == 1])
    assert not node[status != 1].any()
    return status.astype(np.int32), node


def _bolt11_request(fx, rid, items):
    invs = bolt11.invoices(fx)
    blob = b"".join(invs[i] for i in items)
    return W.encode("sigverifyd_bolt11", req_id=rid, n=len(items), lens=[len(invs[i]) for i in items], bloblen=len(blob),
                    blob=blob)


def _check_reply(fx, ref, v, items, rid):
    assert v["req_id"] == rid and v["n"] == len(items), ("order", rid, v["req_id"])
    got = np.frombuffer(v["status"], np.uint8).astype(np.int32)
    got[got == 255] = -1
    assert np.array_equal(got, ref[0][items]), rid
    assert v["node_ids"] == ref[1][items].tobytes(), rid
    e = fx["expected"][items]
    m = e != bolt11.UNCHECKED
    assert np.array_equal(got[m], e[m]), rid
    node = np.frombuffer(v["node_ids"], np.uint8).reshape(-1, 33)
    np.testing.assert_array_equal(node[e == 1], fx["node"][items][e == 1])


def _plan(n_items, fx12):
    """per client, 30 requests: BOLT11 requests of 1-40 items taken in turn from the client's share of a permutation of
    the fixture (so that together they send every item), every tenth a BIP-340 sigverifyd_verify request and every tenth a
    BOLT12 request"""
    perm = np.random.default_rng(1).permutation(n_items)
    parsed = np.nonzero(fx12["status"] >= 0)[0]
    groups = [np.nonzero(fx12["names"] == ni)[0] for ni in range(len(bolt12.NAMES))]
    plans = []
    for ci in range(8):
        rng = np.random.default_rng(300 + ci)
        mine, pos, reqs = perm[ci::8], 0, []
        for j in range(30):
            k = int(rng.integers(1, 41))
            if j % 10 == 9:
                reqs.append(("verify", rng.choice(parsed, size=k), None))
            elif j % 10 == 4:
                ni = int(rng.integers(0, 2))
                reqs.append(("bolt12", rng.choice(groups[ni], size=k), ni))
            else:
                reqs.append(("bolt11", mine[(pos + np.arange(k)) % len(mine)], None))
                pos += k
        plans.append(reqs)
    return plans


def test_coalesced_bolt11_requests(fx, fx12, ref, daemon):
    """8 clients x 30 requests in flight, BOLT11 requests of 1-40 items mixed with BOLT12 and BIP-340 requests: every
    reply in request order and byte-identical to the in-process call; fewer launches than requests"""
    plans = _plan(len(fx["ret"]), fx12)
    sent11 = np.concatenate([items for p in plans for what, items, _ in p if what == "bolt11"])
    assert np.array_equal(np.unique(sent11), np.arange(len(fx["ret"])))  # every item at least once
    streams = bolt12.streams(fx12)
    errors = []

    def client(ci):
        try:
            c = _connect(daemon)
            for j, (what, items, ni) in enumerate(plans[ci]):
                rid = ci * 1000 + j
                if what == "bolt11":
                    c.sendall(_bolt11_request(fx, rid, items))
                elif what == "verify":
                    c.sendall(W.encode("sigverifyd_verify", req_id=rid, kind=2, n=len(items),
                                       hashes=fx12["sighash"][items].tobytes(), keylen=32 * len(items),
                                       keys=fx12["xonly"][items].tobytes(), sigs=fx12["sig"][items].tobytes()))
                else:
                    mn, fn = bolt12.NAMES[ni]
                    blob = b"".join(streams[i] for i in items)
                    c.sendall(W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn),
                                       fieldname=fn, n=len(items), lens=[len(streams[i]) for i in items], bloblen=len(blob),
                                       blob=blob, xonly=fx12["xonly"][items].tobytes(), sigs=fx12["sig"][items].tobytes(),
                                       want_sighash=0))
            for j, (what, items, _) in enumerate(plans[ci]):
                rid = ci * 1000 + j
                name, v = W.read_msg(c)
                assert name == "sigverifyd_%s_reply" % what, (name, rid)
                if what == "bolt11":
                    _check_reply(fx, ref, v, items, rid)
                elif what == "verify":
                    assert v["req_id"] == rid
                    assert np.array_equal(np.frombuffer(v["verdicts"], np.uint8), (fx12["status"][items] == 1).astype(np.uint8))
                else:
                    assert v["req_id"] == rid
                    got = np.frombuffer(v["status"], np.uint8).astype(np.int32)
                    got[got == 255] = -1
                    assert np.array_equal(got, fx12["status"][items].astype(np.int32)), rid
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errors, errors
    st = _stats(daemon)
    assert st["requests"] == 240 and st["launches"] < st["requests"] and st["max_coalesced"] >= 2, st


def test_malformed_bolt11_requests(fx, ref, daemon):
    """spans that do not add up, a truncated frame and n above MAX_ITEMS are each answered with sigverifyd_error code 1;
    the same connection then answers a good request correctly"""
    items = np.nonzero(fx["expected"] == 1)[0][:3]
    good = _bolt11_request(fx, 9, items)
    body = good[4:]
    first = int.from_bytes(body[14:18], "big")

    def frame(b):
        return len(b).to_bytes(4, "big") + b

    bads = [body[:14] + (first + 1).to_bytes(4, "big") + body[18:],
            body[:-1],
            W.encode("sigverifyd_bolt11", req_id=0, n=MAX_ITEMS + 1, lens=bytes(4 * (MAX_ITEMS + 1)), bloblen=0,
                     blob=b"")[4:]]
    c = _connect(daemon)
    for k, b in enumerate(bads):
        b = b[:2] + (100 + k).to_bytes(8, "big") + b[10:]
        c.sendall(frame(b))
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=100 + k, code=1)), k
    c.sendall(good)
    name, v = W.read_msg(c)
    assert name == "sigverifyd_bolt11_reply"
    _check_reply(fx, ref, v, items, 9)
    c.close()


# the drop-in in a process of its own: bolt11_check_signature on every fixture item, then (with a window) every item again
# as tickets kept that many in flight; prints the answers as JSON
CLIENT = r"""
import ctypes, json, select, sys
from lightning_b200 import engine
from tests import bolt11
window = int(sys.argv[1])
lib = ctypes.CDLL(engine.LIB_PATH)
DONE = ctypes.CFUNCTYPE(None, ctypes.c_void_p)
vp = ctypes.c_void_p
lib.bolt11_check_signature.restype = ctypes.c_int
lib.bolt11_check_signature.argtypes = [ctypes.c_char_p, vp]
lib.bolt11_check_signature_start.restype = ctypes.c_uint64
lib.bolt11_check_signature_start.argtypes = [ctypes.c_char_p, vp, vp, DONE, vp]
lib.cln_sigverify_process.restype = ctypes.c_size_t
lib.cln_sigverify_events.restype = ctypes.c_short
invs = bolt11.invoices(bolt11.load_fixture())  # passed as char *: read up to a NUL, as the engine reads a span
out = {"blocking": [], "nodes": []}
for s in invs:
    node = (ctypes.c_uint8 * 33)(*([0xAA] * 33))
    out["blocking"].append(lib.bolt11_check_signature(s, node))
    out["nodes"].append(bytes(node).hex())
order = []
cb = DONE(lambda arg: order.append(arg))
st = (ctypes.c_int * len(invs))(*([99] * len(invs)))
nodes = (ctypes.c_uint8 * (33 * len(invs)))()
tickets = []
for i, s in enumerate(invs):
    tickets.append(lib.bolt11_check_signature_start(s, ctypes.addressof(st) + 4 * i, ctypes.addressof(nodes) + 33 * i, cb, i + 1))
    while lib.cln_sigverify_process() >= window:
        ev = lib.cln_sigverify_events()
        select.select([lib.cln_sigverify_fd()] if ev & 1 else [], [lib.cln_sigverify_fd()] if ev & 4 else [], [])
lib.cln_sigverify_drain()
out["tickets"] = tickets
out["order"] = order
out["async"] = list(st)
out["async_nodes"] = bytes(nodes).hex()
print(json.dumps(out))
"""


def _run_client(tmp_path, env, window=64):
    env = dict(env, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-c", CLIENT, str(window)], env=env, cwd=str(tmp_path), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def _same_as_ref(ref, out):
    n = len(ref[0])
    assert out["blocking"] == ref[0].tolist() and out["async"] == ref[0].tolist()
    assert out["nodes"] == [ref[1][i].tobytes().hex() for i in range(n)]
    assert out["async_nodes"] == ref[1].tobytes().hex()


def test_dropin_client_mode(fx, ref, daemon, tmp_path):
    """no visible GPU, CLN_SIGVERIFYD_SOCKET set: every fixture item through bolt11_check_signature, then again as a
    window of 64 tickets; both match the in-process answers, callbacks in ticket order, and the daemon counts every call"""
    env = dict(os.environ, CLN_SIGVERIFYD_SOCKET=daemon, CUDA_VISIBLE_DEVICES="")
    out = _run_client(tmp_path, env)
    _same_as_ref(ref, out)
    n = len(ref[0])
    assert out["order"] == list(range(1, n + 1))
    assert out["tickets"] == sorted(out["tickets"]) and min(out["tickets"]) > 0
    st = _stats(daemon)
    assert st["requests"] == 2 * n and st["signatures"] == 2 * n, st
    assert st["launches"] < st["requests"], st  # the window shared launches


def test_dropin_in_process(fx, ref, tmp_path):
    """no daemon: the drop-in's own context gives the same answers, and every _start returns 0 with its answer written"""
    env = dict(os.environ)
    env.pop("CLN_SIGVERIFYD_SOCKET", None)
    out = _run_client(tmp_path, env)
    _same_as_ref(ref, out)
    assert out["tickets"] == [0] * len(ref[0]) and out["order"] == []
