"""CPU: sigverifyd_bolt11 (bolt11_decode's signature step through the verifier subdaemon) and the drop-in's
bolt11_check_signature, built with gcc against the fake engine (tests/host_emul/fake_engine.c) and its BOLT11 check
(tests/host_emul/fake_engine_bolt11.c, linked beside it).  The fake answers every invoice with a hash of its bytes, so an
invoice routed to the wrong slot, or cut short, shows up as a wrong answer:
    status = FNV-1a(invoice bytes) % 3 - 1,  receiver_id = fill(h, 33) where the status is 1, zeros elsewhere.
Checked: replies of many clients in request order among other request types, one engine call per pass, call limits at
request boundaries, refusals, a daemon linked without the check, and the drop-in's blocking calls, tickets and in-process
mode."""
import json
import os
import resource
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_daemon
from tests import sigverifyd_fake as sf
from tests.sigverifyd_fake import FAKE_BOLT11, TAGS, bolt12_req, calls, fill, fnv, patched, roundtrip, short, verify_req

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_ITEMS = 1 << 20
SMALL = dict(CALL_ITEMS=8, HASH_CALL_BYTES=200)  # per-call limits of the small-limits daemon


def answer(s):
    """(status, receiver_id) the fake gives the invoice bytes s"""
    h = fnv(s)
    st = h % 3 - 1
    return st, fill(h, 33) if st == 1 else bytes(33)


def invoice(rng, size=None, nul=False):
    """printable invoice-like bytes, with a NUL somewhere inside when nul is set"""
    size = int(rng.integers(0, 400)) if size is None else size
    s = bytearray(rng.integers(33, 127, size=size, dtype=np.uint8).tobytes())
    if nul and size:
        s[int(rng.integers(0, size))] = 0
    return bytes(s)


def bolt11_req(rng, rid, strings):
    blob = b"".join(strings)
    ans = [answer(s) for s in strings]
    return (W.encode("sigverifyd_bolt11", req_id=rid, n=len(strings), lens=[len(s) for s in strings], bloblen=len(blob),
                     blob=blob),
            ("sigverifyd_bolt11_reply", dict(req_id=rid, n=len(strings), status=bytes(st & 0xFF for st, _ in ans),
                                             node_ids=b"".join(node for _, node in ans))))


def sized_req(rng, rid, sizes):
    return bolt11_req(rng, rid, [invoice(rng, s) for s in sizes])


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    """the daemon and the drop-in (client mode and in-process) on the fake engine with its BOLT11 check, a daemon with small
    call limits, and a daemon without the check"""
    d = tmp_path_factory.mktemp("fake_bolt11")
    return dict(daemon=sf.daemon(d / "cln_sigverifyd", FAKE_BOLT11), bare=sf.daemon(d / "cln_sigverifyd_bare"),
                small=sf.daemon(d / "cln_sigverifyd_small", FAKE_BOLT11, limits=SMALL),
                lib=sf.dropin(d / "libcln_dropin_fake.so", FAKE_BOLT11),
                inproc=sf.dropin(d / "libcln_dropin_inproc.so", FAKE_BOLT11, client=False))


@pytest.fixture
def fake(tmp_path, bins):
    """a daemon on the fake engine with its BOLT11 check, and the engine's call log"""
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        yield sock, tmp_path / "engine.log"


def test_clients_get_every_reply_in_order(fake):
    """8 clients x 30 requests: BOLT11 requests of 1-40 invoices (some with a NUL inside, some empty strings) mixed with
    sigverifyd_verify and sigverifyd_bolt12, in writes of 1-4 requests; every reply is the fake's, in request order"""
    sock, log = fake
    errors, invoices = [], [0] * 8

    def client(ci):
        try:
            rng = np.random.default_rng(200 + ci)
            reqs = []
            for j in range(30):
                rid = ci * 1000 + j
                if j % 5 == 3:
                    reqs.append(verify_req(rng, rid, int(rng.integers(0, 3)), int(rng.integers(1, 6))))
                elif j % 5 == 4:
                    reqs.append(bolt12_req(rng, rid, *TAGS[j % 3], [int(x) for x in rng.integers(0, 200, size=3)], j % 2))
                else:
                    k = int(rng.integers(1, 41))
                    reqs.append(bolt11_req(rng, rid, [invoice(rng, nul=rng.random() < 0.1) for _ in range(k)]))
                    invoices[ci] += k
            c = sigverifyd_daemon.connect(sock)
            j = 0
            while j < len(reqs):
                k = int(rng.integers(1, 5))
                roundtrip(c, reqs[j:j + k])
                j += k
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errors, errors
    assert sigverifyd_daemon.stats(sock)["requests"] == 240
    assert sum(c[2] for c in calls(log) if c[0] == "sv_verify_bolt11_host") == sum(invoices)


def test_one_write_is_one_pass(fake):
    """BOLT11 requests written at once among other types: ONE sv_verify_bolt11_host call with every invoice of the pass,
    after the verify and BOLT12 calls; each invoice counts as one signature"""
    sock, log = fake
    rng = np.random.default_rng(7)
    reqs = [sized_req(rng, 1, [30, 0, 7]), verify_req(rng, 2, 0, 2), sized_req(rng, 3, [100]),
            bolt12_req(rng, 4, *TAGS[0], [12], 0), sized_req(rng, 5, []), sized_req(rng, 6, [5, 5, 5, 5])]
    c = sigverifyd_daemon.connect(sock)
    roundtrip(c, reqs)
    c.close()
    assert calls(log) == [("sv_verify_host", 0, 2, 0), ("sv_verify_bolt12_tagged_host", 0, 1, 12),
                           ("sv_verify_bolt11_host", 0, 8, 157)]
    st = sigverifyd_daemon.stats(sock)
    assert st["requests"] == 6 and st["launches"] == 3 and st["signatures"] == 2 + 1 + 8 and st["max_coalesced"] == 4, st


def test_call_limits_split_at_request_boundaries(tmp_path, bins):
    """with small per-call limits (8 invoices, 200 bytes), a pass is cut into sv_verify_bolt11_host calls at request
    boundaries, by invoices and by bytes, a request above a limit alone; every reply is still the fake's"""
    log = tmp_path / "engine.log"
    rng = np.random.default_rng(13)
    with sigverifyd_daemon.running(tmp_path, bins["small"], sf.env(tmp_path)) as sock:
        c = sigverifyd_daemon.connect(sock)
        roundtrip(c, [sized_req(rng, 1, [10, 10, 10]), sized_req(rng, 2, [10] * 4),  # 7 invoices, 70 bytes
                       sized_req(rng, 3, [50] * 3),                                  # 10 invoices > 8: a new call
                       sized_req(rng, 4, [60]),                                      # 150 + 60 bytes > 200: a new call
                       sized_req(rng, 5, []),
                       sized_req(rng, 6, [1] * 9),                                   # 9 invoices > 8: alone
                       sized_req(rng, 7, [250]),                                     # 250 bytes > 200: alone
                       sized_req(rng, 8, [3, 3])])
        c.close()
    assert calls(log) == [("sv_verify_bolt11_host", 0, 7, 70), ("sv_verify_bolt11_host", 0, 3, 150),
                           ("sv_verify_bolt11_host", 0, 1, 60), ("sv_verify_bolt11_host", 0, 9, 9),
                           ("sv_verify_bolt11_host", 0, 1, 250), ("sv_verify_bolt11_host", 0, 2, 6)]


def test_malformed_requests_are_refused(fake):
    """spans that do not add up (short and wrapping past 2^32), a truncated frame and n above MAX_ITEMS: each answered
    with sigverifyd_error code 1 and nothing reaches the engine; the same connection then serves a good request"""
    sock, log = fake
    rng = np.random.default_rng(3)
    c = sigverifyd_daemon.connect(sock)
    frame, want = sized_req(rng, 9, [40, 60])
    big_n = W.encode("sigverifyd_bolt11", req_id=12, n=MAX_ITEMS + 1, lens=bytes(4 * (MAX_ITEMS + 1)), bloblen=0, blob=b"")
    bad = [(patched(frame, 14, (41).to_bytes(4, "big")), 9),                  # 41 + 60 != 100
           (patched(frame, 14, (0xFFFFFFFF).to_bytes(4, "big")), 9),          # the 32-bit sum wraps to 59
           (short(frame), 9),
           (big_n, 12)]
    for b, rid in bad:
        c.sendall(b)
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=rid, code=1))
    assert calls(log) == []
    roundtrip(c, [(frame, want)])
    c.close()
    assert calls(log) == [("sv_verify_bolt11_host", 0, 2, 100)]
    assert sigverifyd_daemon.stats(sock)["requests"] == 1


def test_engine_without_bolt11_refuses(tmp_path, bins):
    """a daemon linked against an engine without sv_verify_bolt11_host answers a BOLT11 request with error 1 and keeps
    serving"""
    rng = np.random.default_rng(5)
    log = tmp_path / "engine.log"
    with sigverifyd_daemon.running(tmp_path, bins["bare"], sf.env(tmp_path)) as sock:
        c = sigverifyd_daemon.connect(sock)
        c.sendall(sized_req(rng, 11, [80])[0])
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=11, code=1))
        roundtrip(c, [verify_req(rng, 12, 0, 2)])
        c.close()
    assert [x[0] for x in calls(log)] == ["sv_verify_host"]


# the drop-in: python -c CLIENT <library> <invoices.json> [window]; prints the answers of the blocking calls and, with a
# window, of the same invoices as tickets kept that many in flight, with the callbacks' order
CLIENT = r"""
import ctypes, json, select, sys
lib = ctypes.CDLL(sys.argv[1])
strings = [bytes.fromhex(s) for s in json.load(open(sys.argv[2]))]
window = int(sys.argv[3]) if len(sys.argv) > 3 else 0
DONE = ctypes.CFUNCTYPE(None, ctypes.c_void_p)
vp = ctypes.c_void_p
lib.bolt11_check_signature.restype = ctypes.c_int
lib.bolt11_check_signature.argtypes = [ctypes.c_char_p, vp]
lib.bolt11_check_signature_start.restype = ctypes.c_uint64
lib.bolt11_check_signature_start.argtypes = [ctypes.c_char_p, vp, vp, DONE, vp]
lib.cln_sigverify_process.restype = ctypes.c_size_t
lib.cln_sigverify_events.restype = ctypes.c_short
out = {"blocking": []}
for s in strings:
    node = (ctypes.c_uint8 * 33)(*([0xAA] * 33))
    st = lib.bolt11_check_signature(s, node)
    out["blocking"].append([st, bytes(node).hex()])
if window:
    order = []
    cb = DONE(lambda arg: order.append(arg))
    st = (ctypes.c_int * len(strings))(*([99] * len(strings)))
    nodes = (ctypes.c_uint8 * (33 * len(strings)))(*([0xAA] * (33 * len(strings))))
    tickets = []
    for i, s in enumerate(strings):
        tickets.append(lib.bolt11_check_signature_start(s, ctypes.addressof(st) + 4 * i, ctypes.addressof(nodes) + 33 * i,
                                                        cb, i + 1))
        while lib.cln_sigverify_process() >= window:  # keep at most `window` tickets in flight
            ev = lib.cln_sigverify_events()
            select.select([lib.cln_sigverify_fd()] if ev & 1 else [], [lib.cln_sigverify_fd()] if ev & 4 else [], [])
    lib.cln_sigverify_drain()
    out["tickets"] = tickets
    out["order"] = order
    out["async"] = [[st[i], bytes(nodes[33 * i:33 * i + 33]).hex()] for i in range(len(strings))]
print(json.dumps(out))
"""


def _env(**kw):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.pop("CLN_SIGVERIFYD_SOCKET", None)
    env.update(kw)
    return env


def _client(tmp_path, lib, strings, window=0, env=None):
    path = tmp_path / "invoices.json"
    path.write_text(json.dumps([s.hex() for s in strings]))
    args = [sys.executable, "-c", CLIENT, lib, str(path)] + ([str(window)] if window else [])
    r = subprocess.run(args, env=env or _env(), cwd=str(tmp_path), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout)


def _strings(rng, n):
    """C strings as bolt11_decode receives them (no NUL inside), the empty one among them"""
    return [b""] + [invoice(rng).replace(b"\0", b"q") for _ in range(n - 1)]


def test_dropin_client_mode(tmp_path, bins):
    """bolt11_check_signature in client mode: one request per call with the string's bytes up to its NUL, the fake's
    answer, *receiver_id zeroed unless 1; then the same strings as a window of 64 tickets: the same answers, callbacks in
    ticket order; the library never reaches sv_create (the fake's aborts), and the daemon counts every call"""
    rng = np.random.default_rng(21)
    strings = _strings(rng, 300)
    want = [[st, node.hex()] for st, node in map(answer, strings)]
    log = tmp_path / "engine.log"
    with sigverifyd_daemon.running(tmp_path, bins["daemon"], sf.env(tmp_path)) as sock:
        out = _client(tmp_path, bins["lib"], strings, window=64, env=_env(CLN_SIGVERIFYD_SOCKET=sock))
        st = sigverifyd_daemon.stats(sock)
    assert out["blocking"] == want and out["async"] == want
    assert {w[0] for w in want} == {-1, 0, 1}
    assert out["order"] == list(range(1, 301))
    assert out["tickets"] == sorted(out["tickets"]) and len(set(out["tickets"])) == 300 and min(out["tickets"]) > 0
    assert st["requests"] == 600 and st["signatures"] == 600, st
    b11 = [c for c in calls(log) if c[0] == "sv_verify_bolt11_host"]
    assert sum(c[2] for c in b11) == 600 and len(b11) < 600  # the window shared engine calls


def test_dropin_reply_with_bad_status_aborts(tmp_path, bins):
    """a reply whose status byte is not 0, 1 or 255 aborts the client rather than be read as an answer"""
    script = r"""
import ctypes, socket, sys
from lightning_b200 import sigverifyd_wire as W
lib = ctypes.CDLL(sys.argv[1])
a, b = socket.socketpair()
assert lib.cln_sigverify_connect_fd(a.detach()) == 0
DONE = ctypes.CFUNCTYPE(None, ctypes.c_void_p)
lib.bolt11_check_signature_start.restype = ctypes.c_uint64
lib.bolt11_check_signature_start.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p, DONE, ctypes.c_void_p]
st, node = ctypes.c_int(), (ctypes.c_uint8 * 33)()
t = lib.bolt11_check_signature_start(b"lnbc1", ctypes.byref(st), node, DONE(0), None)
name, req = W.read_msg(b)
assert name == "sigverifyd_bolt11" and req["req_id"] == t and req["n"] == 1 and req["blob"] == b"lnbc1"
b.sendall(W.encode("sigverifyd_bolt11_reply", req_id=t, n=1, status=b"\x02", node_ids=bytes(33)))
lib.cln_sigverify_drain()
print("drained", flush=True)
"""
    r = subprocess.run([sys.executable, "-c", script, bins["lib"]], env=_env(), cwd=str(tmp_path), capture_output=True,
                       text=True, timeout=120, preexec_fn=lambda: resource.setrlimit(resource.RLIMIT_CORE, (0, 0)))
    assert r.returncode < 0 and "malformed bolt11 reply" in r.stderr and "drained" not in r.stdout, (r.returncode, r.stderr)


def test_dropin_in_process_mode(tmp_path, bins):
    """no daemon: the fake engine linked in; every _start returns 0 with the blocking call's answer already written"""
    rng = np.random.default_rng(22)
    strings = _strings(rng, 40)
    want = [[st, node.hex()] for st, node in map(answer, strings)]
    out = _client(tmp_path, bins["inproc"], strings, window=64)
    assert out["blocking"] == want and out["async"] == want
    assert out["tickets"] == [0] * 40 and out["order"] == []
