"""CPU: the verifier subdaemon (sigverifyd.c) and the drop-in's client mode (cln_dropin.c), both built with gcc against a
fake engine (tests/host_emul/fake_engine.c) whose every result is a hash of its item's bytes.  Checked: every reply
of several clients in request order, how a pass is split into engine calls (the fake's call log), refusals, the
sigverifyd_stats counters, call limits at request boundaries, and every client-mode drop-in function.  The daemon and the
drop-in only route bytes, so a request sent to the wrong slot, tag or key kind shows up as a wrong hash."""
import ctypes
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from lightning_b200 import build
from lightning_b200 import sigverifyd_wire as W
from tests import sigverifyd_daemon, txsig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = os.path.join(ROOT, "tests", "host_emul", "fake_engine.c")
KS = {0: 33, 1: 64, 2: 32}
MAX_FRAME = 32 + (1 << 20) * 161
SMALL = dict(CALL_ITEMS=8, HASH_CALL_BYTES=200, TX_CALL_BYTES=600)  # per-call limits of the small-limits daemon
TESTNET = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


# ---- the fake engine's functions (fake_engine.c) -----------------------------------------------------------------------
def fnv(data, h=0xcbf29ce484222325):
    for b in data:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h


def fill(h, n):
    return bytes(fnv(bytes([k]), h) & 0xFF for k in range(n))


def wire(status):
    return bytes(s & 0xFF for s in status)


def le(v, n):
    return int(v).to_bytes(n, "little")


def tx_hash(kind, key, sig, f, spans):
    """f: version, locktime, sequence, sighash_type, prev_txid, prev_index, flags, input_amount, output_amount"""
    return fnv(bytes([kind]) + key + sig + b"".join(le(f[k], 4) for k in ("version", "locktime", "sequence", "sighash_type")) +
               f["prev_txid"] + le(f["prev_index"], 4) + le(f["flags"], 4) + le(f["input_amount"], 8) +
               le(f["output_amount"], 8) + b"".join(le(len(s), 4) + s for s in spans))


# ---- requests and the replies the fake dictates ---------------------------------------------------------------------
def _rand(rng, n):
    return rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()


def verify_req(rng, rid, kind, n):
    h, k, s = _rand(rng, 32 * n), _rand(rng, KS[kind] * n), _rand(rng, 64 * n)
    ks = KS[kind]
    v = bytes(fnv(bytes([kind]) + h[32 * i:32 * i + 32] + k[ks * i:ks * i + ks] + s[64 * i:64 * i + 64]) % 3 for i in range(n))
    return (W.encode("sigverifyd_verify", req_id=rid, kind=kind, n=n, hashes=h, keylen=ks * n, keys=k, sigs=s),
            ("sigverifyd_verify_reply", dict(req_id=rid, n=n, verdicts=v)))


def bolt12_req(rng, rid, mn, fn, sizes, want):
    n = len(sizes)
    streams = [_rand(rng, x) for x in sizes]
    xo, sg = _rand(rng, 32 * n), _rand(rng, 64 * n)
    hs = [fnv(mn + b"\0" + fn + b"\0" + streams[i] + xo[32 * i:32 * i + 32] + sg[64 * i:64 * i + 64]) for i in range(n)]
    blob = b"".join(streams)
    frame = W.encode("sigverifyd_bolt12", req_id=rid, mnlen=len(mn), messagename=mn, fnlen=len(fn), fieldname=fn, n=n,
                     lens=sizes, bloblen=len(blob), blob=blob, xonly=xo, sigs=sg, want_sighash=want)
    return frame, ("sigverifyd_bolt12_reply", dict(req_id=rid, n=n, status=wire(h % 3 - 1 for h in hs),
                                                   nsighash=n if want else 0,
                                                   sighashes=b"".join(fill(h, 32) for h in hs) if want else b""))


def tx_req(rng, rid, kind, spans, want):
    """spans: per transaction the lengths of (script, outputs, outpoints, sequences)"""
    n = len(spans)
    key, sigs = _rand(rng, KS[kind]), _rand(rng, 64 * n)
    recs, data, hs = [], [], []
    for i, sp in enumerate(spans):
        f = dict(version=int(rng.integers(1, 3)), locktime=int(rng.integers(0, 2**32)), sequence=int(rng.integers(0, 2**32)),
                 sighash_type=int(rng.choice([1, 3, 0x83])), prev_txid=_rand(rng, 32), prev_index=int(rng.integers(0, 9)),
                 flags=1 | (2 if sp[2] or sp[3] else 0), input_amount=int(rng.integers(0, 2**62)),
                 output_amount=int(rng.integers(0, 2**62)))
        b = [_rand(rng, x) for x in sp]
        recs.append(f)
        data += b
        hs.append(tx_hash(kind, key, sigs[64 * i:64 * i + 64], f, b))
    kw = {k: [r[k] for r in recs] for k in txsig.U32_FIELDS}
    blob = b"".join(data)
    frame = W.encode("sigverifyd_tx", req_id=rid, kind=kind, keylen=len(key), key=key, n=n,
                     prev_txid=b"".join(r["prev_txid"] for r in recs), input_amount=[r["input_amount"] for r in recs],
                     output_amount=[r["output_amount"] for r in recs], script_len=[s[0] for s in spans],
                     outputs_len=[s[1] for s in spans], prevouts_len=[s[2] for s in spans],
                     sequences_len=[s[3] for s in spans], bloblen=len(blob), blob=blob, sigs=sigs, want_sighash=want, **kw)
    return frame, ("sigverifyd_tx_reply", dict(req_id=rid, n=n, verdicts=bytes(h % 3 for h in hs), nsighash=n if want else 0,
                                               sighashes=b"".join(fill(h, 32) for h in hs) if want else b""))


def sha_req(rng, rid, sizes):
    bufs = [_rand(rng, x) for x in sizes]
    blob = b"".join(bufs)
    return (W.encode("sigverifyd_sha256d", req_id=rid, n=len(bufs), lens=sizes, bloblen=len(blob), blob=blob),
            ("sigverifyd_sha256d_reply", dict(req_id=rid, n=len(bufs), hashes=b"".join(fill(fnv(b), 32) for b in bufs))))


def key_req(rng, rid, n):
    keys = _rand(rng, 33 * n)
    hs = [fnv(keys[33 * i:33 * i + 33]) for i in range(n)]
    return (W.encode("sigverifyd_pubkey", req_id=rid, n=n, keys=keys),
            ("sigverifyd_pubkey_reply", dict(req_id=rid, n=n, ok=bytes(h % 3 for h in hs),
                                             xy=b"".join(fill(h, 64) for h in hs))))


def gossip_req(rng, rid, n):
    msgs = [_rand(rng, int(rng.integers(2, 300))) for _ in range(n)]
    sg = _rand(rng, 33 * n)
    st = [fnv(m + sg[33 * i:33 * i + 33]) % 6 - 1 for i, m in enumerate(msgs)]
    blob = b"".join(msgs)
    return (W.encode("sigverifyd_gossip", req_id=rid, n=n, lens=[len(m) for m in msgs], signers=sg, bloblen=len(blob),
                     blob=blob), ("sigverifyd_gossip_reply", dict(req_id=rid, n=n, status=wire(st))))


def burst_req(rng, rid, n):
    msgs = [_rand(rng, int(rng.integers(2, 300))) for _ in range(n)]
    kinds, sg = bytes(int(x) for x in rng.integers(0, 3, size=n)), _rand(rng, 33 * n)
    st = [fnv(TESTNET + m + kinds[i:i + 1] + sg[33 * i:33 * i + 33]) % 10 - 4 for i, m in enumerate(msgs)]
    blob = b"".join(msgs)
    return (W.encode("sigverifyd_gossip_burst", req_id=rid, chain_hash=TESTNET, n=n, lens=[len(m) for m in msgs],
                     signer_kind=kinds, signers=sg, bloblen=len(blob), blob=blob),
            ("sigverifyd_gossip_burst_reply", dict(req_id=rid, n=n, status=wire(st))))


TAGS = [(b"invoice", b"signature"), (b"invoice_request", b"signature"), (b"offer", b"signature")]


def any_req(rng, rid):
    """a request of a random type"""
    t = int(rng.integers(0, 8))
    n = int(rng.integers(0, 6)) if rng.random() < 0.1 else int(rng.integers(1, 6))
    if t == 0:
        return verify_req(rng, rid, int(rng.integers(0, 3)), n)
    if t == 1:
        mn, fn = TAGS[int(rng.integers(0, 3))]
        return bolt12_req(rng, rid, mn, fn, [int(x) for x in rng.integers(0, 200, size=n)], int(rng.integers(0, 2)))
    if t == 2:
        sp = [(int(rng.integers(0, 150)), int(rng.integers(0, 100)), 36 * k, 4 * k) for k in rng.integers(0, 3, size=n)]
        return tx_req(rng, rid, int(rng.integers(0, 2)), sp, int(rng.integers(0, 2)))
    if t == 3:
        return sha_req(rng, rid, [int(x) for x in rng.choice([0, 1, 55, 64, 120, 500], size=n)])
    if t == 4:
        return key_req(rng, rid, n)
    if t == 5:
        return gossip_req(rng, rid, n)
    if t == 6:
        return burst_req(rng, rid, n)
    return W.encode("sigverifyd_stats", req_id=rid), None


def patched(frame, at, value):
    """frame with the bytes at offset `at` of its message replaced"""
    body = bytearray(frame[4:])
    body[at:at + len(value)] = value
    return len(body).to_bytes(4, "big") + bytes(body)


def short(frame):
    """frame one byte short of its fields"""
    body = frame[4:-1]
    return len(body).to_bytes(4, "big") + body


# ---- builds and daemons ---------------------------------------------------------------------------------------------
def _gcc(args):
    r = subprocess.run(["gcc"] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.fixture(scope="module")
def bins(tmp_path_factory):
    d = tmp_path_factory.mktemp("fake_engine")
    out = dict(daemon=str(d / "cln_sigverifyd"), lib=str(d / "libcln_dropin_fake.so"))
    _gcc(build.DAEMON_CFLAGS + [os.path.join(build.CSRC, "sigverifyd.c"), FAKE, "-o", out["daemon"]])
    _gcc(build.DROPIN_CFLAGS + ["-shared", "-DFAKE_ENGINE_NO_CONTEXT", os.path.join(build.CSRC, "cln_dropin.c"), FAKE,
                                "-o", out["lib"]])
    return out


def _start(tmp_path, binary):
    log = tmp_path / "engine.log"
    return sigverifyd_daemon.running(tmp_path, binary, env=dict(os.environ, FAKE_ENGINE_LOG=str(log))), log


@pytest.fixture
def fake(tmp_path, bins):
    """a daemon on the fake engine, and the engine's call log"""
    ctx, log = _start(tmp_path, bins["daemon"])
    with ctx as sock:
        yield sock, log


def _calls(log):
    if not log.exists():
        return []
    return [(f, int(k), int(n), int(b)) for f, k, n, b in (line.split() for line in log.read_text().splitlines())]


def _roundtrip(c, reqs):
    """sends the frames in one write, reads one reply per frame and checks each against what the fake dictates"""
    c.sendall(b"".join(f for f, _ in reqs))
    for frame, want in reqs:
        got = W.read_msg(c)
        if want is None:  # a stats request: its counters are checked elsewhere
            assert got[0] == "sigverifyd_stats_reply" and got[1]["req_id"] == W.decode(frame[4:])[1]["req_id"]
        else:
            assert got == want, (got[0], got[1].get("req_id"), want[0], want[1]["req_id"])


# ---- (a)-(e): the daemon ----------------------------------------------------------------------------------------------
def test_clients_get_every_reply_in_order(fake):
    """6 clients send 40 requests of every type each, in writes of 1-4 requests: every per-item result is the fake's,
    and each client's replies come back in its request order"""
    sock, _ = fake
    errors = []

    def client(ci):
        try:
            rng = np.random.default_rng(100 + ci)
            c = sigverifyd_daemon.connect(sock)
            reqs = [any_req(rng, ci * 1000 + j) for j in range(40)]
            j = 0
            while j < len(reqs):
                k = int(rng.integers(1, 5))
                _roundtrip(c, reqs[j:j + k])
                j += k
            c.close()
        except Exception as ex:  # noqa: BLE001
            errors.append((ci, repr(ex)))

    th = [threading.Thread(target=client, args=(i,)) for i in range(6)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errors, errors


def test_one_write_is_one_pass(fake):
    """batched requests written at once are served in one pass: one engine call per type and group, in the pass order
    (verify kinds 0, 1, 2; BOLT12 over all tags; tx kinds 0, 1; sha256d; pubkey), with the summed items and bytes"""
    sock, log = fake
    rng = np.random.default_rng(7)
    reqs = [tx_req(rng, 1, 1, [(10, 20, 0, 0), (5, 9, 72, 8)], 1), verify_req(rng, 2, 2, 3), key_req(rng, 3, 2),
            verify_req(rng, 4, 0, 2), bolt12_req(rng, 5, *TAGS[0], [40, 0], 1), sha_req(rng, 6, [3, 0, 64]),
            verify_req(rng, 7, 0, 1), tx_req(rng, 8, 0, [(30, 0, 0, 0)], 0), bolt12_req(rng, 9, *TAGS[1], [12], 0),
            verify_req(rng, 10, 1, 4), sha_req(rng, 11, [5]), key_req(rng, 12, 3), tx_req(rng, 13, 1, [(7, 7, 0, 0)], 0)]
    c = sigverifyd_daemon.connect(sock)
    _roundtrip(c, reqs)
    c.close()
    assert _calls(log) == [("sv_verify_host", 0, 3, 0), ("sv_verify_host", 1, 4, 0), ("sv_verify_host", 2, 3, 0),
                           ("sv_verify_bolt12_tagged_host", 0, 3, 52), ("sv_verify_tx_host", 0, 1, 30),
                           ("sv_verify_tx_host", 1, 3, 10 + 20 + 5 + 9 + 72 + 8 + 14), ("sv_sha256d_host", 0, 4, 72),
                           ("sv_pubkey_parse_host", 0, 5, 0)]


def test_refusals(fake):
    """malformed requests get error code 1 and unknown types code 3, and the connection keeps serving; a length prefix
    above MAX_FRAME (or below 2) closes it"""
    sock, log = fake
    rng = np.random.default_rng(3)
    c = sigverifyd_daemon.connect(sock)

    def refused(frame, code=1, rid=None):
        c.sendall(frame)
        rid = W.decode(frame[4:])[1]["req_id"] if rid is None else rid
        assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=rid, code=code))

    refused(patched(verify_req(rng, 21, 0, 2)[0], 10, b"\x03"))                          # no such key kind
    v = verify_req(rng, 22, 1, 2)[0]
    refused(patched(v, 2 + 8 + 1 + 4 + 64, (127).to_bytes(4, "big")), rid=22)            # keylen that does not parse
    refused(short(v), rid=22)
    refused(bolt12_req(rng, 23, b"", b"signature", [5], 0)[0])                            # empty tag
    refused(bolt12_req(rng, 24, b"inv\0ice", b"signature", [5], 0)[0])                    # NUL in a tag
    b = bolt12_req(rng, 25, *TAGS[0], [5, 6], 0)[0]
    refused(patched(b, 2 + 8 + 2 + 7 + 2 + 9 + 4, (6).to_bytes(4, "big")))                # spans that do not add up
    t = tx_req(rng, 26, 0, [(5, 5, 0, 0)], 0)[0]
    refused(patched(t, 10, b"\x02"))                                                      # not an ECDSA kind
    flags_at = 2 + 8 + 1 + 4 + 33 + 4 + 5 * 4
    refused(patched(t, flags_at, (8).to_bytes(4, "big")))                                # unknown flag bit
    refused(patched(tx_req(rng, 27, 0, [(5, 5, 36, 4)], 0)[0], flags_at, (1).to_bytes(4, "big")))  # outpoints, no flag
    s = sha_req(rng, 28, [3, 4])[0]
    refused(patched(s, 2 + 8 + 4, (4).to_bytes(4, "big")))                                # spans that do not add up
    refused(short(key_req(rng, 29, 2)[0]), rid=29)
    g = gossip_req(rng, 30, 2)[0]
    refused(patched(g, 2 + 8 + 4, (0xFFFFFFFF).to_bytes(4, "big")))                       # spans that do not add up
    u = burst_req(rng, 31, 2)[0]
    refused(patched(u, 2 + 8 + 32 + 4 + 8 + 1, b"\x03"))                                  # signer kind 3
    refused(short(u), rid=31)
    refused((2).to_bytes(4, "big") + (3003).to_bytes(2, "big"), rid=0)                     # a stats request without its id
    refused((10).to_bytes(4, "big") + (3050).to_bytes(2, "big") + (99).to_bytes(8, "big"), code=3, rid=0)
    good = [sha_req(rng, 40, [1]), burst_req(rng, 41, 1)]
    _roundtrip(c, good)
    assert not any(f == "sv_verify_host" for f, *_ in _calls(log))  # nothing refused reached the engine
    c.sendall((MAX_FRAME + 1).to_bytes(4, "big"))
    c.settimeout(20)
    try:
        assert c.recv(1) == b""
    except ConnectionResetError:
        pass
    c.close()
    c = sigverifyd_daemon.connect(sock)
    c.sendall((1).to_bytes(4, "big") + b"\0")
    try:
        assert c.recv(1) == b""
    except ConnectionResetError:
        pass
    c.close()


def test_stats_counters(fake):
    """requests, launches, signatures and the largest coalesced launch after a fixed sequence"""
    sock, _ = fake
    rng = np.random.default_rng(11)
    c = sigverifyd_daemon.connect(sock)
    # one pass: verify kind 0 (2 requests, 5 signatures) and kind 2 (1), tx kind 1 (2 requests, 3), sha256d (1), pubkey (1)
    _roundtrip(c, [verify_req(rng, 1, 0, 3), verify_req(rng, 2, 0, 2), verify_req(rng, 3, 2, 1),
                   tx_req(rng, 4, 1, [(4, 4, 0, 0)], 0), tx_req(rng, 5, 1, [(4, 4, 0, 0), (1, 1, 0, 0)], 1),
                   sha_req(rng, 6, [5, 6]), key_req(rng, 7, 4)])
    _roundtrip(c, [gossip_req(rng, 8, 3)])                 # one launch of its own
    _roundtrip(c, [burst_req(rng, 9, 2)])                  # likewise
    _roundtrip(c, [verify_req(rng, 10, 1, 0)])             # an empty request still counts as a launch
    c.sendall(short(key_req(rng, 11, 1)[0]))              # refused: not counted
    assert W.read_msg(c) == ("sigverifyd_error", dict(req_id=11, code=1))
    st = sigverifyd_daemon.stats(sock)
    assert st == dict(req_id=77, requests=7 + 1 + 1 + 1, launches=5 + 1 + 1 + 1, signatures=6 + 3 + 3 + 2 + 0,
                      max_coalesced=2), st
    c.close()


def test_call_limits_split_at_request_boundaries(tmp_path):
    """with small per-call limits (SMALL), a pass is cut into engine calls at request boundaries: sha256d by items and by
    bytes, pubkey by items, tx by span bytes, a request above a limit alone; every reply is still the fake's"""
    d = str(tmp_path / "cln_sigverifyd_small")
    _gcc(build.DAEMON_CFLAGS + ["-D%s=%d" % kv for kv in SMALL.items()] + [os.path.join(build.CSRC, "sigverifyd.c"), FAKE,
                                                                           "-o", d])
    ctx, log = _start(tmp_path, d)
    rng = np.random.default_rng(13)
    with ctx as sock:
        c = sigverifyd_daemon.connect(sock)
        _roundtrip(c, [sha_req(rng, 1, [10, 10, 10]), sha_req(rng, 2, [10] * 4),    # 7 items, 70 bytes
                       sha_req(rng, 3, [50] * 3),                                   # 10 items > 8: a new call
                       sha_req(rng, 4, [60]),                                       # 150 + 60 bytes > 200: a new call
                       sha_req(rng, 5, []),
                       key_req(rng, 6, 5), key_req(rng, 7, 3), key_req(rng, 8, 2),  # 8 keys, then 2
                       tx_req(rng, 9, 1, [(100, 50, 0, 0), (60, 40, 0, 0)], 1),     # 250 bytes
                       tx_req(rng, 10, 1, [(200, 100, 0, 0)], 0),                   # 550
                       tx_req(rng, 11, 1, [(50, 50, 0, 0)], 0),                     # 650 > 600: a new call
                       tx_req(rng, 12, 1, [(300, 300, 72, 28)], 1)])                # 700 bytes alone
        c.close()
    assert _calls(log) == [("sv_verify_tx_host", 1, 3, 550), ("sv_verify_tx_host", 1, 1, 100),
                           ("sv_verify_tx_host", 1, 1, 700), ("sv_sha256d_host", 0, 7, 70), ("sv_sha256d_host", 0, 3, 150),
                           ("sv_sha256d_host", 0, 1, 60), ("sv_pubkey_parse_host", 0, 8, 0), ("sv_pubkey_parse_host", 0, 2, 0)]


# ---- (f): the drop-in library in client mode -------------------------------------------------------------------------
CLIENT = r"""
import ctypes, json, sys
from tests.txsig import WallyIn, WallyOut, WallyTx, BitcoinTx
lib = ctypes.CDLL(sys.argv[2])
vp, sz = ctypes.c_void_p, ctypes.c_size_t
for f in ("pubkey_from_der", "check_signed_hash", "check_signed_hash_nodeid", "check_schnorr_sig", "check_tx_sig",
          "bolt12_check_signature"):
    getattr(lib, f).restype = ctypes.c_bool
lib.pubkey_from_der.argtypes = [vp, sz, vp]
for f in ("check_signed_hash", "check_signed_hash_nodeid", "check_schnorr_sig"):
    getattr(lib, f).argtypes = [vp, vp, vp]
lib.sha256_double.argtypes = [vp, vp, sz]
lib.check_tx_sig.argtypes = [vp, sz, vp, vp, vp, vp]
lib.check_tx_sigs_batch.argtypes = [vp, vp, vp, sz, vp]
lib.check_tx_sigs_bip143_batch.argtypes = [vp, vp, sz, vp, vp, sz, vp]
lib.bolt12_check_signature.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p, vp, vp]
for f in ("sigcheck_channel_announcement_batch", "sigcheck_node_announcement_batch"):
    getattr(lib, f).argtypes = [vp, vp, sz, vp]
lib.sigcheck_channel_update_batch.argtypes = [vp, vp, vp, sz, vp]
lib.sigcheck_gossip_batch.argtypes = [vp, vp, vp, sz, vp, vp, vp]
lib.cln_sigverify_set_tx_hooks.argtypes = [vp, vp]
keep, sizes = [], {}
bytelen = ctypes.CFUNCTYPE(sz, vp)(lambda p: sizes[p])
amount = ctypes.CFUNCTYPE(ctypes.c_uint64, vp, sz)(lambda tx, i: sizes[tx])
lib.cln_sigverify_set_tx_hooks(ctypes.cast(bytelen, vp), ctypes.cast(amount, vp))
def buf(b):
    x = (ctypes.c_uint8 * max(len(b), 1)).from_buffer_copy(b or b"\0")
    keep.append(x)
    return ctypes.addressof(x)
H = bytes.fromhex
sc = json.load(open(sys.argv[1]))
out = {}
out["der"] = []
for k in sc["der"]:
    pk = (ctypes.c_uint8 * 64)()
    out["der"].append(bytes(pk).hex() if lib.pubkey_from_der(buf(H(k)), len(H(k)), pk) else None)
out["sha"] = []
for d in sc["sha"]:
    h = (ctypes.c_uint8 * 32)()
    lib.sha256_double(h, buf(H(d)), len(H(d)))
    out["sha"].append(bytes(h).hex())
out["signed"] = [lib.check_signed_hash(buf(H(h)), buf(H(s)), buf(H(k))) for h, s, k in sc["signed"]]
out["nodeid"] = [lib.check_signed_hash_nodeid(buf(H(h)), buf(H(s)), buf(H(k))) for h, s, k in sc["nodeid"]]
out["schnorr"] = [lib.check_schnorr_sig(buf(H(h)), buf(H(k)), buf(H(s))) for h, s, k in sc["schnorr"]]
out["batch"] = []
for h, s, k, n in sc["batch"]:
    ok = (ctypes.c_bool * n)()
    lib.check_tx_sigs_batch(buf(H(h)), buf(H(s)), buf(H(k)), n, ok)
    out["batch"].append(list(ok))
out["tx"] = []
for c in sc["tx"]:
    ins = (WallyIn * len(c["ins"]))()
    for j, (txid, idx, seq) in enumerate(c["ins"]):
        ins[j].txhash[:] = list(H(txid)); ins[j].index = idx; ins[j].sequence = seq
    outs = (WallyOut * len(c["outs"]))()
    for j, (sat, script) in enumerate(c["outs"]):
        outs[j].satoshi = sat; outs[j].script = buf(H(script)) if script else None; outs[j].script_len = len(H(script))
    w = WallyTx(c["version"], c["locktime"], ctypes.addressof(ins), len(ins), len(ins), ctypes.addressof(outs), len(outs), len(outs))
    tx = BitcoinTx(ctypes.pointer(w), None, None)
    keep.extend([ins, outs, w, tx])
    sizes[ctypes.addressof(tx)] = c["amount"]
    script = buf(H(c["script"]))
    sizes[script] = len(H(c["script"]))
    args = (None, script) if c["witness"] else (script, None)
    out["tx"].append(lib.check_tx_sig(ctypes.addressof(tx), c["input"], args[0], args[1], buf(H(c["key"])), buf(H(c["sig"]))))
out["bip143"] = []
for recs, blob, k, sigs, n in sc["bip143"]:
    ok = (ctypes.c_bool * n)()
    lib.check_tx_sigs_bip143_batch(buf(H(recs)), buf(H(blob)), len(H(blob)), buf(H(k)), buf(H(sigs)), n, ok)
    out["bip143"].append(list(ok))
out["bolt12"] = []
for fields, mn, fn, k, s in sc["bolt12"]:
    arr = (ctypes.c_uint64 * (4 * len(fields)))()
    for j, (t, v) in enumerate(fields):
        arr[4 * j + 1], arr[4 * j + 2], arr[4 * j + 3] = t, len(H(v)), buf(H(v)) if v else 0
    keep.append(arr)
    sizes[ctypes.addressof(arr)] = ctypes.sizeof(arr)
    out["bolt12"].append(lib.bolt12_check_signature(ctypes.addressof(arr), mn.encode(), fn.encode(), buf(H(k)), buf(H(s))))
def msgs_args(msgs):
    bufs = [buf(H(m)) for m in msgs]
    return buf(b"".join(b.to_bytes(8, "little") for b in bufs)), buf(b"".join(len(H(m)).to_bytes(8, "little") for m in msgs))
out["gossip"] = []
for fn, msgs, signers in sc["gossip"]:
    st = (ctypes.c_int * len(msgs))()
    p, l = msgs_args(msgs)
    if fn == "sigcheck_channel_update_batch":
        lib.sigcheck_channel_update_batch(p, l, buf(H(signers)), len(msgs), st)
    else:
        getattr(lib, fn)(p, l, len(msgs), st)
    out["gossip"].append(list(st))
out["burst"] = []
for msgs, kinds, signers in sc["burst"]:
    st = (ctypes.c_int * len(msgs))()
    p, l = msgs_args(msgs)
    lib.sigcheck_gossip_batch(buf(H(sc["chain"])), p, l, len(msgs), buf(H(kinds)) if kinds else None,
                              buf(H(signers)) if signers else None, st)
    out["burst"].append(list(st))
print(json.dumps(out))
"""


def _rev(b):
    """libsecp256k1's opaque structs hold two 32-byte numbers as little-endian limbs"""
    return b[31::-1] + b[:31:-1]


def _ser_out(sat, s):
    return le(sat, 8) + (bytes([len(s)]) if len(s) < 0xFD else b"\xfd" + le(len(s), 2)) + s


def _bigsize(v):
    return bytes([v]) if v < 0xFD else b"\xfd" + v.to_bytes(2, "big") if v <= 0xFFFF else b"\xfe" + v.to_bytes(4, "big")


def test_dropin_client_mode(tmp_path, bins):
    """every client-mode drop-in function returns what the fake dictates for the request it should have sent, and no
    in-process path is taken (the fake library's sv_create aborts)"""
    rng = np.random.default_rng(21)
    H = lambda b: b.hex()  # noqa: E731
    sc, want = dict(chain=H(TESTNET)), {}
    ders = [_rand(rng, 33) for _ in range(12)] + [b"", _rand(rng, 32), _rand(rng, 34)]
    sc["der"] = [H(d) for d in ders]
    want["der"] = []
    for d in ders:
        h = fnv(d) if len(d) == 33 else None
        want["der"].append(H(_rev(fill(h, 64))) if h is not None and h % 3 else None)
    data = [_rand(rng, x) for x in (0, 1, 55, 64, 300)]
    sc["sha"], want["sha"] = [H(d) for d in data], [H(fill(fnv(d), 32)) for d in data]

    def verdict(kind, msg, key, sig):
        return fnv(bytes([kind]) + msg + key + sig) % 3 == 1

    items = [(_rand(rng, 32), _rand(rng, 64), _rand(rng, 64)) for _ in range(24)]
    sc["signed"] = [(H(m), H(s), H(k)) for m, s, k in items]
    want["signed"] = [verdict(1, m, _rev(k), _rev(s)) for m, s, k in items]
    nid = [(m, s, _rand(rng, 33)) for m, s, _ in items]
    sc["nodeid"] = [(H(m), H(s), H(k)) for m, s, k in nid]
    want["nodeid"] = [verdict(0, m, k, _rev(s)) for m, s, k in nid]
    sc["schnorr"] = [(H(m), H(s), H(k)) for m, s, k in items]
    want["schnorr"] = [verdict(2, m, _rev(k)[:32], s) for m, s, k in items]
    key = _rand(rng, 64)
    sc["batch"], want["batch"] = [], []
    for n in (1, 9):
        hs, ss = [_rand(rng, 32) for _ in range(n)], [_rand(rng, 64) for _ in range(n)]
        sc["batch"].append((H(b"".join(hs)), H(b"".join(s + le(1, 4) for s in ss)), H(key), n))
        want["batch"].append([verdict(1, h, _rev(key), _rev(s)) for h, s in zip(hs, ss)])
    # check_tx_sig: transactions of 1-3 inputs and 1-4 outputs, every sighash type the gate passes or refuses
    sc["tx"], want["tx"] = [], []
    for it in range(30):
        nin, nout = int(rng.integers(1, 4)), int(rng.integers(1, 5))
        ins = [(_rand(rng, 32), int(rng.integers(0, 5)), int(rng.integers(0, 2**32))) for _ in range(nin)]
        outs = [(int(rng.integers(0, 2**40)), _rand(rng, int(rng.choice([0, 22, 34, 300])))) for _ in range(nout)]
        inp, script = int(rng.integers(0, nin)), _rand(rng, int(rng.choice([1, 71, 300])))
        sht, witness = int(rng.choice([1, 1, 0x83, 0x83, 2, 3])), bool(rng.random() < 0.8)
        c = dict(version=2, locktime=int(rng.integers(0, 2**31)), ins=[(H(t), i, s) for t, i, s in ins],
                 outs=[(sat, H(s)) for sat, s in outs], input=inp, script=H(script), witness=witness,
                 amount=int(rng.integers(0, 2**45)), key=H(_rand(rng, 64)), sig=H(_rand(rng, 64) + le(sht, 4)))
        sc["tx"].append(c)
        if sht != 1 and not (witness and sht == 0x83):
            want["tx"].append(False)
            continue
        if sht & 0x1F == 3:
            o = _ser_out(*outs[inp]) if inp < nout else b""
            flags = 1 if inp < nout else 4
        else:
            o, flags = b"".join(_ser_out(*x) for x in outs), 1
        pv = b"".join(t + le(i, 4) for t, i, _ in ins) if nin > 1 else b""
        sq = b"".join(le(s, 4) for _, _, s in ins) if nin > 1 else b""
        f = dict(version=2, locktime=c["locktime"], sequence=ins[inp][2], sighash_type=sht, prev_txid=ins[inp][0],
                 prev_index=ins[inp][1], flags=flags | (2 if nin > 1 else 0), input_amount=c["amount"], output_amount=0)
        sig = bytes.fromhex(c["sig"])[:64]
        want["tx"].append(tx_hash(1, _rev(bytes.fromhex(c["key"])), _rev(sig), f, [script, o, pv, sq]) % 3 == 1)
    # check_tx_sigs_bip143_batch on sv_tx records (tests/txsig.py), the sighash type of each signature gated
    txs, blob = txsig.make_multi_txs(rng, 12)
    shts = [int(x) for x in rng.choice([1, 0x83, 2, 3], size=12)]
    sigs = [_rand(rng, 64) for _ in range(12)]
    sc["bip143"] = [(H(bytes(txs)), H(blob), H(key), H(b"".join(s + le(t, 4) for s, t in zip(sigs, shts))), 12)]
    want["bip143"] = [[]]
    for t, s, sht in zip(txs, sigs, shts):
        f = {k: getattr(t, k) for k in txsig.U32_FIELDS + ["input_amount", "output_amount"]}
        f["prev_txid"], f["sighash_type"] = bytes(t.prev_txid), sht
        ok = tx_hash(1, _rev(key), _rev(s), f, list(txsig.spans(t, blob))) % 3 == 1
        want["bip143"][0].append(ok and sht in (1, 0x83))
    # bolt12_check_signature: the fields serialised as one TLV stream, sent under the call's tag
    sc["bolt12"], want["bolt12"] = [], []
    for it in range(12):
        fields = [(int(t), _rand(rng, int(rng.choice([0, 3, 40, 300])))) for t in sorted(rng.choice(70000, 4, replace=False))]
        mn, fn = TAGS[it % 3]
        k, s = _rand(rng, 64), _rand(rng, 64)
        sc["bolt12"].append(([(t, H(v)) for t, v in fields], mn.decode(), fn.decode(), H(k), H(s)))
        stream = b"".join(_bigsize(t) + _bigsize(len(v)) + v for t, v in fields)
        want["bolt12"].append(fnv(mn + b"\0" + fn + b"\0" + stream + _rev(k)[:32] + s) % 3 - 1 == 1)
    # the typed gossip entry points (a message of another type is -1 whatever the daemon says) and bursts
    sc["gossip"], want["gossip"] = [], []
    for fn, typ in (("sigcheck_channel_announcement_batch", 256), ("sigcheck_node_announcement_batch", 257),
                    ("sigcheck_channel_update_batch", 258)):
        msgs = [(t if rng.random() < 0.8 else 259).to_bytes(2, "big") + _rand(rng, int(rng.integers(0, 200)))
                for t in [typ] * 15] + [b"\x01"]
        signers = _rand(rng, 33 * len(msgs)) if typ == 258 else bytes(33 * len(msgs))
        sc["gossip"].append((fn, [H(m) for m in msgs], H(signers)))
        want["gossip"].append([fnv(m + signers[33 * i:33 * i + 33]) % 6 - 1 if m[:2] == typ.to_bytes(2, "big") else -1
                               for i, m in enumerate(msgs)])
    sc["burst"], want["burst"] = [], []
    for with_kinds in (False, True):
        msgs = [_rand(rng, int(rng.integers(2, 200))) for _ in range(20)]
        kinds = bytes(int(x) for x in rng.integers(0, 3, size=20)) if with_kinds else bytes(20)
        signers = _rand(rng, 33 * 20) if with_kinds else bytes(33 * 20)
        sc["burst"].append(([H(m) for m in msgs], H(kinds) if with_kinds else None, H(signers) if with_kinds else None))
        want["burst"].append([fnv(TESTNET + m + kinds[i:i + 1] + signers[33 * i:33 * i + 33]) % 10 - 4
                              for i, m in enumerate(msgs)])
    path = tmp_path / "scenario.json"
    path.write_text(json.dumps(sc))
    ctx, log = _start(tmp_path, bins["daemon"])
    with ctx as sock:
        env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CLN_SIGVERIFYD_SOCKET=sock)
        r = subprocess.run([sys.executable, "-c", CLIENT, str(path), bins["lib"]], env=env, cwd=str(tmp_path),
                           capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-3000:]
        got = json.loads(r.stdout)
        sent = sigverifyd_daemon.stats(sock)["requests"]
    for k in want:
        assert got[k] == want[k], k
    assert sum(want["signed"]) and sum(want["tx"]) and sum(want["bolt12"]) and any(want["bip143"][0])
    assert sent == (12 + len(data) + 3 * 24 + 2 + sum(1 for c in sc["tx"] if c["sig"][-8:] in ("01000000",) or
                    (c["witness"] and c["sig"][-8:] == "83000000")) + 1 + 12 + 3 + 2)

