"""GPU: whole gossip_stores (sv_verify_gossip_store_host).  The committed store fixture, the fixture with ~1 % of its
signatures bit-flipped (checksums recomputed) against CLN's own gossipd/sigcheck.c with the channel table of
tests/gossip_store.py, crafted signed stores for every channel-table rule, gate and stop, both verification paths, the
fixture tiled x53, argument errors and the cln_verify_gossip_store tool's exit codes."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200.engine import EngineError, GS_NO_HOLDER
from tests import gossip_store as gs
from tests.test_gossip_store_host import load_fixture
from tests.test_gpu_gossip_burst import OTHER, TESTNET, _ordered, make_ca, make_cu

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "lightning_b200", "cln_verify_gossip_store")
P = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))  # noqa: E731


def run(engine, store, chain=None):
    """the engine's answer in the model's form"""
    off, typ, st, hold, s = engine.verify_gossip_store(store, chain)
    out = [(int(o), int(t), int(x), None if h == GS_NO_HOLDER else int(h)) for o, t, x, h in zip(off, typ, st, hold)]
    return out, s


def agree(engine, store, chain=None, sigcheck=None):
    """engine == model record for record, and the summary's counts are those of the records"""
    got, s = run(engine, store, chain)
    want, ws = gs.audit(store, sigcheck)
    if sigcheck is None:  # signature statuses from the engine (crafted stores state them), everything else from the model
        want = [(o, t, g[2] if t in (256, 257, 258) and x == 0 else x, h) for (o, t, x, h), g in zip(want, got)]
    assert got == want
    for k in ("version", "stop", "end_offset", "records", "redundant_announcements", "updates_without_channel",
              "ended_equivalent_offset"):
        assert s[k] == ws[k], k
    msg = [x for _, t, x, _ in got if t in (256, 257, 258) and x < 16]
    assert (s["good"], s["bad_signature"], s["malformed"], s["no_channel"], s["wrong_chain"], s["bad_order"]) == (
        msg.count(0), sum(1 <= x <= 4 for x in msg), msg.count(-1), msg.count(-2), msg.count(-3), msg.count(-4))
    return got, s


def cln_sigcheck(cln, chain):
    """gossipd's verdict on one message: CLN's sigcheck_*, then (with a chain hash) its gates; an update is checked
    under the signer the channel table gives (-2 where the scid holds no channel)"""
    zero = np.zeros(33, np.uint8)

    def f(m, signer):
        L = ctypes.c_size_t(len(m))
        t = struct.unpack(">H", m[:2])[0]
        if t == 256:
            s = cln.cln_sigcheck_channel_announcement(m, L)
            if s != -1 and chain is not None:
                ch, _, n1, n2 = gs.ann_fields(m)
                s = -4 if n1 >= n2 else (-3 if ch != chain else s)
            return s
        if t == 257:
            return cln.cln_sigcheck_node_announcement(m, L)
        if len(m) < 138:
            return -1
        k = zero if signer is None else np.frombuffer(bytes(signer), np.uint8).copy()
        s = cln.cln_sigcheck_channel_update(m, L, P(k))
        if s != -1:
            if chain is not None and m[66:98] != chain:
                s = -3
            elif signer is None:
                s = -2
        return s
    return f


def messages(store):
    recs, _, _, _ = gs.walk(store)
    return [store[o + 12:o + 12 + n] for o, t, n, st in recs if st == 0 and t in (256, 257, 258)]


def test_fixture_all_good(engine):
    store = load_fixture()
    for chain in (None, TESTNET):
        got, s = agree(engine, store, chain)
        assert s["version"] == 15 and s["stop"] == gs.EOF and s["records"] == 4600
        assert s["good"] == 3100 and s["store_records"] == 1500
        assert all(x in (0, gs.STORE_RECORD) for _, _, x, _ in got)
        assert sum(t == 258 and h is not None for _, t, _, h in got) == 1200


def test_fixture_both_paths_equal_burst(engine):
    """the latency path (7,600 signatures) and the throughput path give the statuses sv_verify_gossip_burst_host gives
    for the same messages"""
    store = load_fixture()
    burst = engine.verify_gossip_burst(messages(store), TESTNET).tolist()
    small = engine.small_max()
    try:
        for sm in (small, 0):
            engine.set_small_max(sm)
            got, _ = run(engine, store, TESTNET)
            assert [x for _, t, x, _ in got if t in (256, 257, 258)] == burst
    finally:
        engine.set_small_max(small)


def flipped_store():
    """~1 % of the fixture's signatures with one bit flipped, every checksum recomputed"""
    store = bytearray(load_fixture())
    rng = np.random.default_rng(2027)
    recs, _, _, _ = gs.walk(bytes(store))
    for off, t, ln, _ in recs:
        if t not in (256, 257, 258):
            continue
        m = off + 12
        for k in range(4 if t == 256 else 1):
            if rng.random() < 0.01:
                store[m + 2 + 64 * k + int(rng.integers(0, 64))] ^= 1 << int(rng.integers(0, 8))
        struct.pack_into(">I", store, off + 4, gs.crc32c(struct.unpack(">I", store[off + 8:off + 12])[0], store[m:m + ln]))
    return bytes(store)


def test_flipped_vs_cln(engine, cln):
    """every status of the bit-flipped store equals CLN's sigcheck under the model's signer (replayed), without and
    with the chain gates"""
    store = flipped_store()
    for chain in (None, TESTNET):
        got, s = agree(engine, store, chain, cln_sigcheck(cln, chain))
        codes = [x for _, t, x, _ in got if t in (256, 257, 258)]
        assert s["stop"] == gs.EOF and codes.count(0) > 2900
        for c in (1, 2, 3, 4):
            assert c in codes, c


def test_tiled_x53(engine):
    """the fixture's records 53 times over: the copies are redundant announcements and updates that resolve to the first
    copy; throughput kernels and key de-duplication; equal to a burst of the same messages"""
    fx = load_fixture()
    store = fx[:1] + fx[1:] * 53
    got, s = agree(engine, store, TESTNET)
    assert s["records"] == 4600 * 53 and s["good"] == 3100 * 53 and s["redundant_announcements"] == 1500 * 52
    first = {h for _, t, _, h in got if t == 258}
    assert max(first) < len(fx)
    assert [x for _, t, x, _ in got if t in (256, 257, 258)] == engine.verify_gossip_burst(messages(store), TESTNET).tolist()


# ---- crafted signed stores -----------------------------------------------------------------------------------------
A, B = b"\x00\x00\x01\x00\x00\x02\x00\x01", b"\x00\x00\x01\x00\x00\x03\x00\x01"
AMT = gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 1000))


def ann(*a, **k):
    return gs.record(make_ca(*a, **k)) + AMT


def upd(*a, **k):
    return gs.record(make_cu(*a, **k))


def store_of(*recs):
    return bytes([16]) + b"".join(recs)


def statuses(engine, store, chain=None):
    got, _ = agree(engine, store, chain)
    return [x for _, t, x, _ in got if t in (256, 258) and x < 16]


def test_redundant_announcement(engine):
    a, b = _ordered("a", "b")
    x, y = _ordered("x", "y")
    st = store_of(ann(A, a, b), ann(A, x, y), upd(A, a, 0), upd(A, x, 0), upd(A, b, 1), upd(A, y, 1))
    assert statuses(engine, st) == [0, 0, 0, 1, 0, 1]


def test_delete_and_reannounce(engine):
    a, b = _ordered("a", "b")
    x, y = _ordered("x", "y")
    dele = gs.record(struct.pack(">H", gs.DELETE_CHAN) + A)
    st = store_of(ann(A, a, b), upd(A, a, 0), dele, upd(A, a, 0), ann(A, x, y), upd(A, x, 0), upd(A, a, 0))
    assert statuses(engine, st) == [0, 0, -2, 0, 0, 1]
    # a deleted delete_chan takes no part
    dead = gs.record(struct.pack(">H", gs.DELETE_CHAN) + A, flags=gs.COMPLETED | gs.DELETED)
    assert statuses(engine, store_of(ann(A, a, b), dead, upd(A, a, 0))) == [0, 0]


def test_deleted_announcement_and_early_update(engine):
    a, b = _ordered("a", "b")
    x, y = _ordered("x", "y")
    dead = gs.record(make_ca(A, x, y), flags=gs.COMPLETED | gs.DELETED) + AMT
    st = store_of(upd(A, a, 0), dead, upd(A, x, 0), ann(A, a, b), upd(A, a, 0))
    assert statuses(engine, st) == [-2, -2, 0, 0]


def test_failing_announcement_holds_its_channel(engine):
    a, b = _ordered("a", "b")
    x, y = _ordered("x", "y")
    st = store_of(ann(A, a, b, bad=2), ann(A, x, y), upd(A, a, 0), upd(A, x, 0))
    assert statuses(engine, st) == [3, 0, 0, 1]
    # malformed (a bitcoin key cut off): -1, and it still holds its channel
    short = make_ca(B, a, b)[:-40]
    st = store_of(gs.record(short) + AMT, ann(B, x, y), upd(B, a, 0), upd(B, x, 0))
    assert statuses(engine, st) == [-1, 0, 0, 1]


def test_chain_gates(engine):
    a, b = _ordered("a", "b")
    st = store_of(ann(A, a, b, chain=OTHER), upd(A, a, 0, chain=OTHER), ann(B, a, b, swap=True), upd(B, b, 0))
    assert statuses(engine, st) == [0, 0, 0, 0]
    assert statuses(engine, st, TESTNET) == [-3, -3, -4, 0]
    # the other chain for an update without a channel: the chain gate comes first
    assert statuses(engine, store_of(upd(A, a, 0, chain=OTHER)), TESTNET) == [-3]
    assert statuses(engine, store_of(upd(A, a, 0, chain=OTHER))) == [-2]


def test_bad_crc_cuts_verification(engine):
    a, b = _ordered("a", "b")
    recs = [ann(A, a, b), upd(A, a, 0), upd(A, b, 1), upd(A, a, 0, ts=2)]
    st = bytearray(store_of(*recs))
    mid = 1 + len(recs[0]) + len(recs[1])
    st[mid + 12 + 100] ^= 1
    got, s = agree(engine, bytes(st))
    assert [x for _, _, x, _ in got] == [0, gs.STORE_RECORD, 0, gs.BAD_CRC, gs.NOT_REACHED]
    assert s["stop"] == gs.BAD_CRC and s["end_offset"] == mid and s["not_reached"] == 1
    # an announcement at the end without its amount record stops the walk; the same store one byte longer is fine
    tail = store_of(ann(A, a, b), gs.record(make_ca(B, a, b)))
    assert agree(engine, tail)[1]["stop"] == gs.NO_AMOUNT


def test_argument_errors(engine):
    store = load_fixture()
    n = engine.lib.sv_gossip_store_count(store, len(store))
    assert n == 4600
    with pytest.raises(EngineError):
        engine.verify_gossip_store(store, capacity=n - 1)
    with pytest.raises(EngineError):
        engine.verify_gossip_store(bytes([0x20]) + store[1:])
    with pytest.raises(ValueError):
        engine.verify_gossip_store(store, chain_hash=b"\x00" * 31)
    # any minor version; a store of the version byte alone has no records
    off, _, _, _, s = engine.verify_gossip_store(bytes([0x1F]) + store[1:])
    assert s["records"] == 4600 and s["version"] == 0x1F
    assert engine.verify_gossip_store(b"\x10")[4]["records"] == 0
    # the engine still works for ordinary calls afterwards
    assert run(engine, store)[1]["good"] == 3100


def test_cli_exit_codes(tmp_path):
    fx = load_fixture()
    bad = bytearray(fx)
    bad[gs.walk(fx)[0][2300][0] + 12 + 10] ^= 1  # inside a message in the middle of the store
    for name, data, code in (("clean", fx, 0), ("flipped", flipped_store(), 1), ("badcrc", bytes(bad), 2)):
        p = tmp_path / name
        p.write_bytes(data)
        r = subprocess.run([TOOL, "--chain", TESTNET.hex(), str(p)], capture_output=True, text=True, timeout=300)
        assert r.returncode == code, (name, r.stdout[-2000:], r.stderr[-2000:])
        assert "records" in r.stdout
    r = subprocess.run([TOOL, "--chain", "00", str(p)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 3
