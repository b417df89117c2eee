"""CPU: salvaging a gossip_store past damaged record headers.  The host build of gossip_salvage.cuh (the candidate test,
the checksum of a long candidate in the warp's 32 slices, the walk) against the Python model (tests/gossip_store_salvage.py)
on the fixture and on every damage class; what the model makes of each class pruned by the prune's model, cut by the
repair's rule and loaded by Core Lightning's gossmap.c strictly, as gossipd loads its store at start-up; and
sv_salvage_gossip_store_fd (lightning_b200/csrc/gossip_salvage_fd.c) built with gcc against a CPU salvage and the fake
prune of tests/host_emul/fake_engine_prune.c, with every pwrite it makes logged.  CLN's answers are recorded under
tests/golden/oracle/ (tests/oracle_replay.py)."""
import ctypes
import errno
import os
import struct
import subprocess

import numpy as np
import pytest

from lightning_b200 import build
from lightning_b200.engine import SvGossipPruneSummary, SvGossipSalvageSummary
from tests import gossip_store as gs
from tests import gossip_store_prune as gp
from tests import gossip_store_salvage as sv
from tests.test_gossip_store_host import load_fixture
from tests.test_gossip_store_prune_host import oracle, strict_load
from tests.test_sigverifyd_prune_fake import fake_prune
from tests.test_sigverifyd_repair_fake import cut_rule

HE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = ctypes.c_uint64


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---- the stores and the damage classes (tests/test_gpu_gossip_store_salvage.py uses them too) -------------------------
def with_uuid(store):
    """store with a gossip_store_uuid record first, as gossipd starts a store, and one channel_update deleted the way
    gossipd deletes (its checksum kept)"""
    uuid = gs.record(struct.pack(">H", gs.UUID) + bytes(range(32)))
    out = bytearray(store[:1] + uuid + store[1:])
    recs = gs.walk(bytes(out))[0]
    upd = [r for r in recs if r[1] == 258][len(recs) // 5]
    out[upd[0]] |= gs.DELETED >> 8
    return bytes(out)


def x53():
    fx = load_fixture()
    return fx[:1] + fx[1:] * 53


def header_flips(store):
    """name -> store with one bit of one header flipped: the length's high byte (bit 0), its low byte (bit 4), COMPLETED
    cleared; at the records 10 %, 50 % and 90 % into the store.  -> {name: (store, damaged record index)}"""
    recs = gs.walk(store)[0]
    out = {}
    for i in (len(recs) // 10, len(recs) // 2, 9 * len(recs) // 10):
        o = recs[i][0]
        for name, at, mask in (("len_hi", 2, 0x01), ("len_lo", 3, 0x10), ("completed", 0, 0x20)):
            d = bytearray(store)
            d[o + at] ^= mask
            out["%s_%d" % (name, i)] = (bytes(d), i)
    return out


def damage_classes(store):
    """name -> (damaged store, (first, end) of the damaged bytes) of a with_uuid() store"""
    recs = gs.walk(store)[0]
    n = len(recs)
    off = [r[0] for r in recs]

    def flip(d, o, mask):
        d[o] ^= mask
        return o, o + 1

    out = {}
    for name, at, mask in (("len_hi", 2, 0x01), ("len_lo", 3, 0x10), ("completed", 0, 0x20)):
        d = bytearray(store)
        out[name] = (d, flip(d, off[n // 3] + at, mask))
    d = bytearray(store)
    d[off[n // 3]:off[n // 3] + 12] = bytes(12)
    out["header_zeroed"] = (d, (off[n // 3], off[n // 3] + 12))
    d = bytearray(store)
    z = off[n // 4] + 40
    d[z:z + 100000] = bytes(100000)
    out["zeroed_100k"] = (d, (z, z + 100000))
    d = bytearray(store)
    d[off[n // 5] + 2] ^= 0x01
    d[off[3 * n // 5]:off[3 * n // 5] + 12] = bytes(12)
    out["two_breaks"] = (d, (off[n // 5] + 2, off[3 * n // 5] + 12))
    assert recs[0][1] == gs.UUID
    d = bytearray(store)
    out["first_record"] = (d, flip(d, off[0] + 3, 0x04))
    dl = next(i for i, r in enumerate(recs) if r[3] == gs.ST_DELETED)
    d = bytearray(store)
    out["deleted_length"] = (d, flip(d, off[dl] + 2, 0x01))
    d = bytearray(store)
    out["last_payload"] = (d, flip(d, off[-1] + 12 + 50, 0x08))
    d = bytearray(store)
    out["last_length"] = (d, flip(d, off[-1] + 3, 0x04))
    return {k: (bytes(v), s) for k, (v, s) in out.items()}


# ---- the host build against the model --------------------------------------------------------------------------------
def emul_sound(emul, store):
    emul.emul_gs_salvage_sound.restype = U64
    emul.emul_gs_salvage_sound.argtypes = [ctypes.c_char_p, U64, ctypes.c_void_p, U64]
    n = emul.emul_gs_salvage_sound(store, len(store), None, 0)
    out = np.zeros(max(n, 1), np.uint64)
    assert emul.emul_gs_salvage_sound(store, len(store), _p(out), n) == n
    return [int(x) for x in out[:n]]


def emul_salvage(emul, store, sound):
    """the host walk's (bytes, actions, summary) in the model's form"""
    emul.emul_gs_salvage_walk.restype = U64
    emul.emul_gs_salvage_walk.argtypes = [ctypes.c_char_p, U64, ctypes.c_void_p, U64] + [ctypes.c_void_p] * 3 + \
        [U64, ctypes.c_void_p]
    buf = ctypes.create_string_buffer(bytes(store), len(store))
    snd = np.array(sound or [0], np.uint64)
    cap = 4096
    off, res, kind, c5 = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint8), np.zeros(5, np.uint64)
    n = emul.emul_gs_salvage_walk(buf, len(store), _p(snd), len(sound), _p(off), _p(res), _p(kind), cap, _p(c5))
    assert n <= cap
    s = dict(zip(sv.FIELDS, [int(x) for x in c5] + [len(sound)]))
    return buf.raw, [(int(off[k]), int(res[k]), int(kind[k])) for k in range(n)], s


def test_crc_by_pieces(emul):
    """a long candidate's checksum as the warp computes it (32 slices, each shifted past the bytes after it) is ccan's
    crc32c for every length and start value; the shift is crc32c over zero bytes"""
    emul.emul_gs_crc_warp.restype = ctypes.c_uint32
    emul.emul_gs_crc_warp.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32]
    emul.emul_gs_crc_shift.restype = ctypes.c_uint32
    emul.emul_gs_crc_shift.argtypes = [ctypes.c_uint32, U64]
    rng = np.random.default_rng(3)
    for n in (0, 1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 1024, 1025, 2047, 4099, 65535):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        for start in (0, 1, 0xFFFFFFFF, int(rng.integers(0, 2**32))):
            assert emul.emul_gs_crc_warp(start, data, n) == gs.crc32c(start, data), (n, start)
    for n in (0, 1, 2, 3, 100, 1000, 65535, 65547):
        for c in (0, 1, 0x80000000, int(rng.integers(0, 2**32))):
            assert emul.emul_gs_crc_shift(c, n) == gs.crc32c(c, bytes(n)) ^ gs.crc32c(0, bytes(n)), (n, c)


def crafted():
    """sound records longer than 1,024 bytes, a long one with a bad checksum, a record that ends exactly at the end of
    the store, and candidates whose length runs one byte past it"""
    rng = np.random.default_rng(4)
    good = gs.record(struct.pack(">H", 257) + rng.integers(0, 256, 3000, dtype=np.uint8).tobytes(), ts=7)
    bad = bytearray(gs.record(struct.pack(">H", 258) + rng.integers(0, 256, 2000, dtype=np.uint8).tobytes(), ts=9))
    bad[100] ^= 1
    amount = gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 5))
    past = bytearray(gs.record(struct.pack(">HQ", gs.CHANNEL_AMOUNT, 6)))
    past[3] += 1
    return {"long": b"\x0c" + good + bytes(bad) + good + amount,
            "ends_at_end": b"\x0c" + amount + good,
            "runs_past": b"\x0c" + amount + bytes(past)[:-1] + bytes(1)}


def test_sound_offsets(emul):
    """the host build finds the model's sound offsets on the fixture, on the damage classes and on crafted stores"""
    fx = load_fixture()
    base = with_uuid(fx)
    assert emul_sound(emul, fx) == sv.sound_offsets(fx) == [r[0] for r in gs.walk(fx)[0]]
    for k, (st, _) in damage_classes(base).items():
        assert emul_sound(emul, st) == sv.sound_offsets(st), k
    c = crafted()
    for k, st in c.items():
        assert emul_sound(emul, st) == sv.sound_offsets(st), k
    assert sv.sound_offsets(c["long"]) == [1, 1 + 3014 + 2014, 1 + 2 * 3014 + 2014]
    assert sv.sound_offsets(c["ends_at_end"]) == [1, 1 + 22]
    assert sv.sound_offsets(c["runs_past"]) == [1]


def test_walk_against_model(emul):
    """the host walk writes the model's bytes, lists its actions and counts its summary on every damage class"""
    base = with_uuid(load_fixture())
    for k, (st, _) in list(damage_classes(base).items()) + [("clean", (base, None))]:
        snd = sv.sound_offsets(st)
        want = sv.salvage(st, snd)
        assert emul_salvage(emul, st, snd) == want, k


# ---- what the rule does ----------------------------------------------------------------------------------------------
def test_one_header_bit_keeps_every_record():
    """each single header flip of the fixture (length high byte, length low byte, COMPLETED; at 10, 50 and 90 %) is
    restored: the salvaged store is the fixture, with all 4,600 records"""
    fx = load_fixture()
    assert len(gs.walk(fx)[0]) == 4600
    for k, (st, i) in header_flips(fx).items():
        out, acts, s = sv.salvage(st)
        t = gs.walk(fx)[0][i][0]
        assert out == fx, k
        assert acts == [(t, gs.walk(fx)[0][i + 1][0], sv.RESTORED)], k
        assert (s["breaks"], s["restored"], s["bridged"]) == (1, 1, 0), k


def test_bridge_pieces():
    """a bridge takes as few fillers as fit 65,547 bytes each, none under 14 bytes"""
    for span in (14, 15, 65546, 65547, 65548, 65561, 131094, 131095, 200000, 10**6):
        p = sv.pieces(span)
        assert sum(p) == span and len(p) == -(-span // sv.PIECE) and all(14 <= x <= sv.PIECE for x in p), span
        assert max(p) - min(p) <= 1


def test_no_break_writes_nothing():
    """stores without a break: the fixture, stores the prune deletes from (a bad checksum and a record of 1 byte in
    mid-store, an unknown type), torn tails (cut inside the last records, the last record without COMPLETED), and a
    store whose walk ends at a gossip_store_ended record"""
    fx = load_fixture()
    recs = gs.walk(fx)[0]
    mid = recs[2300][0]
    bad = bytearray(fx)
    bad[recs[1200][0] + 12 + 20] ^= 4
    stores = {"fixture": fx, "with_uuid": with_uuid(fx),
              "bad_crc_and_truncated": bytes(bad[:mid]) + gs.record(b"\x01") + bytes(bad[mid:]),
              "truncated_empty": fx[:mid] + gs.record(b"") + fx[mid:],
              "unknown_type": fx[:mid] + gs.record(struct.pack(">HI", 4999, 1)) + fx[mid:],
              "ended": fx[:mid] + gs.record(struct.pack(">HQ", gs.ENDED, mid)) + fx[mid:mid + 5000]}
    for t in (recs[-2][0] + 1, recs[-2][0] + 12, recs[-2][0] + 13, recs[-1][0] - 1, len(fx) - 1):
        stores["torn_%d" % t] = fx[:t]
    inc = bytearray(fx)
    inc[recs[-1][0]] &= ~0x20 & 0xFF
    stores["last_incomplete"] = bytes(inc)
    for k, st in stores.items():
        out, acts, s = sv.salvage(st)
        assert out == st and acts == [] and s["breaks"] == 0, k


def test_salvaging_twice_writes_nothing():
    base = with_uuid(load_fixture())
    for k, (st, _) in damage_classes(base).items():
        once = sv.salvage(st)[0]
        out, acts, s = sv.salvage(once)
        assert out == once and acts == [], k


# ---- gossmap's strict load of the result -----------------------------------------------------------------------------
def repaired(store):
    """the model's salvage, then the prune's model (every message status 0) and the repair's cut: (file, prune rows)"""
    out = sv.salvage(store)[0]
    pruned, rows, s = gp.prune(out)
    return pruned[:cut_rule(pruned, s)], rows


def kept_changes(base, span, want_rows, got_rows):
    """every record of the undamaged store outside the damaged span [first, end) keeps its prune row (want_rows: the
    prune of base, got_rows: the prune of the salvaged store), except the updates, later announcements and their amount
    records of a channel whose holding announcement lay in the span: their status and reason follow the new holder"""
    want = {r[0]: r for r in want_rows}
    got = {r[0]: r for r in got_rows}
    recs = gs.walk(base)[0]
    lost = {gs.ann_fields(base, o + 12)[1] for o, t, ln, _ in recs if t == 256 and o < span[1] and o + 12 + ln > span[0]}
    for i, (o, t, ln, _) in enumerate(recs):
        if span[0] < o + 12 + ln and o < span[1]:
            continue
        assert o in got, o
        if got[o] == want[o]:
            continue
        a = recs[i - 1][0] + 12 if t == gs.CHANNEL_AMOUNT else o + 12
        scid = base[o + 12 + 98:o + 12 + 106] if t == 258 else gs.ann_fields(base, a)[1]
        assert scid in lost and got[o][:2] == want[o][:2], (o, got[o], want[o])


def test_strict_load_accepts_every_class():
    """each damage class salvaged, pruned and cut loads under gossmap's strict load with expected_len = its length; the
    records outside the damage keep their prune; a damaged last record is repaired exactly as without the salvage"""
    o = oracle()
    base = with_uuid(load_fixture())
    want_rows = gp.prune(base)[1]
    for k, (st, span) in damage_classes(base).items():
        f, rows = repaired(st)
        ref = strict_load(o, f)
        assert ref is not None and ref[0] == len(f), k
        kept_changes(base, span, want_rows, rows)
        if k.startswith("last_"):
            pruned, _, s = gp.prune(st)
            assert f == pruned[:cut_rule(pruned, s)], k


# ---- sv_salvage_gossip_store_fd against the fake prune ---------------------------------------------------------------
@pytest.fixture(scope="module")
def fdlib(tmp_path_factory):
    d = tmp_path_factory.mktemp("salvage_fd")
    objs = []
    for src in (os.path.join(build.CSRC, "gossip_store_fd.c"), os.path.join(build.CSRC, "gossip_salvage_fd.c"),
                os.path.join(HE, "fake_engine_prune.c"), os.path.join(HE, "pwrite_log.c")):
        o = str(d / (os.path.basename(src) + ".o"))
        r = subprocess.run(["gcc"] + build.DROPIN_CFLAGS + ["-c", src, "-o", o], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        objs.append(o)
    o = str(d / "fake_engine_salvage.o")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-c",
                        os.path.join(HE, "fake_engine_salvage.cpp"), "-o", o], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = str(d / "libsalvage_fd.so")
    r = subprocess.run(["g++", "-shared", "-Wl,--wrap=pwrite,--wrap=fsync"] + objs + [o, "-o", lib], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = ctypes.CDLL(lib, use_errno=True)
    L.sv_salvage_gossip_store_fd.argtypes = [ctypes.c_void_p, ctypes.c_int, U64, ctypes.c_void_p,
                                             ctypes.POINTER(SvGossipPruneSummary), ctypes.POINTER(SvGossipSalvageSummary),
                                             ctypes.POINTER(U64)]
    return L


SYNC = ((1 << 64) - 1, 0)  # an fsync in the log


def salvage_fd(L, fd, length):
    """(rc, errno, prune summary, salvage summary, new_len, [(offset, length)] of every pwrite, SYNC for every fsync)"""
    ctypes.c_size_t.in_dll(L, "pwrite_log_n").value = 0
    s, v, n = SvGossipPruneSummary(), SvGossipSalvageSummary(), U64(0)
    ctypes.set_errno(0)
    rc = L.sv_salvage_gossip_store_fd(ctypes.c_void_p(1), fd, length, None, ctypes.byref(s), ctypes.byref(v), ctypes.byref(n))
    e = ctypes.get_errno()
    k = ctypes.c_size_t.in_dll(L, "pwrite_log_n").value
    offs, lens = (U64 * 65536).in_dll(L, "pwrite_log_off"), (U64 * 65536).in_dll(L, "pwrite_log_len")
    return (rc, e, {f: getattr(s, f) for f, _ in s._fields_}, {f: getattr(v, f) for f, _ in v._fields_}, n.value,
            [(offs[i], lens[i]) for i in range(k)])


def salvage_writes(out, acts):
    """the pwrites the salvage must make: 4 bytes per header, a bridge's fillers from the last to the first and synced
    before the first overwrites the damaged header, then one fsync"""
    w = []
    for t, q, kind in acts:
        if kind == sv.RESTORED:
            w.append((t, 4))
            continue
        p, fl = t, []
        while p < q:
            fl.append((p, 4))
            p += 12 + struct.unpack(">H", out[p + 2:p + 4])[0]
        w += fl[:0:-1] + ([SYNC] if len(fl) > 1 else []) + fl[:1]
    return w + ([SYNC] if acts else [])


def test_fd_salvage_then_repair(fdlib, tmp_path):
    """the file ends as the fake repair of the model's salvage; the salvage writes only its headers, each bridge from its
    last filler to its first with an fsync before the first, then syncs, before any of the prune's flag writes; a second
    call writes no header"""
    base = with_uuid(load_fixture())
    f = tmp_path / "gossip_store"
    for k, (st, _) in damage_classes(base).items():
        out, acts, vs = sv.salvage(st)
        pruned, ps = fake_prune(out)
        cut = cut_rule(pruned, ps)
        f.write_bytes(st)
        fd = os.open(f, os.O_RDWR)
        try:
            rc, e, s, v, new_len, log = salvage_fd(fdlib, fd, len(st))
            assert (rc, s, v, new_len) == (0, ps, vs, cut), k
            head = salvage_writes(out, acts)
            assert log[:len(head)] == head and all(n == 2 or (o, n) == SYNC for o, n in log[len(head):]), k
            assert f.read_bytes() == pruned[:cut], k
            rc, e, s, v, new_len, log = salvage_fd(fdlib, fd, cut)
            assert rc == 0 and v["breaks"] == 0 and all(n == 2 or (o, n) == SYNC for o, n in log), k
        finally:
            os.close(fd)
    zeroed = sv.salvage(damage_classes(base)["zeroed_100k"][0])
    assert any(a[2] == sv.BRIDGED for a in zeroed[1]) and zeroed[2]["fillers"] > zeroed[2]["bridged"]


def test_fd_refusals(fdlib, tmp_path):
    """a read-only fd (EBADF), a pipe and a length past the end (EINVAL), a store of another major version (EINVAL): the
    repair's errors, nothing written"""
    st = damage_classes(with_uuid(load_fixture()))["len_hi"][0]
    f = tmp_path / "gossip_store"
    f.write_bytes(st)
    fd = os.open(f, os.O_RDONLY)
    try:
        assert salvage_fd(fdlib, fd, len(st))[:2] == (build_rc("IO"), errno.EBADF)
    finally:
        os.close(fd)
    r, w = os.pipe()
    try:
        assert salvage_fd(fdlib, r, 10)[:2] == (build_rc("ARG"), errno.EINVAL)
    finally:
        os.close(r)
        os.close(w)
    for data, length in ((st, len(st) + 1), (bytes([0x20]) + st[1:], len(st)), (st, 0)):
        f.write_bytes(data)
        fd = os.open(f, os.O_RDWR)
        try:
            rc, e, _, _, _, log = salvage_fd(fdlib, fd, length)
            assert (rc, e, log) == (build_rc("ARG"), errno.EINVAL, []), length
        finally:
            os.close(fd)
        assert f.read_bytes() == data


def build_rc(name):
    return {"ARG": -4, "IO": -5}[name]
