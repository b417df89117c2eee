"""gossip_store reading on the host: the committed store fixture against CLN's own checksums, and gossip_store.cuh (host
build: the checksum, the header walk and the channel-event rule the k_store_* kernels run) against the Python model of
gossmap's map_catchup (tests/gossip_store.py), on the fixture and on crafted stores for every stop reason."""
import ctypes
import json
import os
import struct

import numpy as np
import pytest

from tests import gossip_store as gs
from tests.gossip_store import load_fixture

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
P8 = ctypes.POINTER(ctypes.c_uint8)
CHAIN = bytes.fromhex("43497fd7f826957108f4a30fd9cec3aeba79972084e90ead01ea330900000000")


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def emul_audit(emul, store):
    """the host build's answer in the model's form: walk, checksums up to the first bad one, channel events in store
    order; signature statuses are not computed here (0), record statuses and holders are"""
    emul.emul_gs_walk.restype = ctypes.c_longlong
    emul.emul_gs_walk.argtypes = [ctypes.c_char_p, ctypes.c_uint64] + [ctypes.c_void_p] * 4 + [ctypes.c_uint64, ctypes.c_void_p]
    emul.emul_gs_crc_ok.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    emul.emul_gs_resolve.argtypes = [ctypes.c_char_p, ctypes.c_uint64] + [ctypes.c_void_p] * 3 + [ctypes.c_size_t, ctypes.c_void_p]
    end3 = np.zeros(3, np.uint64)
    n = emul.emul_gs_walk(store, len(store), None, None, None, None, 0, _p(end3))
    off, typ, ln, st = (np.zeros(max(n, 1), d) for d in (np.uint64, np.uint32, np.uint32, np.int32))
    assert emul.emul_gs_walk(store, len(store), _p(off), _p(typ), _p(ln), _p(st), n, _p(end3)) == n
    stop = int(end3[1])
    no_amount = None if int(end3[2]) == (1 << 64) - 1 else int(end3[2])
    live = [i for i in range(n) if st[i] in (0, gs.ST_ENDED)]
    ok = np.zeros(max(len(live), 1), np.uint8)
    emul.emul_gs_crc_ok(store, _p(np.array([off[i] for i in live] or [0], np.uint64)), len(live), _p(ok))
    bad = [i for k, i in enumerate(live) if not ok[k]]
    cut, cut_status = (bad[0], gs.BAD_CRC) if bad else (n, 0)
    msgs = [i for i in range(cut) if st[i] == 0 and typ[i] in (256, 257, 258)]
    midx = {r: k for k, r in enumerate(msgs)}
    ev = [i for i in range(cut) if st[i] == 0 and typ[i] in (256, 258, gs.DELETE_CHAN)]
    kinds = np.array([{256: 0, gs.DELETE_CHAN: 1, 258: 2}[int(typ[i])] for i in ev] or [0], np.uint8)
    holder = np.full(max(len(msgs), 1), 0xFFFFFFFF, np.uint32)
    emul.emul_gs_resolve(store, len(store), _p(np.array([off[i] + 12 for i in ev] or [0], np.uint64)), _p(kinds),
                         _p(np.array([midx.get(i, 0xFFFFFFFF) for i in ev] or [0], np.uint32)), len(ev), _p(holder))
    hold = {r: (None if holder[k] == 0xFFFFFFFF else msgs[holder[k]]) for r, k in midx.items()}
    if no_amount is not None and no_amount < cut and hold.get(no_amount) is None:
        cut, cut_status = no_amount, gs.NO_AMOUNT
    out = []
    for i in range(n):
        s, h = int(st[i]), None
        if cut_status and i >= cut:
            s = cut_status if i == cut else gs.NOT_REACHED
        elif s == 0:
            if i in midx:
                h = None if hold[i] is None else int(off[hold[i]])
            else:
                s = gs.STORE_RECORD if typ[i] in gs.STORE_TYPES else gs.UNKNOWN
        out.append((int(off[i]), int(typ[i]), s, h))
    return out, dict(stop=cut_status or stop, end_offset=int(off[cut]) if cut_status else int(end3[0]))


def check_agree(emul, store):
    want, ws = gs.audit(store)
    got, s = emul_audit(emul, store)
    assert got == want
    assert (s["stop"], s["end_offset"]) == (ws["stop"], ws["end_offset"])
    return want, ws


# ---- crafted records (no valid signatures: the host build does not verify) ------------------------------------------
N1, N2, N3, N4 = (bytes([2]) + bytes([k]) * 32 for k in (1, 2, 3, 4))


def ca(scid, n1=N1, n2=N2, extra=b""):
    return b"\x01\x00" + bytes(256) + b"\x00\x00" + CHAIN + scid + n1 + n2 + N3 + N4 + extra


def cu(scid, direction=0):
    return b"\x01\x02" + bytes(64) + CHAIN + scid + bytes(4) + b"\x01" + bytes([direction]) + bytes(26)


def amount():
    return struct.pack(">HQ", gs.CHANNEL_AMOUNT, 1000)


def delete(scid):
    return struct.pack(">H", gs.DELETE_CHAN) + scid


def store_of(*recs, version=16):
    return bytes([version]) + b"".join(recs)


A, B = b"\x00\x00\x01\x00\x00\x02\x00\x01", b"\x00\x00\x01\x00\x00\x03\x00\x01"


def test_fixture_matches_description():
    store = load_fixture()
    j = json.load(open(os.path.join(GOLD, "gossip_store_subset.json")))
    recs, end, stop, no_amount = gs.walk(store)
    assert (len(recs), len(store), end, stop, no_amount) == (j["records"], j["bytes"], len(store), gs.EOF, None)
    assert (len(recs), len(store)) == (4600, 974526)
    # the messages are those of gossip_subset.bin, in the same order
    from tests import gossip
    msgs = [store[o + 12:o + 12 + n] for o, t, n, _ in recs if t in (256, 257, 258)]
    assert msgs == gossip.load_subset()
    out, s = gs.audit(store)
    assert all(st in (0, gs.STORE_RECORD) for _, _, st, _ in out)
    assert sum(t == 258 and h is not None for _, t, _, h in out) == 1200
    assert s["redundant_announcements"] == 0 and s["updates_without_channel"] == 0


def test_every_fixture_crc_equals_clns(emul):
    """the header checksum CLN wrote for each of the 4,600 records, recomputed by the host build and by the model"""
    emul.emul_gs_crc32c.restype = ctypes.c_uint32
    emul.emul_gs_crc32c.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32]
    store = load_fixture()
    recs, _, _, _ = gs.walk(store)
    for off, _, ln, _ in recs:
        crc, ts = struct.unpack(">II", store[off + 4:off + 12])
        msg = store[off + 12:off + 12 + ln]
        assert emul.emul_gs_crc32c(ts, msg, ln) == crc, off
        assert gs.crc32c(ts, msg) == crc, off
    # lengths 0..70 against the model: every tail length of the 8-byte slices
    data = bytes(range(200))
    for n in range(71):
        assert emul.emul_gs_crc32c(0xDEADBEEF, data[n:n + n], n) == gs.crc32c(0xDEADBEEF, data[n:n + n])


def test_fixture_walk_and_channels(emul):
    out, s = check_agree(emul, load_fixture())
    assert s["stop"] == gs.EOF and len(out) == 4600


def test_stop_reasons(emul):
    """each of gossmap's stops on a crafted store: where it stops, with which status, and map_end"""
    good = [gs.record(ca(A)), gs.record(amount()), gs.record(cu(A))]
    base = store_of(*good)
    # a flipped message byte: BAD_CRC at that record, nothing after it reached
    st = bytearray(base)
    third = 1 + len(good[0]) + len(good[1])
    st[third + 12 + 70] ^= 1
    out, s = check_agree(emul, bytes(st))
    assert [r[2] for r in out] == [0, gs.STORE_RECORD, gs.BAD_CRC] and s["stop"] == gs.BAD_CRC and s["end_offset"] == third
    # a flipped byte in the first record: every later record is not reached
    st = bytearray(base)
    st[1 + 12 + 300] ^= 0x10
    out, s = check_agree(emul, bytes(st))
    assert [r[2] for r in out] == [gs.BAD_CRC, gs.NOT_REACHED, gs.NOT_REACHED]
    # a cleared COMPLETED bit
    rec = bytearray(good[2])
    rec[0] &= ~(gs.COMPLETED >> 8) & 0xFF
    out, s = check_agree(emul, store_of(good[0], good[1], bytes(rec), gs.record(cu(A))))
    assert [r[2] for r in out] == [0, gs.STORE_RECORD, gs.INCOMPLETE] and s["stop"] == gs.INCOMPLETE
    # a store cut mid-record
    out, s = check_agree(emul, base[:-5])
    assert [r[2] for r in out] == [0, gs.STORE_RECORD, gs.PARTIAL] and s["end_offset"] == third
    # a header cut (fewer than 13 bytes left): the walk simply ends
    out, s = check_agree(emul, base + gs.record(cu(A))[:12])
    assert len(out) == 3 and s["stop"] == gs.EOF and s["end_offset"] == len(base)
    # len < 2
    out, s = check_agree(emul, store_of(*good, gs.record(b"\x01"), gs.record(cu(A))))
    assert [r[2] for r in out][-1] == gs.TRUNCATED and len(out) == 4
    # an ENDED record: the walk stops there, its equivalent_offset reported
    ended = struct.pack(">HQ", gs.ENDED, 123456) + bytes(32)
    out, s = check_agree(emul, store_of(*good, gs.record(ended), gs.record(cu(A))))
    assert [r[2] for r in out][-1] == gs.ST_ENDED and len(out) == 4
    assert gs.audit(store_of(*good, gs.record(ended)))[1]["ended_equivalent_offset"] == 123456
    # an announcement at EOF without room for its amount record
    out, s = check_agree(emul, store_of(*good, gs.record(ca(B))))
    assert [r[2] for r in out][-1] == gs.NO_AMOUNT and s["stop"] == gs.NO_AMOUNT
    # ... unless it is redundant: gossmap finds the channel before it looks for the amount
    out, s = check_agree(emul, store_of(*good, gs.record(ca(A, N2, N3))))
    assert [r[2] for r in out][-1] == 0 and s["stop"] == gs.EOF and out[-1][3] == 1


def test_deleted_record_with_wrong_crc_is_skipped(emul):
    good = [gs.record(ca(A)), gs.record(amount())]
    dead = gs.record(cu(A), flags=gs.COMPLETED | gs.DELETED, crc=12345)
    out, s = check_agree(emul, store_of(*good, dead, gs.record(cu(A))))
    assert [r[2] for r in out] == [0, gs.STORE_RECORD, gs.ST_DELETED, 0] and s["stop"] == gs.EOF


def test_channel_rule(emul):
    """redundant announcements, delete_chan and re-announcement, a deleted announcement, an update before its
    announcement, short records (gossmap reads them on into the records after them), both directions"""
    a1, a2, a3 = ca(A), ca(A, N3, N4), ca(A, N2, N4)
    recs = [gs.record(cu(A)),                        # 0 before any announcement: no channel
            gs.record(a1), gs.record(amount()),      # 1 holds A
            gs.record(a2), gs.record(amount()),      # 3 redundant (holder 1)
            gs.record(cu(A, 1)),                     # 5 -> 1
            gs.record(delete(A)),                    # 6 frees A
            gs.record(cu(A)),                        # 7 no channel
            gs.record(a2, flags=gs.COMPLETED | gs.DELETED), gs.record(amount()),  # 8 deleted: takes no part
            gs.record(cu(A)),                        # 10 still no channel
            gs.record(ca(B)[:300]), gs.record(amount()),  # 11 ends after its scid, still holds B: node ids read on
            gs.record(cu(B)),                        # 13 -> 11
            gs.record(a3), gs.record(amount()),      # 14 holds A again
            gs.record(cu(A, 1)),                     # 16 -> 14
            gs.record(delete(B + b"\x00")),          # 17 a delete of an unknown scid (longer than 10 bytes)
            gs.record(struct.pack(">H", 4102) + bytes(20)),  # 18 obsolete type: unknown
            gs.record(struct.pack(">H", gs.DELETE_CHAN) + b"\x00"),  # 19 short: its scid is read from 20's header
            gs.record(cu(A))]                        # 20 -> 14
    store = store_of(*recs)
    out, s = check_agree(emul, store)
    offs = [r[0] for r in out]
    hold = {i: (None if h is None else offs.index(h)) for i, (_, t, _, h) in enumerate(out) if t in (256, 258)}
    assert hold == {0: None, 1: None, 3: 1, 5: 1, 7: None, 8: None, 10: None, 11: None, 13: 11, 14: None, 16: 14, 20: 14}
    assert out[18][2] == gs.UNKNOWN and out[8][2] == gs.ST_DELETED and out[19][2] == gs.STORE_RECORD
    assert s["stop"] == gs.EOF


def test_major_version():
    with pytest.raises(ValueError):
        gs.audit(bytes([0x20]) + gs.record(cu(A)))
