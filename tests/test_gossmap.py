"""The gossip_store audit against Core Lightning's own gossmap.c.

oracle/gossmap_harness.c loads a store with the reference's common/gossmap.c, unmodified, and reports gossmap's map_end and
its final channel table: (scid, cann_off, cupdate_off[0], cupdate_off[1]) per channel.  Each per-record answer of the
audit -- the Python model (tests/gossip_store.py), the host build of gossip_store.cuh, and on the device
sv_verify_gossip_store_host (tests/test_gpu_gossmap.py) -- is turned into the table gossmap would end with and compared
exactly, together with end_offset == map_end.  On crafted stores every prefix that ends after a channel_update is loaded
as well: gossmap's channel for the update's scid must hold that update under the announcement the audit names as its
holder (or there must be no channel), which checks the holder at every position, not only the final state.

Stores where gossmap does not return (a read past the end of the store asserts in map_copy; an ENDED record sends it
looking for the next store file) leave the comparison; each must be one of those two cases.  The answers are recorded on
this module's `cln` tape (tests/oracle_replay.py) and replayed where the reference is not built.
"""
import ctypes
import os
import struct

import numpy as np
import pytest

from tests import gossip_store as gs
from tests import oracle_replay
from tests.test_gossip_store_host import A, B, N2, N3, N4, amount, ca, cu, delete, emul_audit, load_fixture, store_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap.so")
ABORTED = -2

# cln_gossmap_load(store, len, map_end*, chans* (cap x 4 u64), cap) -> channel count, -1 refused, -2 gossmap did not return
oracle_replay.SPEC.setdefault("cln_gossmap_load", (lambda v: {0: v[1]}, lambda v: {2: 8, 3: 32 * v[4]}, ()))


_ORACLE = []


def oracle():
    """gossmap's cln_gossmap_load, recorded on the calling module's `cln` tape (one instance: it saves every module's)"""
    if not _ORACLE:
        o = oracle_replay.Oracle("cln")
        o.lib = ctypes.CDLL(LIB) if (oracle_replay.RECORD_DIR or os.path.exists(LIB)) else None
        if o.lib is not None:
            o.lib.cln_gossmap_load.restype = ctypes.c_longlong
        _ORACLE.append(o)
    return _ORACLE[0]


def gossmap_load(o, store):
    """-> (map_end, [(scid, cann_off, cupdate_off[0], cupdate_off[1])] sorted by cann_off), or None if gossmap did not
    return"""
    cap = sum(t == 256 for _, t, _, _ in gs.walk(store)[0]) + 1 if store[0] >> 5 == 0 else 1
    end = np.zeros(1, np.uint64)
    rows = np.zeros((cap, 4), np.uint64)
    p64 = ctypes.POINTER(ctypes.c_uint64)  # typed pointers: their addresses stay out of the tape's digest
    n = int(o.cln_gossmap_load(bytes(store), ctypes.c_size_t(len(store)), end.ctypes.data_as(p64), rows.ctypes.data_as(p64),
                               ctypes.c_size_t(cap)))
    assert (0 <= n <= cap) or n == ABORTED, n  # -1: refused (major version, never sent here); -3: no temporary file
    if n == ABORTED:
        return None
    return int(end[0]), [tuple(int(x) for x in r) for r in rows[:n]]


# ---- what gossmap reads, and the table it ends with -------------------------------------------------------------------
def reads_past_end(store, off, typ):
    """gossmap's reads of the record at header offset off would pass the end of the store (map_copy asserts)"""
    p, n = off + gs.HDR, len(store)
    if typ == 256:
        r = gs.ann_read(store, p)
        return r is None or p + r > n
    if typ == 258:
        return p + gs.UPD_READ > n
    if typ == gs.DELETE_CHAN:
        return p + gs.DEL_READ > n
    if typ == 257:  # node_announcement (:650-668): features length, then the node id after features and timestamp
        return p + 68 > n or p + 68 + struct.unpack(">H", store[p + 66:p + 68])[0] + 4 + 33 > n
    return False


def gossmap_aborts(store, out):
    """from a per-record answer: gossmap reaches a record it reads past the end of the store, or an ENDED record"""
    for off, typ, st, _ in out:
        if st == gs.ST_ENDED:
            return True
        if (st < 16 or st in (gs.STORE_RECORD, gs.NO_AMOUNT)) and reads_past_end(store, off, typ):
            return True
    return False


def table_of(store, out):
    """gossmap's final channel table from a per-record answer (off, type, status, holder): an announcement reached with
    no holder opens its channel, a reached delete_chan of the scid frees it, a reached update with a holder is the
    channel's update for its direction (channel_flags & 1)"""
    chans = {}
    for off, typ, st, h in out:
        p = off + gs.HDR
        if typ == 256 and st < 16 and h is None:
            chans[gs.ann_fields(store, p)[1]] = [p, 0, 0]
        elif typ == gs.DELETE_CHAN and st == gs.STORE_RECORD:
            chans.pop(store[p + 2:p + 10], None)
        elif typ == 258 and st < 16 and h is not None:
            c = chans[store[p + 98:p + 106]]
            assert c[0] == h + gs.HDR, (off, h)  # an update's holder is the channel its scid holds
            c[1 + (store[p + 111] & 1)] = p
    return sorted(((int.from_bytes(s, "big"), *c) for s, c in chans.items()), key=lambda r: r[1])


class Tally:
    def __init__(self):
        self.stores = self.records = self.positions = self.aborted = self.prefix_aborted = 0

    def report(self, what):
        print(f"\n{what} vs gossmap: {self.stores} stores, {self.records} records, {self.positions} per-position updates "
              f"compared; gossmap did not return on {self.aborted} stores and {self.prefix_aborted} prefixes")


def compare(o, store, answer, tally, prefixes=False):
    """answer(store) -> (per-record list, summary with end_offset) against gossmap, final table and (crafted stores)
    every prefix that ends after a reached channel_update"""
    out, s = answer(store)
    ref = gossmap_load(o, store)
    if ref is None:
        assert gossmap_aborts(store, out), "gossmap did not return on a store it reads inside"
        tally.aborted += 1
        return out, None
    assert not gossmap_aborts(store, out)
    end, table = ref
    assert s["end_offset"] == end
    assert table_of(store, out) == table
    tally.stores += 1
    tally.records += len(out)
    if prefixes:
        for off, typ, st, h in out:
            if typ != 258 or st >= 16:
                continue
            p = off + gs.HDR
            cut = store[:p + struct.unpack(">H", store[off + 2:off + 4])[0]]
            r = gossmap_load(o, cut)
            if r is None:
                tally.prefix_aborted += 1
                continue
            if r[0] != len(cut):  # gossmap stopped before the update (an announcement without room for its amount)
                continue
            scid = int.from_bytes(store[p + 98:p + 106], "big")
            chan = [c for c in r[1] if c[0] == scid]
            if h is None:
                assert chan == [], off
            else:
                assert len(chan) == 1 and chan[0][1] == h + gs.HDR and chan[0][2 + (store[p + 111] & 1)] == p, off
            tally.positions += 1
    return out, table


# ---- stores ---------------------------------------------------------------------------------------------------------
C = b"\x00\x00\x01\x00\x00\x04\x00\x01"
AMT = gs.record(amount())
# a scid whose 8 bytes are those of a deleted record's header (flags COMPLETED|DELETED, len 10, crc field 0x11223344):
# a 2-byte delete_chan right before that record has gossmap read this scid from the header
HDR_SCID = struct.pack(">HHI", gs.COMPLETED | gs.DELETED, 10, 0x11223344)


def tail(n=70):
    """updates of an scid no announcement holds: store bytes for short records to read on into"""
    return [gs.record(cu(C, k & 1)) for k in range(n)]


def issue_store():
    """an announcement cut after its scid, then its update, then the full announcement of the same scid: gossmap reads the
    short one's node ids from the records after it, so it holds the channel and the full one is redundant"""
    return store_of(gs.record(ca(A)), AMT, gs.record(ca(B)[:300]), AMT, gs.record(cu(B, 0)), gs.record(ca(B)), AMT,
                    gs.record(cu(B, 1)))


def stop_reason_stores():
    """the stores of test_gossip_store_host.test_stop_reasons"""
    good = [gs.record(ca(A)), gs.record(amount()), gs.record(cu(A))]
    base = store_of(*good)
    third = 1 + len(good[0]) + len(good[1])
    out = []
    st = bytearray(base)
    st[third + 12 + 70] ^= 1
    out.append(bytes(st))
    st = bytearray(base)
    st[1 + 12 + 300] ^= 0x10
    out.append(bytes(st))
    rec = bytearray(good[2])
    rec[0] &= ~(gs.COMPLETED >> 8) & 0xFF
    out.append(store_of(good[0], good[1], bytes(rec), gs.record(cu(A))))
    out.append(base[:-5])
    out.append(base + gs.record(cu(A))[:12])
    out.append(store_of(*good, gs.record(b"\x01"), gs.record(cu(A))))
    ended = struct.pack(">HQ", gs.ENDED, 123456) + bytes(32)
    out.append(store_of(*good, gs.record(ended), gs.record(cu(A))))
    out.append(store_of(*good, gs.record(ended)))
    out.append(store_of(*good, gs.record(ca(B))))
    out.append(store_of(*good, gs.record(ca(A, N2, N3))))
    dead = gs.record(cu(A), flags=gs.COMPLETED | gs.DELETED, crc=12345)
    out.append(store_of(good[0], good[1], dead, gs.record(cu(A))))
    return out


def channel_rule_store():
    """the store of test_gossip_store_host.test_channel_rule"""
    a1, a2, a3 = ca(A), ca(A, N3, N4), ca(A, N2, N4)
    return store_of(gs.record(cu(A)), gs.record(a1), AMT, gs.record(a2), AMT, gs.record(cu(A, 1)), gs.record(delete(A)),
                    gs.record(cu(A)), gs.record(a2, flags=gs.COMPLETED | gs.DELETED), AMT, gs.record(cu(A)),
                    gs.record(ca(B)[:300]), AMT, gs.record(cu(B)), gs.record(a3), AMT, gs.record(cu(A, 1)),
                    gs.record(delete(B + b"\x00")), gs.record(struct.pack(">H", 4102) + bytes(20)),
                    gs.record(struct.pack(">H", gs.DELETE_CHAN) + b"\x00"), gs.record(cu(A)))


def short_announcement_stores():
    """announcements of B cut at every boundary add_channel reads: the features length (258-260), inside and after 4
    feature bytes, after the chain hash, the scid, node_id_1 and node_id_2; each with and without store bytes after it
    for the reads to run into"""
    feat = struct.pack(">H", 4) + b"\x00\x00\x02\x02"
    full = ca(B)[:258] + feat + ca(B)[260:]
    out = []
    for k in (258, 259, 260, 262, 264, 266, 298, 306, 339, 372):
        m = full[:k]
        body = [gs.record(ca(A)), AMT, gs.record(m), AMT, gs.record(cu(B, 0)), gs.record(cu(B, 1)), gs.record(ca(B)), AMT,
                gs.record(cu(B, 0))]
        out.append(store_of(*body, *tail()))
        out.append(store_of(*body))
    for k in (258, 259, 260, 292, 300, 333, 366):  # no features
        out.append(store_of(gs.record(ca(A)), AMT, gs.record(ca(B)[:k]), AMT, gs.record(cu(B, 1)), gs.record(cu(A, 0)),
                            *tail()))
    return out


def short_update_stores():
    """updates of 100-138 bytes (gossmap reads through byte 138 of every update), and two at the very end of a store"""
    out = []
    for k in range(100, 139):
        out.append(store_of(gs.record(ca(A)), AMT, gs.record(cu(A, k & 1)[:k]), gs.record(cu(A, 1)), gs.record(cu(C)),
                            gs.record(cu(A)[:k]), gs.record(cu(C))))
    for k in (111, 137):
        out.append(store_of(gs.record(ca(A)), AMT, gs.record(cu(A)), gs.record(cu(A, 1)[:k])))
    return out


def short_delete_stores():
    """delete_chan of 2-10 bytes (gossmap reads 8 scid bytes at +2 of every one), and one whose scid is the header of
    the record after it, which equals a live channel's scid"""
    out = []
    for k in range(2, 11):
        out.append(store_of(gs.record(ca(A)), AMT, gs.record(delete(A)[:k]), gs.record(cu(A)), gs.record(cu(A, 1))))
    dead = gs.record(bytes(10), flags=gs.COMPLETED | gs.DELETED, crc=0x11223344)
    out.append(store_of(gs.record(ca(HDR_SCID)), AMT, gs.record(cu(HDR_SCID)), gs.record(delete(A)[:2]), dead,
                        gs.record(cu(HDR_SCID, 1)), gs.record(ca(HDR_SCID, N3, N4)), AMT, gs.record(cu(HDR_SCID))))
    return out


def crafted_stores():
    return ([issue_store(), channel_rule_store()] + stop_reason_stores() + short_announcement_stores() +
            short_update_stores() + short_delete_stores())


def mutation_base():
    """the fixture's first 40 channels: their announcements, amount records and updates, with the node_announcements
    among them, in store order"""
    fx = load_fixture()
    recs = gs.walk(fx)[0]
    scids = [gs.ann_fields(fx, o + 12)[1] for o, t, _, _ in recs if t == 256][:40]
    keep, last_ann = [], None
    for i, (o, t, n, _) in enumerate(recs):
        m = fx[o + 12:o + 12 + n]
        if (t == 256 and gs.ann_fields(m)[1] in scids) or (t == 258 and m[98:106] in scids):
            keep.append(i)
            last_ann = i if t == 256 else last_ann
        elif t == gs.CHANNEL_AMOUNT and last_ann == i - 1:
            keep.append(i)
        elif t == 257 and len(keep) < 120:
            keep.append(i)
    return fx[:1] + b"".join(fx[recs[i][0]:recs[i][0] + 12 + recs[i][2]] for i in keep)


def mutations(n=240, seed=4242):
    """seeded mutations of mutation_base(): COMPLETED/DELETED bits, msglen (with and without a matching checksum), a
    checksum byte, a cut, a duplicated or swapped record, an inserted delete_chan of a live scid"""
    base = mutation_base()
    recs = gs.walk(base)[0]
    raw = [bytearray(base[o:o + 12 + n]) for o, _, n, _ in recs]
    scids = [gs.ann_fields(base, o + 12)[1] for o, t, _, _ in recs if t == 256]
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        rs = [bytearray(r) for r in raw]
        kind = k % 9
        i = int(rng.integers(len(rs)))
        if kind == 0:
            rs[i][0] &= ~(gs.COMPLETED >> 8) & 0xFF
        elif kind == 1:
            rs[i][0] |= gs.DELETED >> 8
        elif kind == 2:  # a deleted record made live again (its checksum still the written one)
            rs[i][0] |= gs.DELETED >> 8
            rs[int(rng.integers(len(rs)))][0] &= ~(gs.DELETED >> 8) & 0xFF
        elif kind in (3, 4):  # msglen altered; with kind 4 the checksum recomputed over the new length
            ln = struct.unpack(">H", rs[i][2:4])[0]
            new = max(0, ln + int(rng.integers(-200, 60)))
            struct.pack_into(">H", rs[i], 2, new)
            if kind == 4:
                flat = b"".join(rs)
                at = sum(len(r) for r in rs[:i]) + 12
                struct.pack_into(">I", rs[i], 4, gs.crc32c(struct.unpack(">I", rs[i][8:12])[0], flat[at:at + new]))
        elif kind == 5:
            rs[i][4 + int(rng.integers(4))] ^= 1 << int(rng.integers(8))
        elif kind == 6:
            j = int(rng.integers(len(rs)))
            rs.insert(j, bytearray(rs[i]))
        elif kind == 7:
            j = int(rng.integers(len(rs)))
            rs[i], rs[j] = rs[j], rs[i]
        else:
            rs.insert(i, bytearray(gs.record(delete(scids[int(rng.integers(len(scids)))]))))
        st = base[:1] + b"".join(rs)
        if k % 5 == 4:  # and every fifth also cut at a random offset
            st = st[:int(rng.integers(2, len(st)))]
        out.append(st)
    return out


def model_answer(store):
    return gs.audit(store)


def test_issue_store_layout():
    """the short-announcement store has the record offsets the rule was found at"""
    recs = gs.walk(issue_store())[0]
    assert [r[0] for r in recs] == [1, 445, 467, 779, 801, 951, 1395, 1417]


@pytest.mark.parametrize("who", ["model", "host_build"])
def test_crafted_vs_gossmap(who, request):
    o = oracle()
    answer = model_answer if who == "model" else (lambda st, e=request.getfixturevalue("emul"): emul_audit(e, st))
    t = Tally()
    stores = crafted_stores()
    for st in stores:
        compare(o, st, answer, t, prefixes=True)
    t.report(who)
    # the issue store: the short announcement at 467 holds B, 801 and 1417 belong to it, 951 is redundant
    out, table = compare(o, issue_store(), answer, Tally())
    hold = {off: h for off, _, _, h in out}
    assert (hold[467], hold[801], hold[951], hold[1417]) == (None, 467, 467, 467)
    assert table == [(int.from_bytes(A, "big"), 13, 0, 0), (int.from_bytes(B, "big"), 479, 813, 1429)]
    assert t.aborted <= len(stores) // 5 and t.stores == len(stores) - t.aborted
    assert t.positions >= 150


@pytest.mark.parametrize("who", ["model", "host_build"])
def test_fixture_and_mutations_vs_gossmap(who, request):
    o = oracle()
    answer = model_answer if who == "model" else (lambda st, e=request.getfixturevalue("emul"): emul_audit(e, st))
    t = Tally()
    out, table = compare(o, load_fixture(), answer, t)
    assert len(table) == 1500 and sum(c[2] != 0 or c[3] != 0 for c in table) > 0
    muts = mutations()
    for st in muts:
        compare(o, st, answer, t)
    t.report(who)
    assert t.stores >= 200 and t.aborted <= len(muts) // 10


def test_tiled_x53_vs_gossmap(emul):
    """the fixture tiled x53 (every copy after the first redundant): the host build against gossmap"""
    fx = load_fixture()
    t = Tally()
    _, table = compare(oracle(), fx[:1] + fx[1:] * 53, lambda st: emul_audit(emul, st), t)
    assert len(table) == 1500 and t.stores == 1
