"""The prune model (tests/gossip_store_prune.py) on crafted stores, checked against Core Lightning's own gossmap.c loaded
the way gossipd loads its store at start-up (oracle/gossmap_strict_harness.c cln_gossmap_load_strict: expected_len = the
store's length, so a bad checksum, a truncated record, a redundant announcement, an unknown record type or a walk that
stops short of the end refuses the whole store).

The crafted messages carry no real signatures; a stand-in sigcheck judges them: an announcement fails when its first
signature byte is 0xBB, and an update verifies only under the node whose 33 bytes open its signature.  The real
signatures are the GPU test's (tests/test_gpu_gossip_store_prune.py)."""
import ctypes
import os
import struct

import numpy as np
import pytest

from tests import gossip_store as gs
from tests import gossip_store_prune as gp
from tests import oracle_replay
from tests.test_gossip_store_host import CHAIN, A, B, N1, N2, N3, N4, amount, ca, delete, load_fixture, store_of
from tests.test_gossmap import table_of

# cln_gossmap_load_strict(store, len, map_end*, chans*, cap, nodes*, ncap, n_nodes*) -> channel count, -1 refused,
# -2 gossmap did not return
oracle_replay.SPEC.setdefault("cln_gossmap_load_strict", (lambda v: {0: v[1]},
                                                          lambda v: {2: 8, 3: 32 * v[4], 5: 8 * v[6], 7: 8}, ()))
BAD = 0xBB
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRICT = os.path.join(ROOT, "oracle", "_ref", "libcln_gossmap_strict.so")
_O = []


def oracle():
    """gossmap's strict load, recorded on the calling module's `cln` tape"""
    if not _O:
        o = oracle_replay.Oracle("cln")
        o.lib = ctypes.CDLL(STRICT) if (oracle_replay.RECORD_DIR or os.path.exists(STRICT)) else None
        _O.append(o)
    return _O[0]


def strict_load(o, store):
    """-> (map_end, channel rows as cln_gossmap_load's, sorted nann_off of every node), or None if the strict load
    refuses the store"""
    recs = gs.walk(store)[0]
    cap = sum(t == 256 for _, t, _, _ in recs) + 1
    ncap = 2 * cap + sum(t == 257 for _, t, _, _ in recs)
    end, nn = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    rows, nodes = np.zeros((cap, 4), np.uint64), np.zeros(ncap, np.uint64)
    p64 = ctypes.POINTER(ctypes.c_uint64)
    if o.lib is not None:
        o.lib.cln_gossmap_load_strict.restype = ctypes.c_longlong
    n = int(o.cln_gossmap_load_strict(bytes(store), ctypes.c_size_t(len(store)), end.ctypes.data_as(p64),
                                      rows.ctypes.data_as(p64), ctypes.c_size_t(cap), nodes.ctypes.data_as(p64),
                                      ctypes.c_size_t(ncap), nn.ctypes.data_as(p64)))
    assert n >= -2 and n <= cap and int(nn[0]) <= ncap, n
    if n < 0:
        return None
    return int(end[0]), [tuple(int(x) for x in r) for r in rows[:n]], [int(x) for x in nodes[:int(nn[0])]]


def fake_sigcheck(m, signer):
    """stand-in for gossipd's sigcheck (see the module docstring), with the audit's -1 and -2"""
    t = struct.unpack(">H", m[:2])[0]
    if t == 256:
        if len(m) < 260 or len(m) < 260 + struct.unpack(">H", m[258:260])[0] + 40 + 132:
            return -1
        return 1 if m[2] == BAD else 0
    if t == 257:
        return -1 if len(m) < 140 else (1 if m[2] == BAD else 0)
    if len(m) < 138:
        return -1
    if signer is None:
        return -2
    return 0 if m[2:35] == bytes(signer) else 1


def ann(scid, n1=N1, n2=N2, bad=False):
    m = bytearray(ca(scid, n1, n2))
    if bad:
        m[2] = BAD
    return gs.record(bytes(m)) + gs.record(amount())


def upd(scid, signer, direction=0, ts=1):
    """a channel_update that verifies under `signer` only"""
    m = b"\x01\x02" + signer + bytes(31) + CHAIN + scid + struct.pack(">I", ts) + b"\x01" + bytes([direction]) + bytes(26)
    return gs.record(m, ts=ts)


def nann(node, bad=False, ts=1):
    m = bytearray(b"\x01\x01" + bytes(64) + b"\x00\x00" + struct.pack(">I", ts) + node + bytes(35) + b"\x00\x00")
    if bad:
        m[2] = BAD
    return gs.record(bytes(m), ts=ts)


def reasons(store):
    return [w for _, _, _, w in gp.prune(store, fake_sigcheck)[1]]


def check_pruned(o, store):
    """prune, then: only flag bits changed, the audit of the result is clean, pruning it again deletes nothing, and the
    strict load of gossmap.c accepts it with the model's channel table and current node_announcements"""
    out, rows, s = gp.prune(store, fake_sigcheck)
    assert len(out) == len(store)
    assert all(a == b or (off < len(store) and a ^ b == 0x80) for off, (a, b) in enumerate(zip(out, store)))
    assert sum(w != gp.GP_KEPT for _, _, _, w in rows) == s["pruned"] == sum(a != b for a, b in zip(out, store))
    answer, a = gs.audit(out, fake_sigcheck)
    assert a["stop"] == gs.EOF and a["redundant_announcements"] == 0
    assert all(st in (0, gs.ST_DELETED, gs.STORE_RECORD) for _, _, st, _ in answer), answer
    again, _, s2 = gp.prune(out, fake_sigcheck)
    assert again == out and s2["pruned"] == 0
    ref = strict_load(o, out)
    assert ref is not None, "gossmap's strict load refused the pruned store"
    end, chans, nodes = ref
    assert end == len(out)
    assert chans == table_of(out, answer)
    kept_nann = {off + gs.HDR for off, t, st, _ in answer if t == 257 and st == 0}
    assert all(n == 0 or n in kept_nann for n in nodes)
    return out, rows, s, nodes


def test_strict_load_refuses_what_prune_deletes():
    """the strict load refuses each store below before pruning and accepts it after"""
    o = oracle()
    x = ann(B, N3, N4)
    bad_crc = bytearray(store_of(ann(A), x, upd(A, N1)))
    bad_crc[1 + len(ann(A)) + 12 + 5] ^= 1
    cases = [store_of(ann(A), ann(A, N3, N4), upd(A, N1)),                         # redundant announcement
             store_of(ann(A), gs.record(struct.pack(">HI", 4999, 7)), upd(A, N1)),  # unknown record type
             bytes(bad_crc),                                                       # bad checksum mid-store
             store_of(ann(A), gs.record(b"\x01"), upd(A, N1))]                     # truncated record mid-store
    for st in cases:
        assert strict_load(o, st) is None
        check_pruned(o, st)
    assert reasons(cases[0]) == [0, 0, gp.GP_REDUNDANT, gp.GP_AMOUNT, 0]
    assert reasons(cases[1]) == [0, 0, gp.GP_UNKNOWN, 0]
    assert reasons(cases[2]) == [0, 0, gp.GP_BAD_CRC, gp.GP_AMOUNT, 0]
    assert reasons(cases[3]) == [0, 0, gp.GP_TRUNCATED, 0]


def test_bad_holder_hands_over_to_the_redundant_announcement():
    """a failing announcement holding the scid, a good redundant one after it, updates before and after: the second
    takes the channel, updates before it lose their channel, updates after it are verified again under its nodes"""
    o = oracle()
    st = store_of(ann(A, bad=True), upd(A, N1), upd(A, N3), ann(A, N3, N4), upd(A, N1, ts=2), upd(A, N3, ts=2),
                  upd(A, N4, 1, ts=2))
    out, rows, s, _ = check_pruned(o, st)
    assert [w for _, _, _, w in rows] == [gp.GP_MESSAGE, gp.GP_AMOUNT, gp.GP_NO_CHANNEL, gp.GP_NO_CHANNEL, 0, 0,
                                          gp.GP_SIGNATURE, 0, 0]
    assert s["reverified"] == 3 and s["message"] == 1 and s["signature"] == 1 and s["no_channel"] == 2


def test_newest_bad_update_and_node_announcement():
    """deleting a bad newest update or node_announcement makes the previous good one current"""
    o = oracle()
    st = store_of(ann(A), nann(N1), upd(A, N1, ts=1), upd(A, N3, ts=2), nann(N1, bad=True, ts=2))
    out, rows, s, nodes = check_pruned(o, st)
    assert [w for _, _, _, w in rows] == [0, 0, 0, 0, gp.GP_SIGNATURE, gp.GP_MESSAGE]
    _, chans, _ = strict_load(o, out)
    assert chans[0][2] == rows[3][0] + gs.HDR                       # the first update is the channel's again
    assert rows[2][0] + gs.HDR in nodes                             # and the first node_announcement is current


def test_delete_chan_and_malformed():
    """an update of a channel a delete_chan removed goes; a malformed announcement goes with its amount; a node
    announcement of a node without channels stays"""
    o = oracle()
    st = store_of(ann(A), upd(A, N1), gs.record(delete(A)), upd(A, N1, ts=2), gs.record(ca(B)[:-40]) +
                  gs.record(amount()), nann(N4), ann(B, N3, N4), upd(B, N3))
    _, rows, s, _ = check_pruned(o, st)
    assert [w for _, _, _, w in rows] == [0, 0, 0, 0, gp.GP_NO_CHANNEL, gp.GP_MESSAGE, gp.GP_AMOUNT, 0, 0, 0, 0]


def test_clean_fixture_untouched():
    store = load_fixture()
    out, rows, s = gp.prune(store)
    assert out == store and s["pruned"] == 0 and s["records"] == 4600 and s["stop"] == gs.EOF


@pytest.mark.parametrize("version", [16, 0x1F])
def test_walk_matches_audit_without_truncated(version):
    """on a store without truncated records the prune's walk is the audit's"""
    st = store_of(ann(A), upd(A, N1), version=version)
    assert [r[:3] for r in gp.prune(st, fake_sigcheck)[1]] == [r[:3] for r in gs.audit(st, fake_sigcheck)[0]]
