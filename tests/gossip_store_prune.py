"""Python model of sv_prune_gossip_store_host: which records of a gossip_store to mark deleted so that gossipd's strict
load (common/gossmap.c with expected_len, :1428-1438) accepts the store and keeps every record that verifies.  Built on
the audit's model (tests/gossip_store.py); the rules are those of include/cln_sigverify.h."""
import struct

from tests.gossip_store import (
    BAD_CRC, CHAN_DYING, CHANNEL_AMOUNT, COMPLETED, DEL_READ, DELETE_CHAN, DELETED, ENDED, EOF, HDR, INCOMPLETE,
    NO_AMOUNT, NOT_REACHED, PARTIAL, ST_DELETED, ST_ENDED, STORE_RECORD, TRUNCATED, UNKNOWN, UPD_READ, UUID, ann_fields,
    ann_ok, crc_ok)

# reasons (include/cln_sigverify.h SV_GP_*; 0 = kept)
GP_KEPT, GP_BAD_CRC, GP_TRUNCATED, GP_MESSAGE, GP_REDUNDANT, GP_NO_CHANNEL, GP_SIGNATURE, GP_AMOUNT, GP_UNKNOWN = range(9)
STORE_TYPES = (CHANNEL_AMOUNT, DELETE_CHAN, CHAN_DYING, UUID)


def walk(store):
    """the prune's header walk: map_catchup's (tests/gossip_store.py walk), except that a TRUNCATED record does not stop
    it -> (records [(off, type, len, status)], map_end, stop, no_amount entry or None)"""
    recs, off, stop, no_amount = [], 1, EOF, None
    while off + HDR < len(store):
        flags, ln = struct.unpack(">HH", store[off:off + 4])
        typ = struct.unpack(">H", store[off + HDR:off + HDR + 2])[0] if off + HDR + 2 <= len(store) else 0
        st = 0
        if not flags & COMPLETED:
            st = INCOMPLETE
        elif flags & DELETED:
            st = ST_DELETED
        elif off + HDR + ln > len(store):
            st = PARTIAL
        elif ln < 2:
            st = TRUNCATED
        elif typ == ENDED:
            st = ST_ENDED
        if st == 0 and typ == 256 and no_amount is None and off + HDR + ln + HDR + 2 + 8 > len(store):
            no_amount = len(recs)
        recs.append((off, typ, ln, st))
        if st not in (0, ST_DELETED, TRUNCATED):
            stop = st
            break
        off += HDR + ln
    return recs, off, stop, no_amount


def holders(store, recs, live):
    """the channel table over the records `live` (indices, store order): {entry: the entry of the announcement its event
    saw, or None} for announcements and updates whose reads stay inside the store"""
    held, holder = {}, {}
    for i in live:
        off, typ = recs[i][0], recs[i][1]
        p = off + HDR
        if typ == 256 and ann_ok(store, p):
            scid = ann_fields(store, p)[1]
            holder[i] = held.get(scid)
            held.setdefault(scid, i)
        elif typ == DELETE_CHAN and p + DEL_READ <= len(store):
            held.pop(store[p + 2:p + 10], None)
        elif typ == 258 and p + UPD_READ <= len(store):
            holder[i] = held.get(store[p + 98:p + 106])
    return holder


def prune(store, sigcheck=None):
    """-> (pruned store bytes, [(off, type, first-round status, reason)], summary dict).  sigcheck(msg, signer33 or None)
    gives a message's status as for tests/gossip_store.py audit(); None leaves every message status 0."""
    if store[0] >> 5:
        raise ValueError("major version")
    recs, end, stop, no_amount = walk(store)
    bad = {i for i, (off, typ, ln, st) in enumerate(recs) if st == 0 and not crc_ok(store, off)}
    live = [i for i, r in enumerate(recs) if r[3] == 0 and i not in bad]

    def signer(i, h):
        return None if h is None else ann_fields(store, recs[h][0] + HDR)[2 + (store[recs[i][0] + HDR + 111] & 1)]

    def check(i, h):
        off, ln = recs[i][0], recs[i][2]
        return sigcheck(store[off + HDR:off + HDR + ln], signer(i, h)) if sigcheck else 0

    # first round: the audit's statuses over the records with good checksums
    h1 = holders(store, recs, live)
    status = {i: check(i, h1.get(i)) for i in live if recs[i][1] in (256, 257, 258)}
    reason = {i: GP_TRUNCATED for i, r in enumerate(recs) if r[3] == TRUNCATED}
    reason.update({i: GP_BAD_CRC for i in bad})
    for i, st in status.items():
        if (st in (-1, -3)) if recs[i][1] == 258 else st != 0:
            reason[i] = GP_MESSAGE
    # second round: the table without the deleted announcements
    h2 = holders(store, recs, [i for i in live if not (recs[i][1] == 256 and i in reason)])
    reverified = 0
    for i in live:
        typ = recs[i][1]
        if i in reason:
            continue
        if typ == 256:
            if h2.get(i) is not None:
                reason[i] = GP_REDUNDANT
        elif typ == 258:
            h = h2.get(i)
            if h is None:
                reason[i] = GP_NO_CHANNEL
            elif h != h1.get(i):
                reverified += 1
                if check(i, h) != 0:
                    reason[i] = GP_SIGNATURE
            elif status[i] != 0:
                reason[i] = GP_SIGNATURE
        elif typ not in (257,) + STORE_TYPES:
            reason[i] = GP_UNKNOWN
    # the amount record right after a deleted announcement goes with it
    for i in range(1, len(recs)):
        if recs[i][3] == 0 and i not in reason and recs[i][1] == CHANNEL_AMOUNT and recs[i - 1][1] == 256 and i - 1 in reason:
            reason[i] = GP_AMOUNT
    # an announcement kept without room for its amount record stops the walk
    cut = no_amount if no_amount is not None and no_amount not in reason else len(recs)
    out = bytearray(store)
    rows = []
    for i, (off, typ, ln, st) in enumerate(recs):
        if i >= cut:
            st = NO_AMOUNT if i == cut else NOT_REACHED
        elif st == 0:
            st = BAD_CRC if i in bad else status[i] if i in status else (STORE_RECORD if typ in STORE_TYPES else UNKNOWN)
        why = reason.get(i, GP_KEPT) if i < cut else GP_KEPT
        if why:
            out[off] |= DELETED >> 8
        rows.append((off, typ, st, why))
    whys = [w for _, _, _, w in rows]
    s = dict(version=store[0], stop=NO_AMOUNT if cut < len(recs) else stop,
             end_offset=recs[cut][0] if cut < len(recs) else end, records=len(recs),
             pruned=sum(w != GP_KEPT for w in whys), reverified=reverified)
    for k, name in enumerate(("bad_crc", "truncated", "message", "redundant", "no_channel", "signature", "amount",
                              "unknown"), 1):
        s[name] = whys.count(k)
    return bytes(out), rows, s
