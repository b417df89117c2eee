"""Python model of how gossmap loads a gossip_store (common/gossmap.c, reference): map_catchup's record walk and
checksums (:815-937), and the channel table that decides which announcement signs each channel_update (add_channel
:440-500, remove_channel_by_deletemsg :612-626).  sv_verify_gossip_store_host must agree with it record for record, and
tests/test_gossmap.py checks both against gossmap.c itself."""
import os
import struct

HDR = 12
COMPLETED, DELETED = 0x2000, 0x8000
CHANNEL_AMOUNT, DELETE_CHAN, ENDED, CHAN_DYING, UUID = 4101, 4103, 4105, 4106, 4107
# record statuses besides the signature statuses (include/cln_sigverify.h SV_GS_*)
EOF, ST_DELETED, STORE_RECORD, UNKNOWN, NOT_REACHED = 0, 16, 17, 18, 19
INCOMPLETE, PARTIAL, TRUNCATED, BAD_CRC, ST_ENDED, NO_AMOUNT = 32, 33, 34, 35, 36, 37
STORE_TYPES = (CHANNEL_AMOUNT, DELETE_CHAN, CHAN_DYING, UUID)  # the store's own records: status STORE_RECORD
NONE = None


def load_fixture():
    """the committed store fixture (tests/golden/gossip_store_subset.bin)"""
    return open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gossip_store_subset.bin"), "rb").read()


def _table():
    t = []
    for i in range(256):
        c = i
        for _ in range(8):
            c = (c >> 1) ^ (0x82F63B78 if c & 1 else 0)
        t.append(c)
    return t


_T = _table()


def crc32c(start, data):
    """ccan's crc32c(start_crc, data, len): CRC-32C, reflected, inverted on entry and exit"""
    c = start ^ 0xFFFFFFFF
    for b in data:
        c = (c >> 8) ^ _T[(c ^ b) & 0xFF]
    return c ^ 0xFFFFFFFF


def record(msg, ts=0, flags=COMPLETED, crc=None):
    """one store record: be16 flags, be16 len, be32 crc, be32 timestamp, message"""
    return struct.pack(">HHII", flags, len(msg), crc32c(ts, msg) if crc is None else crc, ts) + msg


def walk(store, truncated_stops=True):
    """map_catchup's header walk -> (records [(off, type, len, status)], map_end, stop, no_amount entry or None);
    status 0 = live, to be judged by checksum and content.  The prune's walk (truncated_stops=False) steps over a
    TRUNCATED record instead of stopping at it."""
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
        if st not in (0, ST_DELETED) and (truncated_stops or st != TRUNCATED):
            stop = st
            break
        off += HDR + ln
    return recs, off, stop, no_amount


def crc_ok(store, off):
    ln, crc, ts = struct.unpack(">HII", store[off + 2:off + 12])
    return crc32c(ts, store[off + HDR:off + HDR + ln]) == crc


def reseal(store, off):
    """recompute the checksum of the record at header offset off of the bytearray store"""
    ln, ts = struct.unpack(">H", store[off + 2:off + 4])[0], struct.unpack(">I", store[off + 8:off + 12])[0]
    struct.pack_into(">I", store, off + 4, crc32c(ts, bytes(store[off + 12:off + 12 + ln])))


# How far past a message's first byte gossmap reads it, whatever the message's own length: add_channel reads the
# features length, then the scid and both node ids (:466-476); fill_from_update reads through htlc_maximum_msat
# (:531-551); remove_channel_by_deletemsg reads the scid (:620).  A record takes part in the channel table when these
# reads stay inside the store; where they do not, gossmap's map_copy asserts and the load never returns.
UPD_READ, DEL_READ = 138, 10


def ann_read(store, p):
    """bytes add_channel reads from message offset p on (None if even the features length lies past the store end)"""
    return None if p + 260 > len(store) else 260 + struct.unpack(">H", store[p + 258:p + 260])[0] + 32 + 8 + 66


def ann_ok(store, p):
    """the announcement at message offset p takes part in the channel table"""
    n = ann_read(store, p)
    return n is not None and p + n <= len(store)


def ann_fields(m, p=0):
    """(chain_hash, scid, node_id_1, node_id_2) of the announcement at offset p of m (a message, or the store: gossmap
    reads them where they lie, also past the end of a short message)"""
    p += 260 + struct.unpack(">H", m[p + 258:p + 260])[0]
    return m[p:p + 32], m[p + 32:p + 40], m[p + 40:p + 73], m[p + 73:p + 106]


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


def signer(store, recs, i, h):
    """the node key an update at entry i is checked under when entry h holds its channel: node_id_1 or node_id_2 of
    that announcement by the update's direction bit; None without a holder"""
    return None if h is None else ann_fields(store, recs[h][0] + HDR)[2 + (store[recs[i][0] + HDR + 111] & 1)]


def audit(store, sigcheck=None):
    """The whole call: -> (list of (off, type, status, holder_off or None), summary dict).
    sigcheck(msg, signer33 or None) gives a message's status (the signature statuses with whatever gates the caller
    applies; signer is the update's channel node, None where the scid holds no channel); None leaves them 0."""
    if store[0] >> 5:
        raise ValueError("major version")
    recs, end, stop, no_amount = walk(store)
    cut, cut_status = len(recs), 0
    for i, (off, typ, ln, st) in enumerate(recs):
        if st in (0, ST_ENDED) and not crc_ok(store, off):
            cut, cut_status = i, BAD_CRC
            break
    holder = holders(store, recs, [i for i in range(cut) if recs[i][3] == 0])
    if no_amount is not None and no_amount < cut and holder.get(no_amount) is None:
        cut, cut_status = no_amount, NO_AMOUNT
    out = []
    s = dict(version=store[0], stop=cut_status or stop, end_offset=recs[cut][0] if cut_status else end, records=len(recs),
             redundant_announcements=0, updates_without_channel=0, ended_equivalent_offset=0)
    for i, (off, typ, ln, st) in enumerate(recs):
        h = None
        if cut_status and i >= cut:
            st = cut_status if i == cut else NOT_REACHED
        elif st == 0:
            m = store[off + HDR:off + HDR + ln]
            if typ in (256, 257, 258):
                h = holder.get(i)
                st = sigcheck(m, signer(store, recs, i, h) if typ == 258 else None) if sigcheck else 0
                s["redundant_announcements"] += typ == 256 and h is not None
                s["updates_without_channel"] += typ == 258 and off + HDR + UPD_READ <= len(store) and h is None
            else:
                st = STORE_RECORD if typ in STORE_TYPES else UNKNOWN
        elif st == ST_ENDED and ln >= 10:
            s["ended_equivalent_offset"] = struct.unpack(">Q", store[off + HDR + 2:off + HDR + 10])[0]
        out.append((off, typ, st, None if h is None else recs[h][0]))
    return out, s
