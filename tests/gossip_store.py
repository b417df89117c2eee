"""Python model of how gossmap loads a gossip_store (common/gossmap.c, reference): map_catchup's record walk and
checksums (:815-937), and the channel table that decides which announcement signs each channel_update (add_channel
:440-500, remove_channel_by_deletemsg :612-626).  sv_verify_gossip_store_host must agree with it record for record."""
import struct

HDR = 12
COMPLETED, DELETED = 0x2000, 0x8000
CHANNEL_AMOUNT, DELETE_CHAN, ENDED, CHAN_DYING, UUID = 4101, 4103, 4105, 4106, 4107
# record statuses besides the signature statuses (include/cln_sigverify.h SV_GS_*)
EOF, ST_DELETED, STORE_RECORD, UNKNOWN, NOT_REACHED = 0, 16, 17, 18, 19
INCOMPLETE, PARTIAL, TRUNCATED, BAD_CRC, ST_ENDED, NO_AMOUNT = 32, 33, 34, 35, 36, 37
NONE = None


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


def walk(store):
    """map_catchup's header walk -> (records [(off, type, len, status)], map_end, stop, no_amount entry or None);
    status 0 = live, to be judged by checksum and content"""
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
        if st not in (0, ST_DELETED):
            stop = st
            break
        off += HDR + ln
    return recs, off, stop, no_amount


def crc_ok(store, off):
    ln, crc, ts = struct.unpack(">HII", store[off + 2:off + 12])
    return crc32c(ts, store[off + HDR:off + HDR + ln]) == crc


def ann_ok(m):
    """an announcement takes part in the channel table when it holds the fixed layout through node_id_2"""
    return len(m) >= 260 and len(m) >= 260 + struct.unpack(">H", m[258:260])[0] + 32 + 8 + 66


def ann_fields(m):
    """(chain_hash, scid, node_id_1, node_id_2)"""
    p = 260 + struct.unpack(">H", m[258:260])[0]
    return m[p:p + 32], m[p + 32:p + 40], m[p + 40:p + 73], m[p + 73:p + 106]


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
    held, holder = {}, {}
    for i in range(cut):
        off, typ, ln, st = recs[i]
        if st:
            continue
        m = store[off + HDR:off + HDR + ln]
        if typ == 256 and ann_ok(m):
            scid = ann_fields(m)[1]
            holder[i] = held.get(scid)
            held.setdefault(scid, i)
        elif typ == DELETE_CHAN and ln >= 10:
            held.pop(m[2:10], None)
        elif typ == 258 and ln >= 112:
            holder[i] = held.get(m[98:106])
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
                signer = None
                if typ == 258 and h is not None:
                    a = store[recs[h][0] + HDR:recs[h][0] + HDR + recs[h][2]]
                    signer = ann_fields(a)[2 + (m[111] & 1)]
                st = sigcheck(m, signer) if sigcheck else 0
                s["redundant_announcements"] += typ == 256 and h is not None
                s["updates_without_channel"] += typ == 258 and ln >= 112 and h is None
            else:
                st = STORE_RECORD if typ in (CHANNEL_AMOUNT, DELETE_CHAN, CHAN_DYING, UUID) else UNKNOWN
        elif st == ST_ENDED and ln >= 10:
            s["ended_equivalent_offset"] = struct.unpack(">Q", store[off + HDR + 2:off + HDR + 10])[0]
        out.append((off, typ, st, None if h is None else recs[h][0]))
    return out, s
