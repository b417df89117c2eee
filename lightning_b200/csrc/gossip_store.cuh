// gossip_store.cuh — reading a Core Lightning gossip_store: record walk, record checksums and the channel each
// channel_update is signed for.
//
// Reference (paths relative to the Core Lightning tree):
//   layout       1 version byte, then records: be16 flags, be16 len, be32 crc, be32 timestamp, msg   common/gossip_store.h
//   walk         map_catchup                                                        common/gossmap.c:815-937
//   checksum     csum_matches -> crc32c(timestamp, msg, len)                        common/gossmap.c:800-812, ccan/crc32c
//   channels     add_channel (first announcement of an scid holds it, later ones are redundant; no amount record
//                before EOF stops the walk)                                         common/gossmap.c:440-500
//                fill_from_update                                                   common/gossmap.c:525-568
//                remove_channel_by_deletemsg                                        common/gossmap.c:612-626
//                gossmap reads these at fixed offsets without comparing them with the message length, so a short
//                message takes part with the store bytes that follow it (gs_event_ok)
//
// The header walk is host code (it reads 12 header bytes and the 2-byte type of each record, as map_catchup does).
// The checksum and the per-scid event rule are SV_HD: the k_store_* kernels in engine.cu call them, tests/host_emul
// compiles the same code for the host.
#pragma once
#include "common.cuh"

#define GS_HDR 12u
#define GS_COMPLETED 0x2000u
#define GS_DELETED 0x8000u
// store-only message types (common/gossip_store_wire.csv)
#define GS_CHANNEL_AMOUNT 4101u
#define GS_DELETE_CHAN 4103u
#define GS_ENDED 4105u
#define GS_CHAN_DYING 4106u
#define GS_UUID 4107u

// record statuses besides the signature statuses of 256/257/258 (include/cln_sigverify.h SV_GS_*)
#define GS_LIVE 0  // walked, checksum and message still to be judged
#define GS_ST_DELETED 16
#define GS_ST_STORE_RECORD 17
#define GS_ST_UNKNOWN 18
#define GS_ST_NOT_REACHED 19
#define GS_ST_INCOMPLETE 32
#define GS_ST_PARTIAL 33
#define GS_ST_TRUNCATED 34
#define GS_ST_BAD_CRC 35
#define GS_ST_ENDED 36
#define GS_ST_NO_AMOUNT 37

// ---- CRC-32C (Castagnoli, reflected polynomial 0x82F63B78), ccan's crc32c(start_crc, data, len) convention: the
// running value is inverted on entry and on exit.  Slice-by-8: table k maps a byte to its contribution k bytes back.
SV_HD u32 gs_crc_t0(u32 b) {
    u32 c = b;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u)));
    return c;
}
// fills tab[8][256]; tab[k][i] = tab[k-1][i] >> 8 ^ tab[0][tab[k-1][i] & 0xff]
SV_HD void gs_crc_fill(u32* tab, u32 i) {
    u32 c = gs_crc_t0(i);
    tab[i] = c;
    for (int k = 1; k < 8; k++) {
        c = (c >> 8) ^ gs_crc_t0(c & 0xffu);
        tab[256 * k + i] = c;
    }
}
SV_HD u32 gs_crc32c(const u32* tab, u32 start, const u8* p, u32 len) {
    u32 c = ~start, i = 0;
    for (; i + 8 <= len; i += 8) {
        u32 lo = c ^ ((u32)p[i] | ((u32)p[i + 1] << 8) | ((u32)p[i + 2] << 16) | ((u32)p[i + 3] << 24));
        u32 hi = (u32)p[i + 4] | ((u32)p[i + 5] << 8) | ((u32)p[i + 6] << 16) | ((u32)p[i + 7] << 24);
        c = tab[1792 + (lo & 0xff)] ^ tab[1536 + ((lo >> 8) & 0xff)] ^ tab[1280 + ((lo >> 16) & 0xff)] ^ tab[1024 + (lo >> 24)] ^
            tab[768 + (hi & 0xff)] ^ tab[512 + ((hi >> 8) & 0xff)] ^ tab[256 + ((hi >> 16) & 0xff)] ^ tab[hi >> 24];
    }
    for (; i < len; i++) c = (c >> 8) ^ tab[(c ^ p[i]) & 0xffu];
    return ~c;
}
SV_HD u32 gs_be16(const u8* p) { return ((u32)p[0] << 8) | p[1]; }
SV_HD u32 gs_be32(const u8* p) { return ((u32)p[0] << 24) | ((u32)p[1] << 16) | ((u32)p[2] << 8) | p[3]; }
// the record at header offset off (complete, inside the store): does its checksum match?
SV_HD bool gs_record_crc_ok(const u32* tab, const u8* store, u64 off) {
    const u8* h = store + off;
    return gs_crc32c(tab, gs_be32(h + 8), h + GS_HDR, gs_be16(h + 2)) == gs_be32(h + 4);
}

// ---- channel events, one scid at a time in store order (gossmap's channel table for that scid) ----------------------
// An announcement holds the channel unless one already does (then it is redundant); a delete_chan frees it; an update
// is signed for whichever announcement holds it.  *held is that announcement's message index, or GS_NONE.
#define GS_NONE 0xFFFFFFFFu
#define GS_EV_ANN 0
#define GS_EV_DEL 1
#define GS_EV_UPD 2
// returns the holder the event sees: for an announcement the earlier holder (GS_NONE: it takes the channel), for an
// update the announcement it is signed for (GS_NONE: no channel), for a delete_chan the holder it removed
SV_HD u32 gs_event(u32* held, int kind, u32 msg) {
    u32 h = *held;
    if (kind == GS_EV_ANN) { if (h == GS_NONE) *held = msg; }
    else if (kind == GS_EV_DEL) *held = GS_NONE;
    return h;
}
// gossmap reads an event at fixed offsets from the message start whatever the message's own length, so a short message
// reads on into the records after it: an announcement through node_id_2 (add_channel), a delete_chan's scid
// (remove_channel_by_deletemsg), an update through htlc_maximum_msat (fill_from_update).  room = bytes from the message
// start to the end of the store.  An event takes part in the channel table when those reads stay inside the store; only
// where they would not (gossmap's map_copy asserts there and the load never returns) does it take no part.
#define GS_DEL_READ 10u
#define GS_UPD_READ 138u
SV_HD bool gs_event_ok(int kind, const u8* msg, u64 room) {
    if (kind == GS_EV_ANN) return room >= 260 && room >= 260 + (u64)gs_be16(msg + 258) + 32 + 8 + 66;
    if (kind == GS_EV_DEL) return room >= GS_DEL_READ;
    return room >= GS_UPD_READ;
}
// the scid an event is about (big-endian u64; ordering only needs it to be the same for the same 8 bytes)
SV_HD u64 gs_event_scid(int kind, const u8* msg) {
    const u8* s = kind == GS_EV_ANN ? msg + 260 + gs_be16(msg + 258) + 32 : (kind == GS_EV_DEL ? msg + 2 : msg + 98);
    u64 v = 0;
    for (int b = 0; b < 8; b++) v = (v << 8) | s[b];
    return v;
}

// ---- the header walk of map_catchup (host): start at offset 1, stop at the first record gossmap stops at.  Every
// record the walk visits is one entry: its header offset, its type where the store holds the type bytes (else 0) and a
// preliminary status: GS_LIVE, GS_ST_DELETED, or for the record it stopped at GS_ST_INCOMPLETE / _PARTIAL / _TRUNCATED /
// _ENDED.  What the header alone cannot settle is left to the caller: checksums (GS_ST_BAD_CRC) and whether an
// announcement without room for its amount record is redundant (GS_ST_NO_AMOUNT, *no_amount = its entry).
struct gs_rec {
    u64 off;
    u32 type, len;
    int status;
};
struct gs_walk_end {
    u64 end;        // map_end: offset of the record the walk stopped at, or where it ran out of store
    int stop;       // 0 (ran out of store) or the stop status
    u64 no_amount;  // entry of the first live announcement whose amount record would not fit, or ~0
};
// emit(const gs_rec&) receives the entries in store order: one pass, because each header's position depends on the one
// before it (on a store larger than the caches every record costs a memory latency).  past_truncated (the prune's walk,
// which deletes such a record): a GS_ST_TRUNCATED record does not stop the walk.
template <typename Emit>
static inline u64 gs_walk(const u8* s, u64 len, Emit emit, gs_walk_end* e, bool past_truncated = false) {
    auto be16 = [](const u8* p) { return ((u32)p[0] << 8) | p[1]; };
    u64 off = 1, n = 0;
    e->stop = 0;
    e->no_amount = ~(u64)0;
    for (; off + GS_HDR < len; n++) {
        const u8* h = s + off;
        u32 flags = be16(h), msglen = be16(h + 2);
        gs_rec r{off, off + GS_HDR + 2 <= len ? be16(h + GS_HDR) : 0u, msglen, GS_LIVE};
        if (!(flags & GS_COMPLETED)) r.status = GS_ST_INCOMPLETE;
        else if (flags & GS_DELETED) r.status = GS_ST_DELETED;
        else if (off + GS_HDR + msglen > len) r.status = GS_ST_PARTIAL;
        else if (msglen < 2) r.status = GS_ST_TRUNCATED;
        else if (r.type == GS_ENDED) r.status = GS_ST_ENDED;
        if (r.status == GS_LIVE && r.type == 256 && e->no_amount == ~(u64)0 && off + GS_HDR + msglen + GS_HDR + 2 + 8 > len)
            e->no_amount = n;
        emit(r);
        if (r.status != GS_LIVE && r.status != GS_ST_DELETED && !(past_truncated && r.status == GS_ST_TRUNCATED)) {
            e->stop = r.status;
            n++;
            break;
        }
        off += GS_HDR + msglen;
    }
    e->end = off;
    return n;
}
