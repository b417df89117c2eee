// gossip_salvage.cuh — salvaging a gossip_store past a damaged record header (sv_salvage_gossip_store_host, the rule in
// include/cln_sigverify.h): which byte offsets hold a sound record, the CRC-32C of a long candidate split over a warp, and
// the host walk that finds each break and the header writes that restore or bridge it.
//
// A flipped bit in a record's flags or length sends map_catchup's walk (common/gossmap.c:815-937) into the middle of a
// message.  The records after it are intact; only the chain of lengths leading to them is broken.  The device tests
// every byte offset for a sound record (k_salvage_filter, k_salvage_crc in engine.cu); the host walk finds where each
// break resumes by binary search in that sorted list, and k_salvage_restore checks whether each damaged header's checksum
// covers exactly the bytes up to it.  tests/host_emul compiles the same code for the host.
#pragma once
#include "gossip_store.cuh"

#define GS_SV_GAP 14u            // a resume point lies at least this far past the damaged header: a filler's length >= 2
#define GS_SV_PIECE (GS_HDR + 65535u)  // the longest filler: a 16-bit length
#define GS_SV_LONG 1024u         // candidates with longer messages are checksummed by a whole warp

// the message types gossmap's load knows: the three gossip messages and the store's own records
SV_HD bool gs_known_type(u32 t) {
    return t == 256 || t == 257 || t == 258 || t == GS_CHANNEL_AMOUNT || t == GS_DELETE_CHAN || t == GS_ENDED ||
           t == GS_CHAN_DYING || t == GS_UUID;
}
// everything of a sound record at offset o but its checksum: COMPLETED, a length of at least 2 that fits, a known type
SV_HD bool gs_salvage_candidate(const u8* s, u64 len, u64 o) {
    if (o < 1 || o + GS_HDR + 2 > len) return false;
    const u32 flags = gs_be16(s + o), ml = gs_be16(s + o + 2);
    return (flags & GS_COMPLETED) && ml >= 2 && o + GS_HDR + ml <= len && gs_known_type(gs_be16(s + o + GS_HDR));
}

// ---- CRC-32C by pieces (zlib's crc32_combine for the Castagnoli polynomial).  For ccan's crc32c,
// crc32c(s, A || B) = x^(8|B|) * s ^ crc32c(0, B) in GF(2)[x] mod P (reflected), so a message is checksummed as
// independent slices, each shifted past the bytes after it, XORed together.
// a * b mod P, reflected (bit 31 is x^0)
SV_HD u32 gs_crc_mulmod(u32 a, u32 b) {
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0x82F63B78u : b >> 1;
    }
    return p;
}
// x2n[k] = x^(2^k) mod P
SV_HD void gs_crc_x2n(u32* x2n) {
    u32 p = 1u << 30;  // x^1
    for (int k = 0; k < 32; k++) {
        x2n[k] = p;
        p = gs_crc_mulmod(p, p);
    }
}
// c moved past n zero-free bytes: x^(8n) * c mod P
SV_HD u32 gs_crc_shift(const u32* x2n, u32 c, u64 n) {
    u32 k = 3;
    for (; n; n >>= 1, k++)
        if (n & 1) c = gs_crc_mulmod(x2n[k & 31], c);
    return c;
}
// lane's slice [*b, *e) of a len-byte message split into 32 slices of whole 8-byte words
SV_HD void gs_crc_slice(u32 len, u32 lane, u32* b, u32* e) {
    const u32 step = ((len + 31) / 32 + 7) & ~7u;
    *b = lane * step < len ? lane * step : len;
    *e = *b + step < len ? *b + step : len;
}
// lane's part of crc32c(start, p[0, len)) computed by a warp: its slice's checksum moved past the bytes after it.  The
// XOR of the 32 parts and of gs_crc_shift(x2n, start, len) is the checksum.
SV_HD u32 gs_crc_lane(const u32* tab, const u32* x2n, const u8* p, u32 len, u32 lane) {
    u32 b, e;
    gs_crc_slice(len, lane, &b, &e);
    return gs_crc_shift(x2n, gs_crc32c(tab, 0, p + b, e - b), len - e);
}
// a break at t resuming at q is restored when the header's checksum covers exactly store[t + 12, q)
SV_HD bool gs_restore_fits(u64 t, u64 q) { return q - t - GS_HDR <= 0xFFFFu; }

// ---- the salvage walk (host, header bytes only).  sound: the sorted offsets of the sound records.  emit(t, q) receives
// each break in store order.  Restored or bridged, the walk goes on at q, so the breaks do not depend on what the
// restore check (a checksum, on the device) decides for each.
static inline u64 gs_sv_be(const u8* p, int n) {
    u64 v = 0;
    for (int i = 0; i < n; i++) v = (v << 8) | p[i];
    return v;
}
// the pieces a bridge of span bytes is cut into: as few as fit GS_SV_PIECE, their lengths as even as possible (each at
// least GS_SV_GAP: span >= 14, and two or more pieces share more than GS_SV_PIECE bytes)
static inline u64 gs_bridge_pieces(u64 span) { return (span + GS_SV_PIECE - 1) / GS_SV_PIECE; }
static inline u64 gs_bridge_piece(u64 span, u64 k, u64 i) { return span / k + (i < span % k ? 1 : 0); }
// [t, q) already holds the fillers a bridge of it writes (a salvaged store: fillers are never sound)
static inline bool gs_bridged(const u8* s, u64 t, u64 q) {
    const u64 span = q - t, k = gs_bridge_pieces(span);
    for (u64 i = 0, p = t; i < k; p += gs_bridge_piece(span, k, i), i++)
        if (gs_sv_be(s + p, 2) != (GS_DELETED | GS_COMPLETED) || gs_sv_be(s + p + 2, 2) != gs_bridge_piece(span, k, i) - GS_HDR)
            return false;
    return true;
}
template <typename Emit>
static inline void gs_salvage_breaks(const u8* s, u64 len, const u64* sound, size_t nsound, Emit emit) {
    // index of the first sound offset >= o, for o >= t: a galloping binary search from cur, the first sound offset >= t
    // (every lookup of the walk lands on or just past it)
    size_t cur = 0;
    auto first_from = [&](u64 o) {
        size_t lo = cur, step = 1;
        while (lo + step < nsound && sound[lo + step] < o) { lo += step; step *= 2; }
        size_t hi = lo + step < nsound ? lo + step : nsound;
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if (sound[mid] < o) lo = mid + 1;
            else hi = mid;
        }
        return lo;
    };
    auto is_sound = [&](u64 o) { const size_t k = first_from(o); return k < nsound && sound[k] == o; };
    u64 t = 1;
    while (t + GS_HDR < len) {
        cur = first_from(t);
        const u64 flags = gs_sv_be(s + t, 2), end = t + GS_HDR + gs_sv_be(s + t + 2, 2);
        if (is_sound(t)) {
            if (!(flags & GS_DELETED) && gs_sv_be(s + t + GS_HDR, 2) == GS_ENDED) break;
            t = end;
            continue;
        }
        // the length is right when the record's end is sound (a message under 2 bytes ends before any resume point)
        if ((flags & GS_COMPLETED) && is_sound(end)) {
            t = end;
            continue;
        }
        const size_t k = first_from(t + GS_SV_GAP);
        if (k == nsound) break;  // the tail: sv_gossip_prune_cut's
        if (!gs_bridged(s, t, sound[k])) emit(t, sound[k]);
        t = sound[k];
    }
}
// the header writes of the break [t, q) into s: the length q - t - 12 and COMPLETED (restore), or the fillers (bridge);
// returns the fillers written
static inline u64 gs_salvage_fix(u8* s, u64 t, u64 q, bool restore) {
    if (restore) {
        const u64 n = q - t - GS_HDR;
        s[t] |= GS_COMPLETED >> 8;
        s[t + 2] = (u8)(n >> 8);
        s[t + 3] = (u8)n;
        return 0;
    }
    const u64 span = q - t, k = gs_bridge_pieces(span);
    for (u64 i = 0, p = t; i < k; i++) {
        const u64 pl = gs_bridge_piece(span, k, i) - GS_HDR;
        s[p] = (u8)((GS_DELETED | GS_COMPLETED) >> 8);
        s[p + 1] = 0;
        s[p + 2] = (u8)(pl >> 8);
        s[p + 3] = (u8)pl;
        p += GS_HDR + pl;
    }
    return k;
}
struct gs_salvage_count {
    u64 breaks, restored, bridged, bridged_bytes, fillers;
};
// the header writes of the n breaks [t[i], q[i]) into s, restore[i]: what the restore check decided
static inline gs_salvage_count gs_salvage_apply(u8* s, const u64* t, const u64* q, const u8* restore, size_t n) {
    gs_salvage_count c{n, 0, 0, 0, 0};
    for (size_t i = 0; i < n; i++) {
        const u64 k = gs_salvage_fix(s, t[i], q[i], restore[i]);
        c.restored += restore[i] != 0;
        c.bridged += restore[i] == 0;
        c.bridged_bytes += restore[i] ? 0 : q[i] - t[i];
        c.fillers += k;
    }
    return c;
}
