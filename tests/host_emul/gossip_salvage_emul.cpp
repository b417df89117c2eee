// tests/host_emul/gossip_salvage_emul.cpp — TEST-ONLY host build of lightning_b200/csrc/gossip_salvage.cuh (linked into
// libemul.so).
//
// What k_salvage_filter and k_salvage_crc decide for every byte offset, with the warp's 32 checksum slices of a long
// candidate taken one after another and combined as the lanes' XOR reduction combines them; the host walk and header
// writes of sv_salvage_gossip_store_host, with k_salvage_restore's check of each break.  The compaction and the thread
// layout are checked on the device by tests/test_gpu_gossip_store_salvage.py.
#include <vector>

#include "../../lightning_b200/csrc/gossip_salvage.cuh"

static u32 g_tab[2048], g_x2n[32];
static const u32* tab() {
    if (!g_tab[1]) {
        for (u32 i = 0; i < 256; i++) gs_crc_fill(g_tab, i);
        gs_crc_x2n(g_x2n);
    }
    return g_tab;
}

// crc32c(start, p[0, len)) as a warp of k_salvage_crc and k_salvage_restore computes it
extern "C" u32 emul_gs_crc_warp(u32 start, const u8* p, u32 len) {
    const u32* t = tab();
    u32 r = 0;
    for (u32 lane = 0; lane < 32; lane++) r ^= gs_crc_lane(t, g_x2n, p, len, lane);
    return gs_crc_shift(g_x2n, start, len) ^ r;
}

extern "C" u32 emul_gs_crc_shift(u32 c, u64 n) {
    tab();
    return gs_crc_shift(g_x2n, c, n);
}

// the sorted sound offsets of store[0, len) (up to cap written); returns how many there are
extern "C" u64 emul_gs_salvage_sound(const u8* store, u64 len, u64* out, u64 cap) {
    const u32* t = tab();
    u64 n = 0;
    for (u64 o = 1; o < len; o++) {
        if (!gs_salvage_candidate(store, len, o)) continue;
        const u8* h = store + o;
        const u32 ml = gs_be16(h + 2);
        const bool ok = ml > GS_SV_LONG ? emul_gs_crc_warp(gs_be32(h + 8), h + GS_HDR, ml) == gs_be32(h + 4)
                                        : gs_record_crc_ok(t, store, o);
        if (!ok) continue;
        if (n < cap) out[n] = o;
        n++;
    }
    return n;
}

// the same sound offsets by a plain one-core scan: every candidate checksummed in one pass (gs_record_crc_ok), as a CPU
// implementation of the rule would; returns how many there are
extern "C" u64 emul_gs_salvage_sound_plain(const u8* store, u64 len) {
    const u32* t = tab();
    u64 n = 0;
    for (u64 o = 1; o < len; o++) n += gs_salvage_candidate(store, len, o) && gs_record_crc_ok(t, store, o);
    return n;
}

// the walk's breaks over s with the given sound offsets, each break's restore check as k_salvage_restore makes it, and
// the header writes into s: returns the breaks (up to cap listed, kind 1 restored, 2 bridged); count5 = breaks, restored,
// bridged, bridged bytes, fillers
extern "C" u64 emul_gs_salvage_walk(u8* s, u64 len, const u64* sound, u64 nsound, u64* act_off, u64* act_resume,
                                    u8* act_kind, u64 cap, u64* count5) {
    std::vector<u64> t, q;
    std::vector<u8> restore;
    gs_salvage_breaks(s, len, sound, nsound, [&](u64 a, u64 b) {
        t.push_back(a);
        q.push_back(b);
        restore.push_back(gs_restore_fits(a, b) &&
                          emul_gs_crc_warp(gs_be32(s + a + 8), s + a + GS_HDR, (u32)(b - a - GS_HDR)) == gs_be32(s + a + 4));
    });
    for (size_t i = 0; i < t.size() && i < cap; i++) {
        act_off[i] = t[i];
        act_resume[i] = q[i];
        act_kind[i] = restore[i] ? 1 : 2;
    }
    const gs_salvage_count c = gs_salvage_apply(s, t.data(), q.data(), restore.data(), t.size());
    const u64 v[5] = {c.breaks, c.restored, c.bridged, c.bridged_bytes, c.fillers};
    for (int i = 0; i < 5; i++) count5[i] = v[i];
    return t.size();
}
