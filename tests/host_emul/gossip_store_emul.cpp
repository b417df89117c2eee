// tests/host_emul/gossip_store_emul.cpp — TEST-ONLY host build of lightning_b200/csrc/gossip_store.cuh (linked into
// libemul.so).
//
// The checksum the k_store_crc_flags kernel computes per record, the header walk sv_verify_gossip_store_host runs, and the
// per-scid event rule of k_store_resolve applied in store order (the kernel applies it per scid after a stable sort by
// scid, which gives each scid the same sequence).  The sort and the thread layout are checked on the device by
// tests/test_gpu_gossip_store.py.
#include <map>
#include "../../lightning_b200/csrc/gossip_store.cuh"

static u32 g_tab[2048];
static const u32* tab() {
    if (!g_tab[1])
        for (u32 i = 0; i < 256; i++) gs_crc_fill(g_tab, i);
    return g_tab;
}

extern "C" u32 emul_gs_crc32c(u32 start, const u8* p, u32 len) { return gs_crc32c(tab(), start, p, len); }

// ok[i] = 1 iff the record at header offset offs[i] carries the right checksum
extern "C" void emul_gs_crc_ok(const u8* store, const u64* offs, size_t n, u8* ok) {
    for (size_t i = 0; i < n; i++) ok[i] = gs_record_crc_ok(tab(), store, offs[i]);
}

// the header walk: returns the record count (entries written up to cap); end3 = {map_end, stop status, no_amount entry}
extern "C" long long emul_gs_walk(const u8* store, u64 len, u64* off, u32* type, u32* mlen, int* status, u64 cap, u64* end3) {
    gs_walk_end e;
    u64 i = 0;
    u64 n = gs_walk(store, len, [&](const gs_rec& r) {
        if (i < cap) { off[i] = r.off; type[i] = r.type; mlen[i] = r.len; status[i] = r.status; }
        i++;
    }, &e);
    end3[0] = e.end;
    end3[1] = (u64)(long long)e.stop;
    end3[2] = e.no_amount;
    return (long long)n;
}

// channel events in store order (message offsets, kinds GS_EV_*, message index per event) of a store of len bytes:
// holder[msg] as k_store_resolve writes it (GS_NONE where nothing held the scid, or where gossmap's reads of the record
// would pass the end of the store)
extern "C" void emul_gs_resolve(const u8* store, u64 len, const u64* ev_off, const u8* ev_kind, const u32* ev_msg, size_t n,
                                u32* holder) {
    std::map<u64, u32> held;
    for (size_t e = 0; e < n; e++) {
        const u8* p = store + ev_off[e];
        if (!gs_event_ok(ev_kind[e], p, len - ev_off[e])) continue;
        auto it = held.emplace(gs_event_scid(ev_kind[e], p), GS_NONE).first;
        u32 h = gs_event(&it->second, ev_kind[e], ev_msg[e]);
        if (ev_kind[e] != GS_EV_DEL) holder[ev_msg[e]] = h;
    }
}
