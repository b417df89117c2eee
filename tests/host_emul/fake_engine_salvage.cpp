// fake_engine_salvage.cpp — sv_salvage_gossip_store_host on the CPU, with the host build of gossip_salvage.cuh (every
// byte offset tested one after another in place of k_salvage_filter and k_salvage_crc), linked beside
// fake_engine_prune.c so that sv_salvage_gossip_store_fd (lightning_b200/csrc/gossip_salvage_fd.c) can be tested without
// a GPU (tests/test_gossip_store_salvage_host.py).  Arguments and errors are the engine's.
#include <string.h>

#include <vector>

#include "../../include/cln_sigverify.h"
#include "../../lightning_b200/csrc/gossip_salvage.cuh"

extern "C" int sv_salvage_gossip_store_host(sv_ctx* ctx, const uint8_t* store, size_t len, uint8_t* out, uint64_t* act_off,
                                            uint64_t* act_resume, uint8_t* act_kind, size_t act_capacity,
                                            sv_gossip_salvage_summary* sum) {
    if (!ctx || !store || !out || len < 1 || !sum || (act_capacity && (!act_off || !act_resume || !act_kind)))
        return SV_ERR_ARG;
    if (store[0] >> 5) return SV_ERR_ARG;
    static u32 tab[2048];
    if (!tab[1])
        for (u32 i = 0; i < 256; i++) gs_crc_fill(tab, i);
    std::vector<u64> sound;
    for (u64 o = 1; o < len; o++)
        if (gs_salvage_candidate(store, len, o) && gs_record_crc_ok(tab, store, o)) sound.push_back(o);
    std::vector<u64> t, q;
    std::vector<u8> restore;
    gs_salvage_breaks(store, len, sound.data(), sound.size(), [&](u64 a, u64 b) {
        t.push_back(a);
        q.push_back(b);
        restore.push_back(gs_restore_fits(a, b) &&
                          gs_crc32c(tab, gs_be32(store + a + 8), store + a + GS_HDR, (u32)(b - a - GS_HDR)) ==
                              gs_be32(store + a + 4));
    });
    for (size_t i = 0; i < t.size() && i < act_capacity; i++) {
        act_off[i] = t[i];
        act_resume[i] = q[i];
        act_kind[i] = restore[i] ? SV_SALVAGE_RESTORED : SV_SALVAGE_BRIDGED;
    }
    if (out != store) memcpy(out, store, len);
    const gs_salvage_count c = gs_salvage_apply(out, t.data(), q.data(), restore.data(), t.size());
    *sum = sv_gossip_salvage_summary{c.breaks, c.restored, c.bridged, c.bridged_bytes, c.fillers, (uint64_t)sound.size()};
    return SV_OK;
}
