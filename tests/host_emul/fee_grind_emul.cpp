// tests/host_emul/fee_grind_emul.cpp — TEST-ONLY host build of onchaind's fee grind in lightning_b200/csrc/verify.cuh
// (grind_*: the code k_grind_setup and k_grind run), linked into libemul.so beside emul.cpp.
//
// The feerate walk as sv_grind_tx_fee_host bounds it and k_grind filters it, and the candidate check after one
// grind_setup.  The comb table is the one emul.cpp builds (read through emul_gtable_get).
#include <cstring>
#include <vector>
#include "../../lightning_b200/csrc/common.cuh"
#include "../../lightning_b200/csrc/verify.cuh"

extern "C" void emul_gtable_get(u32 e, u32* xy16);  // emul.cpp

static std::vector<ge_mem> g_grind_table;
static const ge_mem* gtable() {
    if (g_grind_table.empty()) {
        g_grind_table.resize(SV_GT_ENTRIES);
        for (u32 e = 0; e < SV_GT_ENTRIES; e++) {
            u32 xy[16];
            emul_gtable_get(e, xy);
            memcpy(g_grind_table[e].x, xy, 32);
            memcpy(g_grind_table[e].y, xy + 8, 32);
        }
    }
    return g_grind_table.data();
}

extern "C" {

// the feerates the walk checks; returns how many (the first cap are written with their fees)
size_t emul_grind_walk(u64 weight, u64 min_feerate, u64 max_feerate, u64 input_amount, size_t cap, u64* feerates, u64* fees) {
    if (min_feerate > max_feerate) return 0;
    const u64 last = grind_last_feerate(min_feerate, max_feerate, weight, input_amount);
    size_t n = 0;
    for (u64 f = min_feerate; f <= last; f++) {
        u64 fee;
        if (!grind_feerate_checked(f, weight, min_feerate, input_amount, &fee)) continue;
        if (n < cap) { feerates[n] = f; fees[n] = fee; }
        n++;
    }
    return n;
}

// the candidate check for each of n output amounts, after one grind_setup (as k_grind_setup, then k_grind)
void emul_grind_candidates(int kind, const void* tx_item, const u8* blob, const u8* key, const u8* sig, const u64* amounts,
                           size_t n, u8* out) {
    const ge_mem* gt = gtable();
    sv_tx_item t;
    memcpy(&t, tx_item, sizeof t);
    sv_grind_state g;
    qtab_entry tab[8];
    grind_setup(&g, tab, kind, key, sig, t, blob);
    for (size_t i = 0; i < n; i++) out[i] = (u8)grind_candidate(&g, t, blob, sig, amounts[i], gt);
}

// the same check on a chosen message instead of a sighash (the state's preimage prefix is unused)
int emul_grind_verify_msg(int kind, const u8* key, const u8* sig, const u8* msg32) {
    const ge_mem* gt = gtable();
    sv_tx_item t;
    memset(&t, 0, sizeof t);
    sv_grind_state g;
    qtab_entry tab[8];
    const u8 blob[1] = {0};
    grind_setup(&g, tab, kind, key, sig, t, blob);
    return (int)grind_verify_msg(&g, msg32, sig, gt);
}
}
