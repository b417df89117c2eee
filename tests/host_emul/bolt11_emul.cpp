// tests/host_emul/bolt11_emul.cpp — TEST-ONLY host build of lightning_b200/csrc/bolt11.cuh (linked into libemul.so).
//
// One invoice through the functions the k_b11_* kernels call, in the order sv_verify_bolt11_host combines them: parse and
// signing hash; then either the compressed-key ECDSA check against the `n` key (ecdsa_parse, ecdsa_finish_prep,
// verify_curve_side: the rules every verification route shares) or the recovery (b11_recover_prep, the x-only key decode
// and ecmult_uniform that k_main<SV_KIND_SCHNORR> runs, schnorr_park, b11_recover_final_batch).  What this cannot check is
// the packing of the two groups and the launches themselves; tests/test_gpu_bolt11.py does that on the device.  The comb
// table is the one emul.cpp builds (read through emul_gtable_get).  The group law logs its branches into emul.cpp's log.
#include <cstring>
#include <vector>
#include "../../lightning_b200/csrc/common.cuh"
#include "ge_trace.h"
#include "../../lightning_b200/csrc/bolt11.cuh"

extern "C" void emul_gtable_get(u32 e, u32* xy16);  // emul.cpp

static std::vector<ge_mem> g_b11_table;
static const ge_mem* b11_gtable() {
    if (g_b11_table.empty()) {
        g_b11_table.resize(SV_GT_ENTRIES);
        for (u32 e = 0; e < SV_GT_ENTRIES; e++) {
            u32 xy[16];
            emul_gtable_get(e, xy);
            memcpy(g_b11_table[e].x, xy, 32);
            memcpy(g_b11_table[e].y, xy + 8, 32);
        }
    }
    return g_b11_table.data();
}

// the recovery up to the parked result, as k_b11_rec_prep and k_main<SV_KIND_SCHNORR> leave it
static void b11_recover_park(sv_jac* j, const u8* sig64, u8 recid, const u8* msg32) {
    sv_work w;
    u8 x32[32];
    b11_recover_prep(w, x32, sig64, recid, msg32);
    ge E;
    bool ok = (w.flags & SV_WF_VALID) != 0;
    ok = key_decode(E, SV_KIND_SCHNORR, x32) && ok;
    qtab_entry tab[8];
    gej R;
    ecmult_uniform(R, &w, E, b11_gtable(), tab);
    schnorr_park(j, R, ok);
}

// the recovery alone: status 1 with the compressed key, 0 (key zeros) where secp256k1_ecdsa_recover fails
static int b11_recover_host(const u8* sig64, u8 recid, const u8* msg32, u8* out33) {
    sv_jac j;
    b11_recover_park(&j, sig64, recid, msg32);
    int st;
    b11_recover_final_batch(&st, out33, &j, 1);
    return st;
}

extern "C" {

// Returns the status the device reports (1 / 0 / -1).  hash32: the signing hash (zeros for -1); node33: the receiver_id
// (zeros unless 1); have_n: 1 if the `n` path was taken.
int emul_bolt11(const u8* s, u32 span, u8* hash32, u8* node33, int* have_n) {
    memset(hash32, 0, 32);
    memset(node33, 0, 33);
    *have_n = 0;
    b11_str b;
    b11_parsed p;
    if (!b11_parse(s, span, &b, &p)) return -1;
    b11_sighash(hash32, s, b);
    *have_n = p.have_n;
    if (!p.have_n) return b11_recover_host(p.sig, p.recid, hash32, node33);
    sc r, sg, m, sinv;
    bool ok = ecdsa_parse(r, sg, m, p.sig, hash32);
    if (ok) sc_inverse(sinv, sg); else sinv = sg;
    sv_work w;
    ecdsa_finish_prep(w, ok, r, m, sinv);
    qtab_entry tab[8];
    u32 v = verify_curve_side(SV_KIND_ECDSA33, &w, p.key33, p.sig, b11_gtable(), tab);
    const int st = (p.recid <= 3 && v) ? 1 : 0;
    if (st) memcpy(node33, p.key33, 33);
    return st;
}

int emul_bolt11_recover(const u8* sig64, int recid, const u8* msg32, u8* out33) {
    return b11_recover_host(sig64, (u8)recid, msg32, out33);
}

// cnt (1 .. SV_FINAL_BATCH) recoveries parked side by side and finished by one b11_recover_final_batch, as one thread of
// k_b11_rec_final finishes them; -1 for any other cnt
int emul_bolt11_recover_batch(const u8* sig64, const int* recid, const u8* msg32, int cnt, int* status, u8* key33) {
    if (cnt < 1 || cnt > SV_FINAL_BATCH) return -1;
    sv_jac j[SV_FINAL_BATCH];
    for (int i = 0; i < cnt; i++) b11_recover_park(&j[i], sig64 + 64 * i, (u8)recid[i], msg32 + 32 * i);
    b11_recover_final_batch(status, key33, j, cnt);
    return 0;
}

}  // extern "C"
