// tests/host_emul/emul.cpp — TEST-ONLY build of the kernel source for the host.
//
// The engine's device headers (lightning_b200/csrc/*.cuh) are written against a handful of
// 256-bit primitives that have a portable uint64_t fallback next to their inline-PTX form.  This
// translation unit compiles those very headers with g++ so that all logic above the primitives
// (field/scalar reduction, addition chains, group law case analysis, GLV + window recoding, table
// construction, accept/reject rules, SHA-256) can be differential-tested against the oracle on a
// machine without a GPU.  It is NOT part of the product: libcln_sigverify.so never contains or
// calls this code, and the engine has no CPU execution path.
#include <atomic>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../lightning_b200/csrc/common.cuh"
// branch log of the group law (ge_trace.h): the second lane of a pair runs on a thread of its own and is not logged, both
// lanes take the same branches
#include "ge_trace.h"
std::vector<unsigned char>*& emul_trace_log() {
    static thread_local std::vector<unsigned char>* log = nullptr;
    return log;
}
struct fe;
// host stand-in for the warp shuffle between the two lanes of a pair (verify.cuh pair_swap): the lanes are two threads
// that meet at a mailbox; a sense-reversing barrier on atomics orders the exchange
struct pair_mailbox {
    std::atomic<int> arrived{0};
    std::atomic<int> gen{0};
    unsigned slot[2][8];
    void barrier() {
        int g = gen.load();
        if (arrived.fetch_add(1) == 1) { arrived.store(0); gen.fetch_add(1); }
        else while (gen.load() == g) std::this_thread::yield();
    }
};
#include "../../lightning_b200/csrc/verify.cuh"
static inline void pair_swap(const pair_lane& L, fe& recv, const fe& send) {
    memcpy(L.mb->slot[L.role], send.v, 32);
    L.mb->barrier();
    memcpy(recv.v, L.mb->slot[1 - L.role], 32);
    L.mb->barrier();
}
#include "../../lightning_b200/csrc/selftest.cuh"
#include "../../lightning_b200/csrc/batch.cuh"

static std::vector<ge_mem> g_table;
static int g_ecdsa33_exact = 0;
static size_t g_last_exact = 0;
static u8* g_aux = nullptr;
static std::vector<ge_mem> g_bases(16);

static void build_gtable_fast() {
    if (!g_table.empty()) return;
    gtable_make_bases(g_bases.data());
    g_table.resize(SV_GT_ENTRIES);
    // incremental: entry(row, d) = entry(row, d-1) + base, Jacobian, then one batched inversion per row
    for (int row = 0; row < 16; row++) {
        size_t cnt = (row == 15) ? 65536 : SV_GT_ROW;
        size_t off = (size_t)row * SV_GT_ROW;
        ge b;
        ge_from_mem(b, &g_bases[row]);
        std::vector<gej> pts(cnt);
        gej acc;
        gej_set_ge(acc, b);
        pts[0] = acc;
        for (size_t d = 1; d < cnt; d++) {
            gej_add_ge(acc, acc, b);
            pts[d] = acc;
        }
        std::vector<fe> pre(cnt);
        pre[0] = pts[0].z;
        for (size_t d = 1; d < cnt; d++) fe_mul(pre[d], pre[d - 1], pts[d].z);
        fe inv;
        fe_inv(inv, pre[cnt - 1]);
        for (size_t d = cnt; d-- > 0;) {
            fe zi;
            if (d > 0) {
                fe_mul(zi, inv, pre[d - 1]);
                fe_mul(inv, inv, pts[d].z);
            } else {
                zi = inv;
            }
            ge a;
            ge_set_gej_zinv(a, pts[d], zi);
            fe_normalize(a.x);
            fe_normalize(a.y);
            ge_to_mem(&g_table[off + d], a);
        }
    }
}

extern "C" {

void emul_fe_op(int op, const u32* a, const u32* b, u32* out) {
    fe x, y, r;
    memcpy(x.v, a, 32);
    if (b) memcpy(y.v, b, 32); else fe_set_zero(y);
    switch (op) {
        case 0: fe_mul(r, x, y); break;
        case 1: fe_sqr(r, x); break;
        case 2: fe_add(r, x, y); break;
        case 3: fe_sub(r, x, y); break;
        case 4: fe_inv(r, x); break;
        case 5: { bool ok = fe_sqrt(r, x); if (!ok) fe_set_zero(r); break; }
        case 6: fe_neg(r, x); break;
        case 7: fe_mul_small(r, x, y.v[0]); break;
        case 8: fe_mul3(r, x); break;
        case 9: fe_mul8(r, x); break;
        default: fe_set_zero(r);
    }
    fe_normalize(r);
    memcpy(out, r.v, 32);
}
// raw (un-normalised) result, to check the weak-form invariant value < 2^256 and congruence
void emul_fe_op_raw(int op, const u32* a, const u32* b, u32* out) {
    fe x, y, r;
    memcpy(x.v, a, 32);
    memcpy(y.v, b, 32);
    switch (op) {
        case 0: fe_mul(r, x, y); break;
        case 2: fe_add(r, x, y); break;
        case 3: fe_sub(r, x, y); break;
        default: fe_set_zero(r);
    }
    memcpy(out, r.v, 32);
}
void emul_sc_op(int op, const u32* a, const u32* b, u32* out) {
    sc x, y, r;
    memcpy(x.v, a, 32);
    if (b) memcpy(y.v, b, 32);
    switch (op) {
        case 0: sc_mul(r, x, y); break;
        case 1: sc_inverse(r, x); break;
        case 2: sc_add(r, x, y); break;
        case 3: sc_negate(r, x); break;
        default: memset(r.v, 0, 32);
    }
    memcpy(out, r.v, 32);
}
void emul_sc_reduce512(const u32* t16, u32* out) {
    sc r;
    sc_reduce512(r, t16);
    memcpy(out, r.v, 32);
}
// GLV + recoding: returns k1[5],k2[5] (sign in bit 31 of limb 4) and gd[16]
void emul_prepare(const u32* u1, const u32* u2, u32* k1, u32* k2, int* gd) {
    sv_work w;
    sc a, b;
    memcpy(a.v, u1, 32);
    memcpy(b.v, u2, 32);
    sc_prepare_u2(w, b);
    sc_prepare_u1(w, a);
    memcpy(k1, w.k1, 20);
    memcpy(k2, w.k2, 20);
    memcpy(gd, w.gd, 64);
}
void emul_sha256d(const u8* p, size_t len, u8* out32) { sha256d_bytes(out32, p, len); }
void emul_bip340_challenge(const u8* r32, const u8* px32, const u8* msg32, u8* out32) {
    sha256_bip340_challenge(out32, r32, px32, msg32);
}

// same-key path: table built once (sharedkey_build), ladder-only verification
void emul_verify_samekey(int kind, const u8* key, const u8* msg, const u8* sig, size_t n, u8* out) {
    build_gtable_fast();
    sv_shared_key sk;
    sharedkey_build(&sk, kind, key);
    for (size_t base = 0; base < n; base += SV_PREP_BATCH) {
        int cnt = (int)((n - base < SV_PREP_BATCH) ? (n - base) : SV_PREP_BATCH);
        sc r[SV_PREP_BATCH], m[SV_PREP_BATCH], sv[SV_PREP_BATCH];
        bool ok[SV_PREP_BATCH];
        for (int j = 0; j < cnt; j++) {
            sc s;
            ok[j] = ecdsa_parse(r[j], s, m[j], sig + 64 * (base + j), msg + 32 * (base + j), nullptr);
            if (!ok[j]) { memset(s.v, 0, 32); s.v[0] = 1; }
            sv[j] = s;
        }
        sc_batch_inverse(sv, cnt);
        for (int j = 0; j < cnt; j++) {
            sv_work w;
            ecdsa_finish_prep(w, ok[j], r[j], m[j], sv[j]);
            out[base + j] = (u8)verify_curve_side_shared(&w, sig + 64 * (base + j), g_table.data(), &sk);
        }
    }
}

int emul_bip143(const void* tx_item, const u8* blob, u8* out32) {
    sv_tx_item t;
    memcpy(&t, tx_item, sizeof t);
    return bip143_sighash(out32, t, blob) ? 1 : 0;
}
size_t emul_sizeof_tx_item(void) { return sizeof(sv_tx_item); }

void emul_gtable_build(void) { build_gtable_fast(); }

// the self-test cases of tests/selftest_cases.py against the host forms of the primitives
void emul_selftest(int op, const u32* a, const u32* b, size_t n, u32* out) {
    for (size_t i = 0; i < n; i++) selftest_item(op, a + 8 * i, b + 8 * i, out + 16 * i, g_table.data());
}
void emul_selftest_group(int op, const u32* in, size_t n, u32* out) {
    for (size_t i = 0; i < n; i++) selftest_group_item(op, in + SV_STG_IN_WORDS * i, out + SV_STG_OUT_WORDS * i, g_table.data());
}

// Branch log: emul_trace_begin() starts logging on the calling thread, emul_trace_end(out, cap) stops it, copies up to cap
// events to out and returns how many were logged.
static std::vector<unsigned char> g_trace_buf;
void emul_trace_begin(void) {
    g_trace_buf.clear();
    emul_trace_log() = &g_trace_buf;
}
size_t emul_trace_end(u8* out, size_t cap) {
    emul_trace_log() = nullptr;
    size_t n = g_trace_buf.size();
    if (out) memcpy(out, g_trace_buf.data(), n < cap ? n : cap);
    return n;
}
// entry computed the way the device kernel does it (double-and-add + Fermat), for cross-checking
void emul_gtable_entry_device_algo(u32 e, u32* xy16) {
    build_gtable_fast();
    std::vector<ge_mem> one(SV_GT_ENTRIES > 0 ? 1 : 1);
    // gtable_make_entry writes table[e]; give it a fake base pointer so that only slot e is touched
    ge_mem slot;
    gtable_make_entry(&slot - e, g_bases.data(), e);
    memcpy(xy16, slot.x, 32);
    memcpy(xy16 + 8, slot.y, 32);
}
void emul_gtable_get(u32 e, u32* xy16) {
    build_gtable_fast();
    memcpy(xy16, g_table[e].x, 32);
    memcpy(xy16 + 8, g_table[e].y, 32);
}

// the small-batch path (k_small): per item, the three warps' phases run one after another
void emul_verify_small_batch(int kind, const u8* msg, const u8* key, const u8* sig, size_t n, u8* out) {
    build_gtable_fast();
    size_t keylen = kind == SV_KIND_ECDSA33 ? 33 : (kind == SV_KIND_ECDSA_XY ? 64 : 32);
    sv_small_item it;
    for (size_t i = 0; i < n; i++)
        out[i] = (u8)verify_small_sequential(kind, msg + 32 * i, key + keylen * i, sig + 64 * i, g_table.data(), &it, !g_ecdsa33_exact);
}

// BIP-340 batch verification (batch.cuh), every stage on the host with the straightforward window sum: ok[i] = encoding
// check, group_ok[g] = the group's equation held
void emul_schnorr_batch(const u8* msg, const u8* xonly, const u8* sig, size_t n, const u8* seed32, u8* ok, u8* group_ok) {
    build_gtable_fast();
    std::vector<qtab_entry> pts(2 * n);
    std::vector<signed char> dig((size_t)SV_SB_WINDOWS * 4 * n);
    std::vector<sc> t(n);
    for (size_t i = 0; i < n; i++)
        ok[i] = sb_prepare(msg + 32 * i, xonly + 32 * i, sig + 64 * i, seed32, i, &pts[2 * i], &dig[4 * i], 4 * n, t[i]) ? 1 : 0;
    size_t groups = (n + SV_SB_GROUP - 1) / SV_SB_GROUP;
    for (size_t g = 0; g < groups; g++) {
        size_t first = g * SV_SB_GROUP, members = (n - first < SV_SB_GROUP) ? (n - first) : SV_SB_GROUP;
        sv_jac S[SV_SB_WINDOWS];
        for (int w = 0; w < SV_SB_WINDOWS; w++) {
            gej W;
            sb_window_sum_reference(W, &pts[2 * first], &dig[(size_t)w * 4 * n + 4 * first], (u32)(members * SV_SB_TERMS));
            small_jac_store(&S[w], W);
        }
        group_ok[g] = sb_group_check(S, &t[first], (u32)members, g_table.data()) ? 1 : 0;
    }
}

// the small-batch path with the half ladders on lane PAIRS (two host threads per half ladder), as k_small runs it
void emul_verify_small_pair_batch(int kind, const u8* msg, const u8* key, const u8* sig, size_t n, u8* out) {
    build_gtable_fast();
    size_t keylen = kind == SV_KIND_ECDSA33 ? 33 : (kind == SV_KIND_ECDSA_XY ? 64 : 32);
    sv_small_item it;
    for (size_t i = 0; i < n; i++) {
        const bool ns = !g_ecdsa33_exact && kind != SV_KIND_ECDSA_XY;  // as k_small<kind, true>
        if (ns) small_key_side_ns(kind, key + keylen * i, &it); else small_key_side(kind, key + keylen * i, &it);
        small_scalar_side(kind, msg + 32 * i, key + keylen * i, sig + 64 * i, &it);
        for (int half = 0; half < 2; half++) {
            pair_mailbox mb;
            std::thread other([&] { pair_lane L; L.role = 1; L.mb = &mb; small_half_ladder_pair(L, &it, half); });
            pair_lane L;
            L.role = 0;
            L.mb = &mb;
            small_half_ladder_pair(L, &it, half);
            other.join();
        }
        small_comb(&it, g_table.data());
        bool kd = false;
        out[i] = ns ? (u8)small_finish_ns(kind, &it, key + keylen * i, sig + 64 * i, g_table.data(), g_aux ? &kd : nullptr)
                    : (u8)small_finish(kind, &it, sig + 64 * i, &kd);
        if (g_aux) g_aux[i] = (u8)((kd ? 1u : 0u) | ((it.w.flags & SV_WF_PARSED) ? 2u : 0u));  // as k_small
    }
}
void emul_verify_small_pair_batch_aux(int kind, const u8* msg, const u8* key, const u8* sig, size_t n, u8* out, u8* aux) {
    g_aux = aux;
    emul_verify_small_pair_batch(kind, msg, key, sig, n, out);
    g_aux = nullptr;
}

// full verification of a batch, same data flow as the kernels (prep in groups of SV_PREP_BATCH)
void emul_verify_batch(int kind, const u8* msg, const u8* key, const u8* sig, size_t n, u8* out) {
    build_gtable_fast();
    size_t keylen = kind == SV_KIND_ECDSA33 ? 33 : (kind == SV_KIND_ECDSA_XY ? 64 : 32);
    std::vector<sv_work> work(n);
    if (kind == SV_KIND_SCHNORR) {
        for (size_t i = 0; i < n; i++) schnorr_prep(work[i], sig + 64 * i, key + keylen * i, msg + 32 * i);
    } else {
        for (size_t base = 0; base < n; base += SV_PREP_BATCH) {
            int cnt = (int)((n - base < SV_PREP_BATCH) ? (n - base) : SV_PREP_BATCH);
            sc r[SV_PREP_BATCH], m[SV_PREP_BATCH], sv[SV_PREP_BATCH];
            bool ok[SV_PREP_BATCH], parsed[SV_PREP_BATCH];
            for (int j = 0; j < cnt; j++) {
                sc s;
                ok[j] = ecdsa_parse(r[j], s, m[j], sig + 64 * (base + j), msg + 32 * (base + j), &parsed[j]);
                if (!ok[j]) { memset(s.v, 0, 32); s.v[0] = 1; }
                sv[j] = s;
            }
            sc_batch_inverse(sv, cnt);
            for (int j = 0; j < cnt; j++) ecdsa_finish_prep(work[base + j], ok[j], r[j], m[j], sv[j], parsed[j]);
        }
    }
    qtab_entry tab[8];
    if (kind == SV_KIND_SCHNORR && !g_ecdsa33_exact) {  // as k_main<BIP-340 without square root> + k_final_schnorr_ns
        size_t exact = 0;
        for (size_t i = 0; i < n; i++) {
            out[i] = (u8)schnorr_nosqrt_curve_side(&work[i], key + 32 * i, sig + 64 * i, g_table.data(), tab,
                                                   reinterpret_cast<sv_ns_park_schnorr*>(&work[i]), true);
            exact += out[i] == SV_NS_EXACT;
        }
        g_last_exact = exact;
        for (size_t base = 0; base < n; base += SV_FINAL_BATCH) {
            int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
            schnorr_nosqrt_final_batch(out + base, work.data() + base, key + 32 * base, sig + 64 * base, g_table.data(), cnt);
        }
        return;
    }
    if (kind == SV_KIND_SCHNORR) {  // as k_main<SCHNORR> + k_final_schnorr: park R, then batched inversion
        for (size_t i = 0; i < n; i++) {
            bool ok = (work[i].flags & SV_WF_VALID) != 0;
            ge Q;
            ok = key_decode(Q, kind, key + keylen * i) && ok;
            gej R;
            ecmult_uniform(R, &work[i], Q, g_table.data(), tab);
            schnorr_park(reinterpret_cast<sv_jac*>(&work[i]), R, ok);
        }
        for (size_t base = 0; base < n; base += SV_FINAL_BATCH) {
            int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
            schnorr_final_batch(out + base, reinterpret_cast<const sv_jac*>(work.data()) + base, sig + 64 * base, cnt);
        }
        return;
    }
    if (kind == SV_KIND_ECDSA33 && !g_ecdsa33_exact) {  // as k_main<ECDSA33 without square root> + k_final_ecdsa33
        size_t exact = 0;
        for (size_t i = 0; i < n; i++) {
            out[i] = (u8)ecdsa33_nosqrt_curve_side(&work[i], key + 33 * i, sig + 64 * i, g_table.data(), tab,
                                                   reinterpret_cast<sv_ns_park*>(&work[i]), true);
            exact += out[i] == SV_NS_EXACT;
        }
        g_last_exact = exact;
        for (size_t base = 0; base < n; base += SV_FINAL_BATCH) {
            int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
            ecdsa33_nosqrt_final_batch(out + base, work.data() + base, key + 33 * base, sig + 64 * base, g_table.data(), cnt,
                                       g_aux ? g_aux + base : nullptr);
        }
        return;
    }
    for (size_t i = 0; i < n; i++) {
        bool kd;
        out[i] = (u8)verify_curve_side(kind, &work[i], key + keylen * i, sig + 64 * i, g_table.data(), tab, &kd);
        if (g_aux) g_aux[i] = (u8)((kd ? 1u : 0u) | ((work[i].flags & SV_WF_PARSED) ? 2u : 0u));  // as k_main
    }
}
// ECDSA kinds, with the per-item byte the gossip path consumes: bit 0 = key decodes, bit 1 = r, s < n
void emul_verify_batch_aux(int kind, const u8* msg, const u8* key, const u8* sig, size_t n, u8* out, u8* aux) {
    g_aux = aux;
    emul_verify_batch(kind, msg, key, sig, n, out);
    g_aux = nullptr;
}
// Algebra of the linear form (verify.cuh ns_linear_form) against the plain Jacobian addition.  P1, P2: affine curve points
// (x || y, 8 limbs each), zr, tz, y: non-zero field elements.  S = P1 in Jacobian coordinates with Z = zr, written as
// (X, Y, y * Zs) with Zs = zr / y; T = P2 with Z = tz; c = y^2; r = x(S + T).  Checked: D == y*B, N == Y3*B, CG*y == Z3^3,
// and that r + 1 breaks D == y*B.  Returns a bit per check (15 = all hold), or -1 if the form reports an exceptional input.
int emul_ns_linear_check(const u32* p1, const u32* p2, const u32* zr_, const u32* tz_, const u32* y_) {
    fe x1, y1, x2, y2, zr, tz, y, t, zz;
    for (int i = 0; i < 8; i++) { x1.v[i] = p1[i]; y1.v[i] = p1[8 + i]; x2.v[i] = p2[i]; y2.v[i] = p2[8 + i]; zr.v[i] = zr_[i]; tz.v[i] = tz_[i]; y.v[i] = y_[i]; }
    gej S, T, R;
    fe_sqr(zz, zr); fe_mul(S.x, x1, zz); fe_mul(t, zz, zr); fe_mul(S.y, y1, t); S.z = zr; S.inf = 0;
    fe_sqr(zz, tz); fe_mul(T.x, x2, zz); fe_mul(t, zz, tz); fe_mul(T.y, y2, t); T.z = tz; T.inf = 0;
    gej_add_gej(R, S, T);
    if (R.inf) return -1;
    fe c, yi, Zs, zi, rfe, D, B, ext[2];
    fe_sqr(c, y);
    fe_inv(yi, y);
    fe_mul(Zs, zr, yi);
    fe_inv(zi, R.z);
    fe_sqr(t, zi);
    fe_mul(rfe, R.x, t);  // affine x of S + T
    fe_normalize(rfe);
    if (ns_linear_form(D, B, S.x, S.y, Zs, T, c, rfe, ext)) return -1;
    int ok = 0;
    fe_mul(t, y, B);
    if (fe_equal(t, D)) ok |= 1;
    fe_mul(t, R.y, B);
    if (fe_equal(t, ext[0])) ok |= 2;
    fe z3c;
    fe_sqr(z3c, R.z); fe_mul(z3c, z3c, R.z);
    fe_mul(t, ext[1], y);
    if (fe_equal(t, z3c)) ok |= 4;
    fe one, r2, D2, B2;
    fe_set_u32(one, 1);
    fe_add(r2, rfe, one);
    ns_linear_form(D2, B2, S.x, S.y, Zs, T, c, r2);
    fe_mul(t, y, B2);
    if (!fe_equal(t, D2) && fe_equal(B2, B)) ok |= 8;
    return ok;
}
// kinds ECDSA33 and SCHNORR: 1 = the plain flow with the square root, 0 = the flow without it (the engine's default)
void emul_set_ecdsa33_exact(int on) { g_ecdsa33_exact = on; }
size_t emul_last_exact_count(void) { return g_last_exact; }
}
