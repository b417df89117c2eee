// selftest.cuh — ONE primitive of the engine's arithmetic on caller operands (test support).
//
// Shared by the k_selftest kernel (engine.cu; the inline-PTX device forms, reached through sv_selftest_host) and by
// tests/host_emul (the uint64 host forms), so that the same test code runs against both.  Operands A, B are 8
// little-endian 32-bit limbs each, R receives 16 limbs (see the SV_ST_* list in include/cln_sigverify.h).
// Model: libsecp256k1 tests.c:3023-3176 (field self-tests), :2354 (scalar tests).
#pragma once
#include "../../include/cln_sigverify.h"
#include "verify.cuh"

SV_HD void selftest_item(int op, const u32 A[8], const u32 B[8], u32 R[16], const ge_mem* gtab) {
    SV_UNROLL
    for (int k = 0; k < 16; k++) R[k] = 0;
    fe x, y, r;
    sc p, q, s;
SV_UNROLL
    for (int k = 0; k < 8; k++) { x.v[k] = A[k]; y.v[k] = B[k]; p.v[k] = A[k]; q.v[k] = B[k]; }
    fe_set_zero(r);
    bool is_fe = false, is_sc = false;
    switch (op) {
        case SV_ST_FE_MUL: fe_mul(r, x, y); is_fe = true; break;
        case SV_ST_FE_SQR: fe_sqr(r, x); is_fe = true; break;
        case SV_ST_FE_ADD: fe_add(r, x, y); is_fe = true; break;
        case SV_ST_FE_SUB: fe_sub(r, x, y); is_fe = true; break;
        case SV_ST_FE_NEG: fe_neg(r, x); is_fe = true; break;
        case SV_ST_FE_NORMALIZE: r = x; fe_normalize(r); is_fe = true; R[8] = fe_is_zero(x); R[9] = fe_gte_p(x); R[10] = fe_equal(x, y); break;
        case SV_ST_FE_INV: fe_inv(r, x); is_fe = true; break;
        case SV_ST_FE_SQRT: R[8] = fe_sqrt(r, x) ? 1u : 0u; is_fe = true; break;
        case SV_ST_FE_MUL3: fe_mul3(r, x); is_fe = true; break;
        case SV_ST_FE_MUL8: fe_mul8(r, x); is_fe = true; break;
        case SV_ST_FE_MUL_SMALL: fe_mul_small(r, x, B[0] & 0xFFFFu); is_fe = true; break;
        case SV_ST_FE_DBL: fe_dbl(r, x); is_fe = true; break;
        case SV_ST_FE_B32: {  // set_b32 / get_b32 round trip of the big-endian bytes held in A (as memory order)
            u8 bytes[32], back[32];
SV_UNROLL
            for (int k = 0; k < 8; k++) { bytes[4 * k] = (u8)A[k]; bytes[4 * k + 1] = (u8)(A[k] >> 8); bytes[4 * k + 2] = (u8)(A[k] >> 16); bytes[4 * k + 3] = (u8)(A[k] >> 24); }
            R[8] = fe_set_b32(r, bytes) ? 1u : 0u;
            fe_get_b32(back, r);
SV_UNROLL
            for (int k = 0; k < 8; k++) R[k] = (u32)back[4 * k] | ((u32)back[4 * k + 1] << 8) | ((u32)back[4 * k + 2] << 16) | ((u32)back[4 * k + 3] << 24);
            break;
        }
        case SV_ST_U256_MUL_WIDE: u256_mul_wide(R, A, B); break;
        case SV_ST_U256_SQR_WIDE: u256_sqr_wide(R, A); break;
        case SV_ST_FE_REDUCE512: {
            u32 t[16];
SV_UNROLL
            for (int k = 0; k < 8; k++) { t[k] = A[k]; t[8 + k] = B[k]; }
            fe_reduce512(r, t);
            is_fe = true;
            break;
        }
        case SV_ST_U256_ADD: R[8] = u256_add(R, A, B); break;
        case SV_ST_U256_SUB: R[8] = u256_sub(R, A, B); break;
        case SV_ST_SC_MUL: sc_mul(s, p, q); is_sc = true; break;
        case SV_ST_SC_SQR: sc_sqr(s, p); is_sc = true; break;
        case SV_ST_SC_ADD: sc_add(s, p, q); is_sc = true; break;
        case SV_ST_SC_NEGATE: sc_negate(s, p); is_sc = true; R[8] = sc_is_high(p); R[9] = sc_is_zero(p); R[10] = sc_gte_n(A); break;
        case SV_ST_SC_INVERSE: sc_inverse(s, p); is_sc = true; break;
        case SV_ST_SC_INVERSE_VAR: sc_inverse_var(s, p); is_sc = true; break;
        case SV_ST_FE_INV_VAR: fe_inv_var(r, x); is_fe = true; break;
        case SV_ST_SC_REDUCE512: {
            u32 t[16];
SV_UNROLL
            for (int k = 0; k < 8; k++) { t[k] = A[k]; t[8 + k] = B[k]; }
            sc_reduce512(s, t);
            is_sc = true;
            break;
        }
        case SV_ST_SC_SPLIT_LAMBDA: {
            sc r1, r2;
            sc_split_lambda(r1, r2, p);
SV_UNROLL
            for (int k = 0; k < 8; k++) { R[k] = r1.v[k]; R[8 + k] = r2.v[k]; }
            break;
        }
        case SV_ST_SC_SET_B32: {  // scalar_set_b32 of the 32 bytes held in A (memory order): reduced value + overflow flag
            u8 bytes[32];
            bool ov;
SV_UNROLL
            for (int k = 0; k < 8; k++) { bytes[4 * k] = (u8)A[k]; bytes[4 * k + 1] = (u8)(A[k] >> 8); bytes[4 * k + 2] = (u8)(A[k] >> 16); bytes[4 * k + 3] = (u8)(A[k] >> 24); }
            sc_set_b32(s, bytes, &ov);
            is_sc = true;
            R[8] = ov ? 1u : 0u;
            break;
        }
        case SV_ST_ECMULT_GEN: {  // A = scalar k (< n): affine k*G through the fixed-base comb table (x -> R[0..7], y -> R[8..15])
            ge P;
            if (sc_is_zero(p)) break;  // infinity: all-zero output
            ecmult_gen_comb(P, p, gtab);
SV_UNROLL
            for (int k = 0; k < 8; k++) { R[k] = P.x.v[k]; R[8 + k] = P.y.v[k]; }
            break;
        }
        case SV_ST_PREPARE_U2: {  // B = u2: GLV split forced odd, sign/magnitude halves as the work record stores them
            sv_work w;
            sc_prepare_u2(w, q);
SV_UNROLL
            for (int k = 0; k < 5; k++) { R[k] = w.k1[k]; R[5 + k] = w.k2[k]; }
            break;
        }
        case SV_ST_PREPARE_U1: {  // A = u1: the 16 signed comb digits
            sv_work w;
            sc_prepare_u1(w, p);
SV_UNROLL
            for (int k = 0; k < 16; k++) R[k] = (u32)w.gd[k];
            break;
        }
        default: break;
    }
    if (is_fe) {
SV_UNROLL
        for (int k = 0; k < 8; k++) R[k] = r.v[k];
    }
    if (is_sc) {
SV_UNROLL
        for (int k = 0; k < 8; k++) R[k] = s.v[k];
    }
}

// ONE group-law operation or scalar-multiplication schedule of the engine on a caller record (test support): IN holds
// SV_STG_IN_WORDS words, OUT receives SV_STG_OUT_WORDS (layouts in the SV_STG_* list of include/cln_sigverify.h).  Every op
// calls the production function unchanged.
SV_HD void stg_load_gej(gej& r, const u32* w) {
    for (int k = 0; k < 8; k++) { r.x.v[k] = w[k]; r.y.v[k] = w[8 + k]; r.z.v[k] = w[16 + k]; }
    r.inf = w[24];
}
SV_HD void stg_store_gej(u32* w, const gej& r) {
    for (int k = 0; k < 8; k++) { w[k] = r.x.v[k]; w[8 + k] = r.y.v[k]; w[16 + k] = r.z.v[k]; }
    w[24] = r.inf;
}
SV_HD void stg_load_fe(fe& r, const u32* w) {
    for (int k = 0; k < 8; k++) r.v[k] = w[k];
}
SV_HD void stg_store_fe(u32* w, const fe& r) {
    for (int k = 0; k < 8; k++) w[k] = r.v[k];
}
SV_HD void stg_load_work(sv_work& w, const u32* in) {  // k1 <- in[32..36], k2 <- in[40..44], u1 <- in[48..55] (comb digits)
    for (int k = 0; k < 5; k++) { w.k1[k] = in[32 + k]; w.k2[k] = in[40 + k]; w.pad[k] = 0; }
    sc u1;
    for (int k = 0; k < 8; k++) u1.v[k] = in[48 + k];
    sc_prepare_u1(w, u1);
    w.flags = SV_WF_VALID;
}

SV_HD void selftest_group_item(int op, const u32* in, u32* out, const ge_mem* gtab) {
    for (int k = 0; k < SV_STG_OUT_WORDS; k++) out[k] = 0;
    gej a, b, r;
    ge q;
    qtab_entry tab[8];
    fe zc;
    switch (op) {
        case SV_STG_GEJ_DOUBLE:
            stg_load_gej(a, in);
            gej_double(r, a);
            stg_store_gej(out, r);
            break;
        case SV_STG_GEJ_ADD_GE: {
            fe rzr;
            fe_set_zero(rzr);
            stg_load_gej(a, in);
            stg_load_fe(q.x, in + 32);
            stg_load_fe(q.y, in + 40);
            r = a;
            if (in[60] & 1u) gej_add_ge(r, r, q, &rzr); else gej_add_ge(r, a, q, &rzr);  // in[60] bit 0: r aliases a
            stg_store_gej(out, r);
            stg_store_fe(out + 32, rzr);
            break;
        }
        case SV_STG_GEJ_ADD_GEJ:
            stg_load_gej(a, in);
            stg_load_gej(b, in + 32);
            if (in[60] == 1u) { gej_add_gej(a, a, b); r = a; }       // r aliases a
            else if (in[60] == 2u) { gej_add_gej(b, a, b); r = b; }  // r aliases b
            else gej_add_gej(r, a, b);
            stg_store_gej(out, r);
            break;
        case SV_STG_GE_SET_XO: {
            fe x;
            stg_load_fe(x, in);
            out[16] = ge_set_xo(q, x, in[8] != 0) ? 1u : 0u;
            stg_store_fe(out, q.x);
            stg_store_fe(out + 8, q.y);
            break;
        }
        case SV_STG_QTABLE_BUILD:
            stg_load_fe(q.x, in);
            stg_load_fe(q.y, in + 8);
            qtable_build(tab, zc, q);
            for (int e = 0; e < 8; e++)
                for (int k = 0; k < 8; k++) { out[24 * e + k] = tab[e].x[k]; out[24 * e + 8 + k] = tab[e].y[k]; out[24 * e + 16 + k] = tab[e].h[k]; }
            stg_store_fe(out + 192, zc);
            break;
        case SV_STG_ECMULT_LADDER_Q:
        case SV_STG_ECMULT_HALF_LADDER:
        case SV_STG_ECMULT_LADDER: {
            sv_work w;
            stg_load_work(w, in);
            stg_load_fe(q.x, in);
            stg_load_fe(q.y, in + 8);
            qtable_build(tab, zc, q);
            if (op == SV_STG_ECMULT_LADDER_Q) ecmult_ladder_q(r, &w, tab, zc);
            else if (op == SV_STG_ECMULT_LADDER) ecmult_ladder(r, &w, gtab, tab, zc);
            else ecmult_half_ladder(r, w.k1, in[60] != 0, tab);  // on the scaled curve: true Z = Z * zc
            stg_store_gej(out, r);
            stg_store_fe(out + 32, zc);
            break;
        }
        case SV_STG_ECMULT_COMB_ADD: {
            sv_work w;
            stg_load_work(w, in);
            stg_load_gej(r, in);
            ecmult_comb_add(r, &w, gtab);
            stg_store_gej(out, r);
            break;
        }
        case SV_STG_SMALL_COMB: {
            sv_small_item it;
            stg_load_work(it.w, in);
            small_comb(&it, gtab);
            small_jac_load(r, &it.p3);
            stg_store_gej(out, r);
            break;
        }
        case SV_STG_NS_LINEAR_FORM: {
            fe X1, Y1, Zs, c, rfe, D, B, ext[2];
            stg_load_fe(X1, in);
            stg_load_fe(Y1, in + 8);
            stg_load_fe(Zs, in + 16);
            stg_load_fe(c, in + 24);
            stg_load_gej(b, in + 32);
            stg_load_fe(rfe, in + 56);
            out[32] = ns_linear_form(D, B, X1, Y1, Zs, b, c, rfe, ext) ? 1u : 0u;
            stg_store_fe(out, D);
            stg_store_fe(out + 8, B);
            stg_store_fe(out + 16, ext[0]);
            stg_store_fe(out + 24, ext[1]);
            break;
        }
        default: break;
    }
}
