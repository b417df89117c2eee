// sc.cuh — arithmetic modulo the group order n and the scalar-side preparation of a verify.
//
// Semantics follow the reference's scalar module (libsecp256k1 scalar_4x64_impl.h, scalar_impl.h;
// cited per function); representation is 8x32-bit limbs, always fully reduced (< n).  Scalar work
// is a few percent of a verification, so this file favours clarity: products go through the same
// IMAD.WIDE 256x256 multiplier as the field code, everything else is plain 64-bit column code.
#pragma once
#include "u256.cuh"

struct sc {
    u32 v[8];
};

// group order n (reference: scalar_4x64_impl.h:16-20), 2^256-n (:23-25), (n-1)/2 (:28-31)
static SV_CDATA const u32 SC_N[8] = {0xD0364141u, 0xBFD25E8Cu, 0xAF48A03Bu, 0xBAAEDCE6u,
                                     0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
static SV_CDATA const u32 SC_NC[5] = {0x2FC9BEBFu, 0x402DA173u, 0x50B75FC4u, 0x45512319u, 0x00000001u};
static SV_CDATA const u32 SC_NHALF[8] = {0x681B20A0u, 0xDFE92F46u, 0x57A4501Du, 0x5D576E73u,
                                         0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0x7FFFFFFFu};
// GLV constants (reference: scalar_impl.h:79-82 lambda; :140-155 g1, g2, -b1, -b2)
static SV_CDATA const u32 SC_MINUS_LAMBDA[8] = {0xB51283CFu, 0xE0CFC810u, 0x8EC739C2u, 0xA880B9FCu,
                                                0x77ED9BA4u, 0x5AD9E3FDu, 0x3FA3CF1Fu, 0xAC9C52B3u};
static SV_CDATA const u32 SC_G1[8] = {0x45DBB031u, 0xE893209Au, 0x71E8CA7Fu, 0x3DAA8A14u,
                                      0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u};
static SV_CDATA const u32 SC_G2[8] = {0x8AC47F71u, 0x1571B4AEu, 0x9DF506C6u, 0x221208ACu,
                                      0x0ABFE4C4u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u};
static SV_CDATA const u32 SC_MINUS_B1[8] = {0x0ABFE4C3u, 0x6F547FA9u, 0x010E8828u, 0xE4437ED6u, 0, 0, 0, 0};
static SV_CDATA const u32 SC_MINUS_B2[8] = {0x3DB1562Cu, 0xD765CDA8u, 0x0774346Du, 0x8A280AC5u,
                                            0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
// lattice vectors (a,b) with a + b*lambda == 0 (mod n), 160-bit two's complement, used to force
// both GLV halves odd:  v1 = (a1, b1), v2 = (a2, b2 = a1)
static SV_CDATA const u32 SC_LAT_A1[5] = {0x9284EB15u, 0xE86C90E4u, 0xA7D46BCDu, 0x3086D221u, 0x00000000u};
static SV_CDATA const u32 SC_LAT_B1[5] = {0xF5401B3Du, 0x90AB8056u, 0xFEF177D7u, 0x1BBC8129u, 0xFFFFFFFFu};  // -0xE4437ED6010E88286F547FA90ABFE4C3
static SV_CDATA const u32 SC_LAT_A2[5] = {0x9D44CFD8u, 0x57C1108Du, 0xA8E2F3F6u, 0x14CA50F7u, 0x00000001u};
static SV_CDATA const u32 SC_LAT_A1PA2[5] = {0x2FC9BAEDu, 0x402DA172u, 0x50B75FC4u, 0x45512319u, 0x00000001u};
static SV_CDATA const u32 SC_LAT_B1PB2[5] = {0x87C50652u, 0x7918113Bu, 0xA6C5E3A5u, 0x4C43534Bu, 0xFFFFFFFFu};
// n - 2 (Fermat exponent)
static SV_CDATA const u32 SC_NM2[8] = {0xD036413Fu, 0xBFD25E8Cu, 0xAF48A03Bu, 0xBAAEDCE6u,
                                       0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};

SV_HD bool sc_is_zero(const sc& a) { return u256_is_zero(a.v); }
SV_HD bool sc_gte_n(const u32 a[8]) { return u256_gte(a, SC_N); }

// big-endian 32 bytes -> scalar reduced mod n; *overflow = (value >= n)
// reference: secp256k1_scalar_set_b32 (scalar_4x64_impl.h:158-170)
SV_HD void sc_set_b32(sc& r, const u8* b, bool* overflow) {
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        const u8* q = b + 28 - 4 * i;
        r.v[i] = ((u32)q[0] << 24) | ((u32)q[1] << 16) | ((u32)q[2] << 8) | (u32)q[3];
    }
    u32 t[8];
    u32 bw = u256_sub(t, r.v, SC_N);
    bool over = (bw == 0);
    if (over) {
        SV_UNROLL
        for (int i = 0; i < 8; i++) r.v[i] = t[i];
    }
    if (overflow) *overflow = over;
}
SV_HD void sc_get_b32(u8* b, const sc& a) {
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        u8* q = b + 28 - 4 * i;
        q[0] = (u8)(a.v[i] >> 24);
        q[1] = (u8)(a.v[i] >> 16);
        q[2] = (u8)(a.v[i] >> 8);
        q[3] = (u8)a.v[i];
    }
}

// a > (n-1)/2 ?   reference: secp256k1_scalar_is_high (scalar_4x64_impl.h:255-267)
SV_HD bool sc_is_high(const sc& a) {
    u32 t[8];
    return u256_sub(t, SC_NHALF, a.v) != 0;  // borrow <=> a > nhalf
}

// r = -a mod n  (0 -> 0)   reference: secp256k1_scalar_negate (scalar_4x64_impl.h:217)
SV_HD void sc_negate(sc& r, const sc& a) {
    bool z = sc_is_zero(a);
    u32 t[8];
    u256_sub(t, SC_N, a.v);
    SV_UNROLL
    for (int i = 0; i < 8; i++) r.v[i] = z ? 0u : t[i];
}

// r = a + b mod n   reference: secp256k1_scalar_add (scalar_4x64_impl.h:110)
SV_HD void sc_add(sc& r, const sc& a, const sc& b) {
    u32 s[8], t[8];
    u32 c = u256_add(s, a.v, b.v);
    u32 bw = u256_sub(t, s, SC_N);
    bool use_t = c || (bw == 0);
    SV_UNROLL
    for (int i = 0; i < 8; i++) r.v[i] = use_t ? t[i] : s[i];
}

// 512-bit -> mod n, by folding with 2^256 == NC (mod n), NC = 2^256 - n (129 bits)
// reference: secp256k1_scalar_reduce_512 (scalar_4x64_impl.h:384) — same idea, other limb size
SV_HD void sc_reduce512(sc& r, const u32 t[16]) {
#if SV_DEVICE_CODE
    // Device form: NC = 2^128 + c with a 4-limb c, so a fold is one 8x4 (then 5x4) IMAD.WIDE product plus a limb-shifted
    // add; both folds are one generated PTX body (tools/gen_mul.py, checked there against big-int arithmetic).  Same
    // folds, same intermediate values as the portable code below.
    u32 B[9];
    sv_sc_fold2_dev(B, t);
    // fold 3: B[8] < 8
    u32 kc[8];
    {
        u64 acc = 0;
        SV_UNROLL
        for (int i = 0; i < 5; i++) {
            acc += (u64)B[8] * SC_NC[i];
            kc[i] = (u32)acc;
            acc >>= 32;
        }
        kc[5] = kc[6] = kc[7] = 0;
    }
    u32 s[8];
    u32 c = u256_add(s, B, kc);
    // fold 4: possible carry (value then tiny), then the final conditional subtraction
    u32 mask = 0u - c;
    SV_UNROLL
    for (int i = 0; i < 8; i++) kc[i] = (i < 5) ? (SC_NC[i] & mask) : 0u;
    (void)u256_add(s, s, kc);
    u32 tt[8];
    u32 bw = u256_sub(tt, s, SC_N);
    SV_UNROLL
    for (int i = 0; i < 8; i++) r.v[i] = (bw == 0) ? tt[i] : s[i];
#else
    // fold 1: m[0..12] = t[0..7] + t[8..15] * NC           (< 2^386)
    u32 m[14];
    {
        u64 acc = 0, hi = 0;  // acc: running column sum (needs > 64 bits: keep overflow in hi)
        SV_UNROLL
        for (int k = 0; k < 13; k++) {
            if (k < 8) { acc += t[k]; }
            SV_UNROLL
            for (int j = 0; j < 5; j++) {
                int i = k - j;
                if (i >= 0 && i < 8) {
                    u64 p = (u64)t[8 + i] * SC_NC[j];
                    u64 old = acc;
                    acc += p;
                    hi += (acc < old);
                }
            }
            m[k] = (u32)acc;
            acc = (acc >> 32) | (hi << 32);
            hi = 0;
        }
        m[13] = (u32)acc;
    }
    // fold 2: q[0..8] = m[0..7] + m[8..13] * NC            (m[8..13] < 2^131 -> < 2^261)
    u32 q[10];
    {
        u64 acc = 0, hi = 0;
        SV_UNROLL
        for (int k = 0; k < 10; k++) {
            if (k < 8) { acc += m[k]; }
            SV_UNROLL
            for (int j = 0; j < 5; j++) {
                int i = k - j;
                if (i >= 0 && i < 6) {
                    u64 p = (u64)m[8 + i] * SC_NC[j];
                    u64 old = acc;
                    acc += p;
                    hi += (acc < old);
                }
            }
            q[k] = (u32)acc;
            acc = (acc >> 32) | (hi << 32);
            hi = 0;
        }
    }
    // fold 3: q[8] (< 2^6), q[9] == 0
    u32 s[8];
    u64 acc = 0;
    SV_UNROLL
    for (int k = 0; k < 8; k++) {
        acc += q[k];
        if (k < 5) acc += (u64)q[8] * SC_NC[k];
        s[k] = (u32)acc;
        acc >>= 32;
    }
    // fold 4: possible carry (value then tiny) + final conditional subtraction
    u32 c = (u32)acc;
    acc = 0;
    SV_UNROLL
    for (int k = 0; k < 8; k++) {
        acc += s[k];
        if (k < 5) acc += (u64)c * SC_NC[k];
        s[k] = (u32)acc;
        acc >>= 32;
    }
    u32 tt[8];
    u32 bw = u256_sub(tt, s, SC_N);
    SV_UNROLL
    for (int i = 0; i < 8; i++) r.v[i] = (bw == 0) ? tt[i] : s[i];
#endif
}

// reference: secp256k1_scalar_mul (scalar_4x64_impl.h:1009)
SV_HD void sc_mul(sc& r, const sc& a, const sc& b) {
    u32 t[16];
    u256_mul_wide(t, a.v, b.v);
    sc_reduce512(r, t);
}
SV_HD void sc_sqr(sc& r, const sc& a) {
    u32 t[16];
    u256_sqr_wide(t, a.v);  // dedicated squaring: 36 products instead of 64
    sc_reduce512(r, t);
}

// r = a^(n-2) = 1/a mod n (0 -> 0).  The reference uses safegcd (secp256k1_scalar_inverse_var,
// scalar_4x64_impl.h:1139 -> modinv64_impl.h:638): data-dependent branching, poor fit for SIMT.
// A fixed 4-bit-window exponentiation is uniform across lanes; callers amortise it with
// Montgomery's trick over several signatures (see sc_batch_inverse).
SV_HD void sc_inverse(sc& r, const sc& a) {
    sc tbl[16];  // tbl[i] = a^i
    tbl[1] = a;
    sc_sqr(tbl[2], a);
#if SV_DEVICE_CODE
#pragma unroll 1
#endif
    for (int i = 3; i < 16; i++) sc_mul(tbl[i], tbl[i - 1], a);
    sc acc = tbl[15];  // top nibble of n-2 is 0xF
#if SV_DEVICE_CODE
#pragma unroll 1
#endif
    for (int i = 62; i >= 0; i--) {
        sc_sqr(acc, acc);
        sc_sqr(acc, acc);
        sc_sqr(acc, acc);
        sc_sqr(acc, acc);
        u32 nib = (SC_NM2[i >> 3] >> ((i & 7) * 4)) & 15u;
        if (nib) sc_mul(acc, acc, tbl[nib]);
    }
    r = acc;
}

// 1/a mod n by binary extended Euclid (variable time; 0 -> 0): the inversion of ONE scalar on the critical path of the
// small-batch kernel.  Same value as sc_inverse.
SV_HD void sc_inverse_var(sc& r, const sc& a) { u256_modinv_var(r.v, a.v, SC_N); }

// (a*b) >> 384 rounded to nearest: reference secp256k1_scalar_mul_shift_var (scalar_4x64_impl.h:1049)
SV_HD void sc_mul_shift384(sc& r, const sc& a, const u32 b[8]) {
    u32 t[16];
    u256_mul_wide(t, a.v, b);
    u32 rnd = (t[11] >> 31) & 1u;
    u64 acc = rnd;
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        if (i < 4) acc += t[12 + i];
        r.v[i] = (u32)acc;
        acc >>= 32;
    }
}

// GLV decomposition k = r1 + r2*lambda (mod n) with |r1|,|r2| < 2^128 as signed residues.
// reference: secp256k1_scalar_split_lambda (scalar_impl.h:138-176)
SV_HD void sc_split_lambda(sc& r1, sc& r2, const sc& k) {
    sc c1, c2, mb1, mb2, ml;
    SV_UNROLL
    for (int i = 0; i < 8; i++) { mb1.v[i] = SC_MINUS_B1[i]; mb2.v[i] = SC_MINUS_B2[i]; ml.v[i] = SC_MINUS_LAMBDA[i]; }
    sc_mul_shift384(c1, k, SC_G1);
    sc_mul_shift384(c2, k, SC_G2);
    sc_mul(c1, c1, mb1);
    sc_mul(c2, c2, mb2);
    sc_add(r2, c1, c2);
    sc_mul(r1, r2, ml);
    sc_add(r1, r1, k);
}

// -------------------------------------------------------------------------------------------------
// Work record: everything the EC kernel needs from the scalar side of one verification,
// R = u1*G + u2*Q with u2 = k1 + k2*lambda.  128 bytes, 16-byte aligned (LDG.128 x 8).
// -------------------------------------------------------------------------------------------------
struct sv_work {
    u32 k1[5];   // |k1| (odd, < 2^131); bit 31 of k1[4] = sign of k1
    u32 k2[5];   // |k2| likewise
    int gd[16];  // comb digits of u1: u1 = sum gd[i] * 2^(16 i); gd[0..14] in [-32768, 32768], gd[15] in [0, 65536]
    u32 flags;   // SV_WF_*
    u32 pad[5];
};
#define SV_WF_VALID 1u       // scalar-side checks passed (range checks; s != 0 ...)
#define SV_WF_R_PLUS_N 2u    // ECDSA: r < p - n, so r + n is a second x candidate
#define SV_WF_PARSED 4u      // r < n and s < n: secp256k1_ecdsa_signature_parse_compact would accept the encoding

// 160-bit two's complement helpers (5 limbs)
SV_HD void s160_add(u32 r[5], const u32 a[5], const u32 b[5]) {
    u64 c = 0;
    SV_UNROLL
    for (int i = 0; i < 5; i++) { c += (u64)a[i] + b[i]; r[i] = (u32)c; c >>= 32; }
}
SV_HD void s160_neg(u32 r[5], const u32 a[5]) {
    u64 c = 1;
    SV_UNROLL
    for (int i = 0; i < 5; i++) { c += (u64)(~a[i]); r[i] = (u32)c; c >>= 32; }
}

// Split u2, force both halves odd (adding a lattice vector leaves k1 + k2*lambda unchanged mod n),
// and emit sign/magnitude.  Odd halves let the EC kernel use a *regular* signed-odd-digit window
// recoding: every 4-bit window is a non-zero odd digit in +-{1..15}, so all lanes of a warp add
// at the same ladder steps (a wNAF like the reference's ecmult_impl.h:162-218 would diverge).
SV_HD void sc_prepare_u2(sv_work& w, const sc& u2) {
    sc r1, r2;
    sc_split_lambda(r1, r2, u2);
    u32 a[5], b[5];
    bool n1 = sc_is_high(r1), n2 = sc_is_high(r2);
    sc t;
    if (n1) sc_negate(t, r1); else t = r1;
    SV_UNROLL
    for (int i = 0; i < 5; i++) a[i] = t.v[i];
    if (n1) s160_neg(a, a);
    if (n2) sc_negate(t, r2); else t = r2;
    SV_UNROLL
    for (int i = 0; i < 5; i++) b[i] = t.v[i];
    if (n2) s160_neg(b, b);
    bool o1 = a[0] & 1u, o2 = b[0] & 1u;
    if (!o1 && !o2) { s160_add(a, a, SC_LAT_A1); s160_add(b, b, SC_LAT_B1); }
    else if (o1 && !o2) { s160_add(a, a, SC_LAT_A2); s160_add(b, b, SC_LAT_A1); }
    else if (!o1 && o2) { s160_add(a, a, SC_LAT_A1PA2); s160_add(b, b, SC_LAT_B1PB2); }
    u32 s1 = a[4] >> 31, s2 = b[4] >> 31;
    if (s1) s160_neg(a, a);
    if (s2) s160_neg(b, b);
    SV_UNROLL
    for (int i = 0; i < 5; i++) { w.k1[i] = a[i]; w.k2[i] = b[i]; }
    w.k1[4] |= s1 << 31;
    w.k2[4] |= s2 << 31;
}

// Signed 16-bit comb digits of u1 for the fixed-base table (see gtable.cuh).
SV_HD void sc_prepare_u1(sv_work& w, const sc& u1) {
    u32 carry = 0;
    SV_UNROLL
    for (int i = 0; i < 16; i++) {
        u32 win = (u1.v[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu;
        win += carry;
        if (i < 15 && win > 0x8000u) {
            w.gd[i] = (int)win - 0x10000;
            carry = 1;
        } else {
            w.gd[i] = (int)win;
            carry = 0;
        }
    }
}
