// fe.cuh — arithmetic in F_p, p = 2^256 - 2^32 - 977 (secp256k1 base field).
//
// Mirrors the *semantics* of the reference's field module (libsecp256k1 field.h / field_impl.h /
// field_5x52_impl.h, cited per function) but not its representation: the reference uses 5x52-bit
// lazily-reduced limbs with magnitude tracking (field_5x52.h:14-34); here an element is 8x32-bit
// saturated limbs holding ANY value in [0, 2^256) congruent to the residue ("weak" form).  Only
// fe_normalize() produces the canonical representative, and only comparisons / byte export need it.
// Reduction uses 2^256 == 2^32 + 977 (mod p) (reference constant: field_5x52_impl.h:482), folded
// twice; no Montgomery form is needed for this prime (saves a second 64-IMAD product per multiply).
#pragma once
#include "u256.cuh"

struct fe {
    u32 v[8];
};

#define SV_P0 0xFFFFFC2Fu
#define SV_P1 0xFFFFFFFEu
#define SV_PC 977u  // 2^256 mod p = 2^32 + 977

SV_HD void fe_set_zero(fe& r) {
    SV_UNROLL
    for (int i = 0; i < 8; i++) r.v[i] = 0;
}
SV_HD void fe_set_u32(fe& r, u32 x) {
    fe_set_zero(r);
    r.v[0] = x;
}

// value >= p ?   (p = FFFFFFFF x6, FFFFFFFE, FFFFFC2F)
SV_HD bool fe_gte_p(const fe& a) {
    u32 hi = a.v[7] & a.v[6] & a.v[5] & a.v[4] & a.v[3] & a.v[2];
    return (hi == 0xFFFFFFFFu) && ((a.v[1] == 0xFFFFFFFFu) || (a.v[1] == SV_P1 && a.v[0] >= SV_P0));
}

// canonical representative in [0,p)   (reference: secp256k1_fe_normalize_var, field_5x52_impl.h:106)
SV_HD void fe_normalize(fe& a) {
    if (fe_gte_p(a)) {
        // a - p = a + (2^32 + 977) - 2^256 ; a >= p so only the low limbs survive
        u64 t = (u64)a.v[0] + SV_PC;
        a.v[0] = (u32)t;
        t = (u64)a.v[1] + 1u + (t >> 32);
        a.v[1] = (u32)t;
        SV_UNROLL
        for (int i = 2; i < 8; i++) a.v[i] = 0;
    }
}

// residue == 0 ?  (reference: secp256k1_fe_normalizes_to_zero_var, field_5x52_impl.h:160)
SV_HD bool fe_is_zero(const fe& a) {
    u32 o = a.v[0] | a.v[1] | a.v[2] | a.v[3] | a.v[4] | a.v[5] | a.v[6] | a.v[7];
    u32 hi = a.v[7] & a.v[6] & a.v[5] & a.v[4] & a.v[3] & a.v[2];
    return (o == 0) || (hi == 0xFFFFFFFFu && a.v[1] == SV_P1 && a.v[0] == SV_P0);
}

SV_HD bool fe_equal(const fe& a, const fe& b) {  // reference: secp256k1_fe_equal (field_impl.h:21)
    fe x = a, y = b;
    fe_normalize(x);
    fe_normalize(y);
    return u256_eq(x.v, y.v);
}
SV_HD bool fe_is_odd(const fe& a) {  // a must be normalized (reference: field_5x52_impl.h:205)
    return a.v[0] & 1u;
}

// r = a + b   (weak result)
// Fold of the carry: + c * (2^32 + 977).  The ripple past limb 1 needs limb 1 to overflow (probability ~2^-32 on
// random data), so it sits behind a branch that is practically never taken; the slow path keeps the result exact
// for adversarial operands.
SV_HD void fe_add(fe& r, const fe& a, const fe& b) {
    u32 c = u256_add(r.v, a.v, b.v);
#if SV_DEVICE_CODE
    u32 k;
    asm("mad.lo.cc.u32 %0, %3, 977, %0;\n\t"
        "addc.cc.u32 %1, %1, %3;\n\t"
        "addc.u32 %2, 0, 0;"
        : "+r"(r.v[0]), "+r"(r.v[1]), "=r"(k)
        : "r"(c));
    if (k) {
        u32 c2;
        asm("add.cc.u32 %0, %0, 1;\n\t"
            "addc.cc.u32 %1, %1, 0;\n\t"
            "addc.cc.u32 %2, %2, 0;\n\t"
            "addc.cc.u32 %3, %3, 0;\n\t"
            "addc.cc.u32 %4, %4, 0;\n\t"
            "addc.cc.u32 %5, %5, 0;\n\t"
            "addc.u32 %6, 0, 0;"
            : "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]), "=r"(c2));
        // wrapped a second time: the value is now < 2^34, adding 2^32+977 touches two limbs
        asm("mad.lo.cc.u32 %0, %2, 977, %0;\n\t"
            "addc.u32 %1, %1, %2;"
            : "+r"(r.v[0]), "+r"(r.v[1])
            : "r"(c2));
    }
#else
    u64 t = (u64)r.v[0] + (u64)c * SV_PC;
    r.v[0] = (u32)t;
    t = (u64)r.v[1] + c + (t >> 32);
    r.v[1] = (u32)t;
    for (int i = 2; i < 8; i++) { t = (u64)r.v[i] + (t >> 32); r.v[i] = (u32)t; }
    u32 c2 = (u32)(t >> 32);
    t = (u64)r.v[0] + (u64)c2 * SV_PC;
    r.v[0] = (u32)t;
    r.v[1] = (u32)((u64)r.v[1] + c2 + (t >> 32));
#endif
}

// r = a - b   (weak result)
SV_HD void fe_sub(fe& r, const fe& a, const fe& b) {
    u32 bw = u256_sub(r.v, a.v, b.v);
    // a - b + 2^256 == a - b + (2^32+977): take the constant back out; the borrow past limb 1 is as rare as the
    // carry in fe_add and handled the same way.
#if SV_DEVICE_CODE
    u32 k;
    u32 kc = bw * SV_PC;
    asm("sub.cc.u32 %0, %0, %4;\n\t"
        "subc.cc.u32 %1, %1, %3;\n\t"
        "subc.u32 %2, 0, 0;"
        : "+r"(r.v[0]), "+r"(r.v[1]), "=r"(k)
        : "r"(bw), "r"(kc));
    if (k) {
        u32 b2;
        asm("sub.cc.u32 %0, %0, 1;\n\t"
            "subc.cc.u32 %1, %1, 0;\n\t"
            "subc.cc.u32 %2, %2, 0;\n\t"
            "subc.cc.u32 %3, %3, 0;\n\t"
            "subc.cc.u32 %4, %4, 0;\n\t"
            "subc.cc.u32 %5, %5, 0;\n\t"
            "subc.u32 %6, 0, 0;"
            : "+r"(r.v[2]), "+r"(r.v[3]), "+r"(r.v[4]), "+r"(r.v[5]), "+r"(r.v[6]), "+r"(r.v[7]), "=r"(b2));
        b2 &= 1u;
        u32 k2 = b2 * SV_PC;
        asm("sub.cc.u32 %0, %0, %3;\n\t"
            "subc.u32 %1, %1, %2;"
            : "+r"(r.v[0]), "+r"(r.v[1])
            : "r"(b2), "r"(k2));
    }
#else
    u64 d = (u64)r.v[0] - (u64)bw * SV_PC;
    r.v[0] = (u32)d;
    u64 br = (d >> 32) & 1;
    d = (u64)r.v[1] - bw - br;
    r.v[1] = (u32)d;
    br = (d >> 32) & 1;
    for (int i = 2; i < 8; i++) { d = (u64)r.v[i] - br; r.v[i] = (u32)d; br = (d >> 32) & 1; }
    u32 b2 = (u32)br;
    d = (u64)r.v[0] - (u64)b2 * SV_PC;
    r.v[0] = (u32)d;
    br = (d >> 32) & 1;
    r.v[1] = (u32)((u64)r.v[1] - b2 - br);
#endif
}

SV_HD void fe_neg(fe& r, const fe& a) {  // reference: secp256k1_fe_negate (field_5x52_impl.h:336)
    fe z;
    fe_set_zero(z);
    fe_sub(r, z, a);
}
SV_HD void fe_dbl(fe& r, const fe& a) { fe_add(r, a, a); }

// reduce a 512-bit value t (16 limbs) mod p into weak form
SV_HD void fe_reduce512(fe& r, const u32 t[16]) {
#if SV_DEVICE_CODE
    // s[0..8] = lo + (hi << 32)
    u32 s[10];
    s[0] = t[0];
    asm("add.cc.u32 %0, %9, %17;\n\t"
        "addc.cc.u32 %1, %10, %18;\n\t"
        "addc.cc.u32 %2, %11, %19;\n\t"
        "addc.cc.u32 %3, %12, %20;\n\t"
        "addc.cc.u32 %4, %13, %21;\n\t"
        "addc.cc.u32 %5, %14, %22;\n\t"
        "addc.cc.u32 %6, %15, %23;\n\t"
        "addc.cc.u32 %7, %16, 0;\n\t"
        "addc.u32 %8, 0, 0;"
        : "=r"(s[1]), "=r"(s[2]), "=r"(s[3]), "=r"(s[4]), "=r"(s[5]), "=r"(s[6]), "=r"(s[7]), "=r"(s[8]), "=r"(s[9])
        : "r"(t[8]), "r"(t[9]), "r"(t[10]), "r"(t[11]), "r"(t[12]), "r"(t[13]), "r"(t[14]), "r"(t[15]),
          "r"(t[1]), "r"(t[2]), "r"(t[3]), "r"(t[4]), "r"(t[5]), "r"(t[6]), "r"(t[7]));
#ifdef SV_REDUCE_NOACC
    // VARIANT: products with a zero accumulator (fresh aligned register pairs, no pair-forming moves on the multiplier
    // pipe), added with ALU carry chains
    u32 pe[8];
    asm("mul.lo.u32 %0, %8, %12;\n\t"
        "mul.hi.u32 %1, %8, %12;\n\t"
        "mul.lo.u32 %2, %9, %12;\n\t"
        "mul.hi.u32 %3, %9, %12;\n\t"
        "mul.lo.u32 %4, %10, %12;\n\t"
        "mul.hi.u32 %5, %10, %12;\n\t"
        "mul.lo.u32 %6, %11, %12;\n\t"
        "mul.hi.u32 %7, %11, %12;"
        : "=r"(pe[0]), "=r"(pe[1]), "=r"(pe[2]), "=r"(pe[3]), "=r"(pe[4]), "=r"(pe[5]), "=r"(pe[6]), "=r"(pe[7])
        : "r"(t[8]), "r"(t[10]), "r"(t[12]), "r"(t[14]), "r"(SV_PC));
    asm("add.cc.u32 %0, %0, %10;\n\t"
        "addc.cc.u32 %1, %1, %11;\n\t"
        "addc.cc.u32 %2, %2, %12;\n\t"
        "addc.cc.u32 %3, %3, %13;\n\t"
        "addc.cc.u32 %4, %4, %14;\n\t"
        "addc.cc.u32 %5, %5, %15;\n\t"
        "addc.cc.u32 %6, %6, %16;\n\t"
        "addc.cc.u32 %7, %7, %17;\n\t"
        "addc.cc.u32 %8, %8, 0;\n\t"
        "addc.u32 %9, %9, 0;"
        : "+r"(s[0]), "+r"(s[1]), "+r"(s[2]), "+r"(s[3]), "+r"(s[4]), "+r"(s[5]), "+r"(s[6]), "+r"(s[7]),
          "+r"(s[8]), "+r"(s[9])
        : "r"(pe[0]), "r"(pe[1]), "r"(pe[2]), "r"(pe[3]), "r"(pe[4]), "r"(pe[5]), "r"(pe[6]), "r"(pe[7]));
#else
    // s[0..8] += {hi0,hi2,hi4,hi6} * 977  (even columns)
    asm("mad.lo.cc.u32 %0, %10, %14, %0;\n\t"
        "madc.hi.cc.u32 %1, %10, %14, %1;\n\t"
        "madc.lo.cc.u32 %2, %11, %14, %2;\n\t"
        "madc.hi.cc.u32 %3, %11, %14, %3;\n\t"
        "madc.lo.cc.u32 %4, %12, %14, %4;\n\t"
        "madc.hi.cc.u32 %5, %12, %14, %5;\n\t"
        "madc.lo.cc.u32 %6, %13, %14, %6;\n\t"
        "madc.hi.cc.u32 %7, %13, %14, %7;\n\t"
        "addc.cc.u32 %8, %8, 0;\n\t"
        "addc.u32 %9, %9, 0;"
        : "+r"(s[0]), "+r"(s[1]), "+r"(s[2]), "+r"(s[3]), "+r"(s[4]), "+r"(s[5]), "+r"(s[6]), "+r"(s[7]),
          "+r"(s[8]), "+r"(s[9])
        : "r"(t[8]), "r"(t[10]), "r"(t[12]), "r"(t[14]), "r"(SV_PC));
#endif
    // o[0..7] = {hi1,hi3,hi5,hi7} * 977 (odd columns: limb positions 1..8)
    u32 o[8];
    asm("mul.lo.u32 %0, %8, %12;\n\t"
        "mul.hi.u32 %1, %8, %12;\n\t"
        "mul.lo.u32 %2, %9, %12;\n\t"
        "mul.hi.u32 %3, %9, %12;\n\t"
        "mul.lo.u32 %4, %10, %12;\n\t"
        "mul.hi.u32 %5, %10, %12;\n\t"
        "mul.lo.u32 %6, %11, %12;\n\t"
        "mul.hi.u32 %7, %11, %12;"
        : "=r"(o[0]), "=r"(o[1]), "=r"(o[2]), "=r"(o[3]), "=r"(o[4]), "=r"(o[5]), "=r"(o[6]), "=r"(o[7])
        : "r"(t[9]), "r"(t[11]), "r"(t[13]), "r"(t[15]), "r"(SV_PC));
    asm("add.cc.u32 %0, %0, %9;\n\t"
        "addc.cc.u32 %1, %1, %10;\n\t"
        "addc.cc.u32 %2, %2, %11;\n\t"
        "addc.cc.u32 %3, %3, %12;\n\t"
        "addc.cc.u32 %4, %4, %13;\n\t"
        "addc.cc.u32 %5, %5, %14;\n\t"
        "addc.cc.u32 %6, %6, %15;\n\t"
        "addc.cc.u32 %7, %7, %16;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(s[1]), "+r"(s[2]), "+r"(s[3]), "+r"(s[4]), "+r"(s[5]), "+r"(s[6]), "+r"(s[7]), "+r"(s[8]), "+r"(s[9])
        : "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]), "r"(o[4]), "r"(o[5]), "r"(o[6]), "r"(o[7]));
    // second fold: T = s[8] + s[9]*2^32 (< 2^35);  T*(2^32+977) < 2^68 -> three limbs f0,f1,f2
    u64 T = ((u64)s[9] << 32) | s[8];
    u64 m = T * SV_PC;
    u64 mid = (m >> 32) + T;
    u32 f0 = (u32)m, f1 = (u32)mid, f2 = (u32)(mid >> 32);
    u32 c;
    asm("add.cc.u32 %0, %9, %17;\n\t"
        "addc.cc.u32 %1, %10, %18;\n\t"
        "addc.cc.u32 %2, %11, %19;\n\t"
        "addc.cc.u32 %3, %12, 0;\n\t"
        "addc.cc.u32 %4, %13, 0;\n\t"
        "addc.cc.u32 %5, %14, 0;\n\t"
        "addc.cc.u32 %6, %15, 0;\n\t"
        "addc.cc.u32 %7, %16, 0;\n\t"
        "addc.u32 %8, 0, 0;"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]),
          "=r"(r.v[7]), "=r"(c)
        : "r"(s[0]), "r"(s[1]), "r"(s[2]), "r"(s[3]), "r"(s[4]), "r"(s[5]), "r"(s[6]), "r"(s[7]), "r"(f0), "r"(f1),
          "r"(f2));
    // third fold (rare): wrapped value is < 2^68, adding 2^32+977 cannot wrap again
    asm("mad.lo.cc.u32 %0, %3, 977, %0;\n\t"
        "addc.cc.u32 %1, %1, %3;\n\t"
        "addc.u32 %2, %2, 0;"
        : "+r"(r.v[0]), "+r"(r.v[1]), "+r"(r.v[2])
        : "r"(c));
#else
    // lo + hi*977 + (hi<<32) in 64-bit column arithmetic
    u64 acc = 0;
    u32 s[10];
    for (int i = 0; i < 8; i++) {
        acc += (u64)t[i] + (u64)t[8 + i] * SV_PC;
        if (i > 0) acc += t[8 + i - 1];
        s[i] = (u32)acc;
        acc >>= 32;
    }
    acc += t[15];
    s[8] = (u32)acc;
    s[9] = (u32)(acc >> 32);
    u64 T = ((u64)s[9] << 32) | s[8];
    u64 m = T * SV_PC;
    u64 mid = (m >> 32) + T;
    u32 f[3] = {(u32)m, (u32)mid, (u32)(mid >> 32)};
    u64 c = 0;
    for (int i = 0; i < 8; i++) {
        c += (u64)s[i] + (i < 3 ? f[i] : 0);
        r.v[i] = (u32)c;
        c >>= 32;
    }
    u32 cc = (u32)c;
    u64 q = (u64)r.v[0] + (u64)cc * SV_PC;
    r.v[0] = (u32)q;
    q = (u64)r.v[1] + cc + (q >> 32);
    r.v[1] = (u32)q;
    r.v[2] = (u32)((u64)r.v[2] + (q >> 32));
#endif
}

// reference: secp256k1_fe_mul (field_5x52_int128_impl.h:18), secp256k1_fe_sqr (:154)
//
// Two device forms, chosen per translation unit:
//   -DSV_FE_INLINE (engine.cu, every kernel but the batch ones): inlined.  The curve kernel keeps the warps of a CTA at the
//     same program counter with CTA-wide barriers so that they share instruction fetches of the large straight-line code
//     (without the barriers the inlined ladder starves on instruction fetch).
//   otherwise (batch.cu): REAL FUNCTIONS, operands and result by value (the device ABI keeps all 24 words in registers, no
//     stack traffic): the two bodies (~4 KB together) stay cache resident; costs ~17 % call-marshalling IMAD.MOVs
//     (slower for the curve kernel in this form).
#if SV_DEVICE_CODE && !defined(SV_FE_INLINE)
static __device__ __noinline__ fe fe_mul_fn(fe a, fe b) {
    u32 t[16];
    fe r;
    u256_mul_wide(t, a.v, b.v);
    fe_reduce512(r, t);
    return r;
}
static __device__ __noinline__ fe fe_sqr_fn(fe a) {
    u32 t[16];
    fe r;
    u256_sqr_wide(t, a.v);
    fe_reduce512(r, t);
    return r;
}
SV_HD void fe_mul(fe& r, const fe& a, const fe& b) { r = fe_mul_fn(a, b); }
SV_HD void fe_sqr(fe& r, const fe& a) { r = fe_sqr_fn(a); }
#else
SV_HD void fe_mul(fe& r, const fe& a, const fe& b) {
    u32 t[16];
    u256_mul_wide(t, a.v, b.v);
    fe_reduce512(r, t);
}
SV_HD void fe_sqr(fe& r, const fe& a) {
    u32 t[16];
    u256_sqr_wide(t, a.v);
    fe_reduce512(r, t);
}
#endif

// r = a * k for a small constant k (k <= 2^16)   (reference: secp256k1_fe_mul_int)
SV_HD void fe_mul_small(fe& r, const fe& a, u32 k) {
    u64 c = 0;
    u32 s[8];
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        c += (u64)a.v[i] * k;
        s[i] = (u32)c;
        c >>= 32;
    }
    // fold c (< 2^16) : c * (2^32 + 977)
    u64 m = c * SV_PC;
    u64 q = (u64)s[0] + (u32)m;
    r.v[0] = (u32)q;
    q = (u64)s[1] + (m >> 32) + c + (q >> 32);
    r.v[1] = (u32)q;
    SV_UNROLL
    for (int i = 2; i < 8; i++) {
        q = (u64)s[i] + (q >> 32);
        r.v[i] = (u32)q;
    }
    u32 c2 = (u32)(q >> 32);
    q = (u64)r.v[0] + (u64)c2 * SV_PC;
    r.v[0] = (u32)q;
    q = (u64)r.v[1] + c2 + (q >> 32);
    r.v[1] = (u32)q;
    r.v[2] = (u32)((u64)r.v[2] + (q >> 32));
}

// Small multiples on the ALU pipe only (the multiplier pipe is the bottleneck of the curve-side kernel):
// 3a = a + a + a ; 8a = (a << 3) with the three bits shifted out folded back through 2^256 == 2^32 + 977.
SV_HD void fe_mul3(fe& r, const fe& a) {
    fe t;
    fe_add(t, a, a);
    fe_add(r, t, a);
}
SV_HD void fe_mul8(fe& r, const fe& a) {
    u32 top = a.v[7] >> 29;  // < 8
    u32 s[8];
    SV_UNROLL
    for (int i = 7; i > 0; i--) s[i] = (a.v[i] << 3) | (a.v[i - 1] >> 29);
    s[0] = a.v[0] << 3;
    // + top * (2^32 + 977): top*977 < 2^13
    u32 add0 = top * SV_PC;
    fe x, y;
    SV_UNROLL
    for (int i = 0; i < 8; i++) { x.v[i] = s[i]; y.v[i] = 0; }
    y.v[0] = add0;
    y.v[1] = top;
    fe_add(r, x, y);
}

SV_HD void fe_sqr_n(fe& r, const fe& a, int n) {
    r = a;
#if SV_DEVICE_CODE
#pragma unroll 1
#endif
    for (int i = 0; i < n; i++) fe_sqr(r, r);
}

// x^(2^223 - 1) and the shared sub-powers of the sqrt / inverse addition chains.  The chain is
// the classic one for this prime (reference: field_impl.h:33-138 uses the same block structure:
// the exponents' binary forms are [223 ones][0][22 ones][...]).
struct fe_pow_ladder {
    fe x2, x22, x223;
};
SV_HD void fe_pow_common(fe_pow_ladder& L, const fe& a) {
    fe x3, x6, x9, x11, x44, x88, x176, x220, t;
    fe_sqr(t, a);
    fe_mul(L.x2, t, a);
    fe_sqr(t, L.x2);
    fe_mul(x3, t, a);
    fe_sqr_n(t, x3, 3);
    fe_mul(x6, t, x3);
    fe_sqr_n(t, x6, 3);
    fe_mul(x9, t, x3);
    fe_sqr_n(t, x9, 2);
    fe_mul(x11, t, L.x2);
    fe_sqr_n(t, x11, 11);
    fe_mul(L.x22, t, x11);
    fe_sqr_n(t, L.x22, 22);
    fe_mul(x44, t, L.x22);
    fe_sqr_n(t, x44, 44);
    fe_mul(x88, t, x44);
    fe_sqr_n(t, x88, 88);
    fe_mul(x176, t, x88);
    fe_sqr_n(t, x176, 44);
    fe_mul(x220, t, x44);
    fe_sqr_n(t, x220, 3);
    fe_mul(L.x223, t, x3);
}

// r = sqrt(a) if it exists (returns true), computed as a^((p+1)/4) and verified by squaring.
// (p+1)/4 = [223 ones][0][22 ones][0000][11][00]b.   reference: secp256k1_fe_sqrt (field_impl.h:33)
SV_HD bool fe_sqrt(fe& r, const fe& a) {
    fe_pow_ladder L;
    fe t;
    fe_pow_common(L, a);
    fe_sqr_n(t, L.x223, 23);
    fe_mul(t, t, L.x22);
    fe_sqr_n(t, t, 6);
    fe_mul(t, t, L.x2);
    fe_sqr_n(r, t, 2);
    fe_sqr(t, r);
    return fe_equal(t, a);
}

// r = a^(p-2) = 1/a  (0 -> 0).  p-2 = [223 ones][0][22 ones][0000][1][011][01]b.
// reference computes the same value with safegcd (secp256k1_fe_inv_var, field_5x52_impl.h:496);
// a uniform exponentiation suits SIMT better than the branchy divsteps.
SV_HD void fe_inv(fe& r, const fe& a) {
    fe_pow_ladder L;
    fe t;
    fe_pow_common(L, a);
    fe_sqr_n(t, L.x223, 23);
    fe_mul(t, t, L.x22);
    fe_sqr_n(t, t, 5);
    fe_mul(t, t, a);
    fe_sqr_n(t, t, 3);
    fe_mul(t, t, L.x2);
    fe_sqr_n(t, t, 2);
    fe_mul(r, t, a);
}

// 1/a by binary extended Euclid (variable time; 0 -> 0; result canonical): see u256_modinv_var
SV_HD void fe_inv_var(fe& r, const fe& a) {
    const u32 P[8] = {SV_P0, SV_P1, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    fe t = a;
    fe_normalize(t);
    u256_modinv_var(r.v, t.v, P);
}

// big-endian 32 bytes -> limbs; returns false if value >= p (reference: secp256k1_fe_set_b32_limit,
// field_5x52_impl.h:272)
SV_HD bool fe_set_b32(fe& r, const u8* b) {
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        const u8* q = b + 28 - 4 * i;
        r.v[i] = ((u32)q[0] << 24) | ((u32)q[1] << 16) | ((u32)q[2] << 8) | (u32)q[3];
    }
    return !fe_gte_p(r);
}
// limbs (normalised first) -> big-endian bytes (reference: secp256k1_fe_get_b32, field_5x52_impl.h:278)
SV_HD void fe_get_b32(u8* b, const fe& a) {
    fe t = a;
    fe_normalize(t);
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        u8* q = b + 28 - 4 * i;
        q[0] = (u8)(t.v[i] >> 24);
        q[1] = (u8)(t.v[i] >> 16);
        q[2] = (u8)(t.v[i] >> 8);
        q[3] = (u8)t.v[i];
    }
}
