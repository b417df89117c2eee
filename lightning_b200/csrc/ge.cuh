// ge.cuh — secp256k1 group law in Jacobian coordinates on top of fe.cuh.
//
// Follows the case analysis of the reference's group module (libsecp256k1 group_impl.h:
// gej_double_var :474, gej_add_ge_var :569 incl. the H==0 branch :595-605, ge_set_xo_var :334),
// with our own formula scheduling.  The formulas never use the curve constant b, so the same code
// runs on any isomorphic curve y^2 = x^3 + 7c^6 — the effective-affine ("global Z") trick of
// ecmult_impl.h:73-115 relies on exactly that.
#pragma once
#include "fe.cuh"

// Which branch of the case analysis each addition took.  The host build of the tests (tests/host_emul) defines
// SV_GE_TRACE to log these so that tests/group_schedule.py can be checked against the code, addition by addition;
// everywhere else it expands to nothing.
#define SV_GE_ADD_GENERIC 0
#define SV_GE_ADD_DOUBLE 1
#define SV_GE_ADD_INFINITY 2
#define SV_GE_ADD_A_INF 3
#define SV_GE_ADD_B_INF 4
#define SV_GE_MIXED 0  // gej_add_ge / pair_add_ge
#define SV_GE_FULL 8   // gej_add_gej
#ifndef SV_GE_TRACE
#define SV_GE_TRACE(ev) ((void)0)
#endif

struct ge {  // affine point (never infinity)
    fe x, y;
};
struct gej {  // Jacobian point; inf != 0 means the point at infinity (coordinates then meaningless)
    fe x, y, z;
    u32 inf;
};

static SV_CDATA const u32 GE_BETA[8] = {0x719501EEu, 0xC1396C28u, 0x12F58995u, 0x9CF04975u,
                                        0xAC3434E9u, 0x6E64479Eu, 0x657C0710u, 0x7AE96A2Bu};  // field.h:69-72
static SV_CDATA const u32 GE_GX[8] = {0x16F81798u, 0x59F2815Bu, 0x2DCE28D9u, 0x029BFCDBu,
                                      0xCE870B07u, 0x55A06295u, 0xF9DCBBACu, 0x79BE667Eu};  // group_impl.h:38-43
static SV_CDATA const u32 GE_GY[8] = {0xFB10D4B8u, 0x9C47D08Fu, 0xA6855419u, 0xFD17B448u,
                                      0x0E1108A8u, 0x5DA4FBFCu, 0x26A3C465u, 0x483ADA77u};

SV_HD void gej_set_ge(gej& r, const ge& a) {
    r.x = a.x;
    r.y = a.y;
    fe_set_u32(r.z, 1);
    r.inf = 0;
}

// r = 2a.  a=0 curve: A=X^2 B=Y^2 C=B^2 D=2((X+B)^2-A-C) E=3A  X3=E^2-2D  Y3=E(D-X3)-8C  Z3=2YZ
// (2M + 5S).  No point of order 2 exists on secp256k1, so Y != 0 for finite points.
SV_HD void gej_double(gej& r, const gej& a) {
    fe A, B, C, D, E, t;
    fe_sqr(A, a.x);
    fe_sqr(B, a.y);
    fe_sqr(C, B);
    fe_add(t, a.x, B);
    fe_sqr(t, t);
    fe_sub(t, t, A);
    fe_sub(t, t, C);
    fe_dbl(D, t);
    fe_mul3(E, A);
    fe_mul(t, a.y, a.z);
    fe_dbl(r.z, t);
    fe_sqr(t, E);
    fe_sub(t, t, D);
    fe_sub(r.x, t, D);
    fe_sub(t, D, r.x);
    fe_mul(t, t, E);
    fe_mul8(C, C);
    fe_sub(r.y, t, C);
    r.inf = a.inf;
}

// r = a + b, b affine (8M + 3S).  Full case analysis as in gej_add_ge_var (group_impl.h:569-629):
//   a = inf -> b ; H == 0 and R == 0 -> double ; H == 0 and R != 0 -> infinity.
// If rzr != nullptr it receives H, the ratio Z3/Z1 (used when building effective-affine tables).
SV_HD void gej_add_ge(gej& r, const gej& a, const ge& b, fe* rzr = nullptr) {
    if (a.inf) {
        SV_GE_TRACE(SV_GE_MIXED | SV_GE_ADD_A_INF);
        gej_set_ge(r, b);
        if (rzr) fe_set_u32(*rzr, 1);  // not meaningful (reference asserts this never happens in table builds)
        return;
    }
    fe zz, u2, s2, h, rr, hh, hhh, v, t;
    fe_sqr(zz, a.z);
    fe_mul(u2, b.x, zz);
    fe_mul(t, a.z, zz);
    fe_mul(s2, b.y, t);
    fe_sub(h, u2, a.x);
    fe_sub(rr, s2, a.y);
    if (fe_is_zero(h)) {
        if (fe_is_zero(rr)) {
            SV_GE_TRACE(SV_GE_MIXED | SV_GE_ADD_DOUBLE);
            if (rzr) fe_dbl(*rzr, a.y);
            gej_double(r, a);
        } else {
            SV_GE_TRACE(SV_GE_MIXED | SV_GE_ADD_INFINITY);
            r.inf = 1;
            if (rzr) fe_set_zero(*rzr);
        }
        return;
    }
    SV_GE_TRACE(SV_GE_MIXED | SV_GE_ADD_GENERIC);
    if (rzr) *rzr = h;
    fe_sqr(hh, h);
    fe_mul(hhh, h, hh);
    fe_mul(v, a.x, hh);
    fe_mul(r.z, a.z, h);
    fe_sqr(t, rr);
    fe_sub(t, t, hhh);
    fe_sub(t, t, v);
    fe x3;
    fe_sub(x3, t, v);
    fe_sub(t, v, x3);
    fe_mul(t, t, rr);
    fe_mul(hhh, hhh, a.y);
    fe_sub(r.y, t, hhh);
    r.x = x3;
    r.inf = 0;
}

// r = a + b, both Jacobian (12M + 4S), full case analysis as secp256k1_gej_add_var (group_impl.h:504-567):
// either operand at infinity; H == 0 with R == 0 -> double; H == 0 with R != 0 -> infinity.  r may alias a or b.
// Used where independently computed partial sums meet (the small-batch path adds its two half-ladders and the comb sum).
SV_HD void gej_add_gej(gej& r, const gej& a, const gej& b) {
    if (a.inf) {
        SV_GE_TRACE(SV_GE_FULL | SV_GE_ADD_A_INF);
        r = b;
        return;
    }
    if (b.inf) {
        SV_GE_TRACE(SV_GE_FULL | SV_GE_ADD_B_INF);
        r = a;
        return;
    }
    fe z22, z12, u1, u2, s1, s2, h, rr, t;
    fe_sqr(z22, b.z);
    fe_sqr(z12, a.z);
    fe_mul(u1, a.x, z22);
    fe_mul(u2, b.x, z12);
    fe_mul(t, b.z, z22);
    fe_mul(s1, a.y, t);
    fe_mul(t, a.z, z12);
    fe_mul(s2, b.y, t);
    fe_sub(h, u2, u1);
    fe_sub(rr, s2, s1);
    if (fe_is_zero(h)) {
        if (fe_is_zero(rr)) {
            SV_GE_TRACE(SV_GE_FULL | SV_GE_ADD_DOUBLE);
            gej_double(r, a);
        } else {
            SV_GE_TRACE(SV_GE_FULL | SV_GE_ADD_INFINITY);
            r.inf = 1;
            fe_set_zero(r.x);
            fe_set_zero(r.y);
            fe_set_zero(r.z);
        }
        return;
    }
    SV_GE_TRACE(SV_GE_FULL | SV_GE_ADD_GENERIC);
    fe hh, hhh, v, x3;
    fe_sqr(hh, h);
    fe_mul(hhh, h, hh);
    fe_mul(v, u1, hh);
    fe_mul(t, a.z, b.z);
    fe_mul(r.z, t, h);
    fe_sqr(t, rr);
    fe_sub(t, t, hhh);
    fe_sub(t, t, v);
    fe_sub(x3, t, v);
    fe_sub(t, v, x3);
    fe_mul(t, t, rr);
    fe_mul(hhh, hhh, s1);
    fe_sub(r.y, t, hhh);
    r.x = x3;
    r.inf = 0;
}

// y^2 == x^3 + 7 ?   reference: secp256k1_ge_is_valid_var (group_impl.h:356)
SV_HD bool ge_is_on_curve(const ge& a) {
    fe y2, x3, seven;
    fe_sqr(y2, a.y);
    fe_sqr(x3, a.x);
    fe_mul(x3, x3, a.x);
    fe_set_u32(seven, 7);
    fe_add(x3, x3, seven);
    return fe_equal(y2, x3);
}

// Lift x to the curve point with the requested y parity; false if x^3+7 is a non-residue.
// reference: secp256k1_ge_set_xo_var (group_impl.h:334-346) / ge_set_xquad (:318-332)
SV_HD bool ge_set_xo(ge& r, const fe& x, bool odd) {
    fe c, seven, y;
    fe_sqr(c, x);
    fe_mul(c, c, x);
    fe_set_u32(seven, 7);
    fe_add(c, c, seven);
    bool ok = fe_sqrt(y, c);  // no early exit: see key_decode
    fe_normalize(y);
    if (fe_is_odd(y) != odd) fe_neg(y, y);
    r.x = x;
    r.y = y;
    return ok;
}

// Jacobian -> affine with a supplied 1/Z.   reference: secp256k1_ge_set_gej_zinv (group_impl.h:99)
SV_HD void ge_set_gej_zinv(ge& r, const gej& a, const fe& zi) {
    fe zi2, zi3;
    fe_sqr(zi2, zi);
    fe_mul(zi3, zi2, zi);
    fe_mul(r.x, a.x, zi2);
    fe_mul(r.y, a.y, zi3);
}
