// bolt11.cuh — BOLT11 invoice signatures: bech32, the tagged-field walk, the signing hash and the recovery scalars.
//
// Reference (paths relative to the Core Lightning tree):
//   bech32        bech32_decode (no length limit)                     common/bech32.c:94-155
//   field walk    bolt11_decode_nosig: timestamp, tag / length walk    common/bolt11.c:882-936
//   `n` field     decode_n -> pull_expected_length, pubkey_from_node_id   common/bolt11.c:152-166, 315-342
//   signing hash  hash_u5_init / hash_u5 / hash_u5_done                common/hash_u5.c
//   signature     bolt11_decode's tail: recid, parse_compact, verify or recover   common/bolt11.c:1010-1059
//                 secp256k1_ecdsa_sig_recover                          modules/recovery/main_impl.h
//
// Only what locates the signed bytes, the signature and the key is checked here.  Field values (the hrp's prefix, chain
// and amount, the presence of p / s / d / h, trailing bits of p / h / s, UTF-8 in d, x c f r m 9) are left to the caller's
// own decode, as the BOLT12 path leaves field semantics to its caller.
//
// Every function here is SV_HD: the k_b11_* kernels in engine.cu call them per thread, tests/host_emul compiles the
// same code for the host.
#pragma once
#include "verify.cuh"

#define SV_B11_SIG_WORDS 104  // 520 bits: r || s || recovery id
#define SV_B11_N_WORDS 53     // 33-byte key + one trailing bit
#define SV_B11_TAG_N 19       // bech32_charset_rev['n']

// bech32_charset_rev (common/bech32.c) for 0..127; -1 outside the charset
SV_HD int b11_rev(u8 c) {
    if (c & 0x80) return -1;
    if (c >= 'A' && c <= 'Z') c = (u8)(c - 'A' + 'a');
    switch (c) {
        case 'q': return 0;  case 'p': return 1;  case 'z': return 2;  case 'r': return 3;
        case 'y': return 4;  case '9': return 5;  case 'x': return 6;  case '8': return 7;
        case 'g': return 8;  case 'f': return 9;  case '2': return 10; case 't': return 11;
        case 'v': return 12; case 'd': return 13; case 'w': return 14; case '0': return 15;
        case 's': return 16; case '3': return 17; case 'j': return 18; case 'n': return 19;
        case '5': return 20; case '4': return 21; case 'k': return 22; case 'h': return 23;
        case 'c': return 24; case 'e': return 25; case '6': return 26; case 'm': return 27;
        case 'u': return 28; case 'a': return 29; case '7': return 30; case 'l': return 31;
        default: return -1;
    }
}

SV_HD u32 b11_polymod(u32 pre) {
    u32 b = pre >> 25;
    return ((pre & 0x1FFFFFFu) << 5) ^ (-((b >> 0) & 1u) & 0x3b6a57b2u) ^ (-((b >> 1) & 1u) & 0x26508e6du) ^
           (-((b >> 2) & 1u) & 0x1ea119fau) ^ (-((b >> 3) & 1u) & 0x3d4233ddu) ^ (-((b >> 4) & 1u) & 0x2a1462b3u);
}

// The string's layout once bech32_decode has accepted it (with the BECH32 constant; BECH32M is a refusal here).
struct b11_str {
    u32 hrp_len;  // characters before the separator
    u32 words;    // data words, checksum excluded: word k is character hrp_len + 1 + k
};

// bech32_decode over s[0 .. strnlen(s, span)).  False where it returns BECH32_ENCODING_NONE or BECH32M.
SV_HD bool b11_bech32(const u8* s, u32 span, b11_str* out) {
    u32 L = 0;
    while (L < span && s[L]) L++;
    if (L < 8) return false;
    u32 dl = 0;
    while (dl < L && s[L - 1 - dl] != '1') dl++;
    if (1 + dl >= L || dl < 6) return false;
    const u32 hl = L - 1 - dl;
    bool lower = false, upper = false;
    u32 chk = 1;
    for (u32 i = 0; i < hl; i++) {
        int ch = (signed char)s[i];
        if (ch < 33 || ch > 126) return false;
        if (ch >= 'a' && ch <= 'z') lower = true;
        else if (ch >= 'A' && ch <= 'Z') { upper = true; ch = ch - 'A' + 'a'; }
        chk = b11_polymod(chk) ^ (u32)(ch >> 5);
    }
    chk = b11_polymod(chk);
    for (u32 i = 0; i < hl; i++) chk = b11_polymod(chk) ^ (s[i] & 0x1fu);
    for (u32 i = hl + 1; i < L; i++) {
        u8 c = s[i];
        if (c >= 'a' && c <= 'z') lower = true;
        if (c >= 'A' && c <= 'Z') upper = true;
        int v = b11_rev(c);
        if (v < 0) return false;
        chk = b11_polymod(chk) ^ (u32)v;
    }
    if ((lower && upper) || chk != 1u) return false;
    out->hrp_len = hl;
    out->words = dl - 6;
    return true;
}

SV_HD u32 b11_word(const u8* s, const b11_str& b, u32 k) { return (u32)b11_rev(s[b.hrp_len + 1 + k]); }

// big-endian bytes of words [w0, w0 + nw), 8 bits at a time (bech32_convert_bits 5 -> 8, no padding); returns the bits
// left over (their value in *rest, as many bits as the return says)
SV_HD u32 b11_pull_bytes(const u8* s, const b11_str& b, u32 w0, u32 nw, u8* out, u32* rest) {
    u32 acc = 0, bits = 0, o = 0;
    for (u32 k = 0; k < nw; k++) {
        acc = (acc << 5) | b11_word(s, b, w0 + k);
        bits += 5;
        if (bits >= 8) {
            bits -= 8;
            out[o++] = (u8)(acc >> bits);
        }
    }
    *rest = acc & ((1u << bits) - 1u);
    return bits;
}

// What the parse stage hands to the signature step.
struct b11_parsed {
    u8 sig[64];   // r || s
    u8 recid;
    u8 have_n;    // a 53-word `n` field was decoded: key33 holds it and it is a valid compressed key
    u8 key33[33];
};

// bolt11_decode_nosig's structure (bech32, timestamp, tag walk, the 104 signature words, the first 53-word `n`) and the
// signature bytes.  False where the device reports status -1.
SV_HD bool b11_parse(const u8* s, u32 span, b11_str* bs, b11_parsed* p) {
    b11_str b;
    if (!b11_bech32(s, span, &b)) return false;
    const u32 W = b.words;
    if (W < 7) return false;  // 35-bit timestamp
    u32 pos = 7;
    p->have_n = 0;
    while (W - pos > SV_B11_SIG_WORDS) {
        // tag (5 bits) and length (10 bits): at least 105 words are left, so both can be read
        const u32 type = b11_word(s, b, pos);
        const u32 flen = (b11_word(s, b, pos + 1) << 5) | b11_word(s, b, pos + 2);
        pos += 3;
        if (flen > W - pos) return false;
        if (type == SV_B11_TAG_N && !p->have_n && flen == SV_B11_N_WORDS) {
            // decode_n: 265 bits into 33 bytes, the one trailing bit must be zero; then the key must parse
            p->have_n = 1;
            u32 rest;
            b11_pull_bytes(s, b, pos, SV_B11_N_WORDS, p->key33, &rest);
            if (rest) return false;
            ge Q;
            if (!key_decode(Q, SV_KIND_ECDSA33, p->key33)) return false;
        }
        pos += flen;
    }
    if (W - pos != SV_B11_SIG_WORDS) return false;
    u8 sig65[65];
    u32 rest;
    b11_pull_bytes(s, b, pos, SV_B11_SIG_WORDS, sig65, &rest);  // 520 bits: nothing left over
    for (int i = 0; i < 64; i++) p->sig[i] = sig65[i];
    p->recid = sig65[64];
    b.words = pos;  // the signed words
    *bs = b;
    return true;
}

// hash_u5's signing hash: SHA-256 of the lowercased hrp and the signed words packed to bytes, the last byte zero-padded
SV_HD void b11_sighash(u8 out32[32], const u8* s, const b11_str& b) {
    sha256_stream c;
    sha_stream_init(c);
    for (u32 i = 0; i < b.hrp_len; i++) {
        u8 ch = s[i];
        sha_stream_byte(c, (ch >= 'A' && ch <= 'Z') ? (u8)(ch - 'A' + 'a') : ch);
    }
    u32 acc = 0, bits = 0;
    for (u32 k = 0; k < b.words; k++) {
        acc = (acc << 5) | b11_word(s, b, k);
        bits += 5;
        if (bits >= 8) {
            bits -= 8;
            sha_stream_byte(c, (u8)(acc >> bits));
        }
    }
    if (bits) sha_stream_byte(c, (u8)(acc << (8 - bits)));
    const u64 total = c.total * 8;
    sha_stream_byte(c, 0x80);
    while (c.fill != 56) sha_stream_byte(c, 0);
    c.blk[14] = (u32)(total >> 32);
    c.blk[15] = (u32)total;
    sha256_compress(c.st, c.blk);
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (u8)(c.st[i] >> 24);
        out32[4 * i + 1] = (u8)(c.st[i] >> 16);
        out32[4 * i + 2] = (u8)(c.st[i] >> 8);
        out32[4 * i + 3] = (u8)c.st[i];
    }
}

// ---- recovery (secp256k1_ecdsa_recover): Q = r^-1 (s R - e G), R the point with x = r (+ n when recid & 2) and y parity
// recid & 1.  The ladder lifts x to the even-y point E (key_decode, x-only), and s R = (+-s) E, so the work record carries
// u1 = -e / r for G and u2 = +-s / r for E.  False (status 0) where secp256k1_ecdsa_recover returns 0 before any point
// arithmetic: recid > 3, r or s out of range or zero, r + n >= p for recid & 2.  An x off the curve and Q = infinity are
// caught after the ladder.
SV_HD bool b11_recover_prep(sv_work& w, u8 x32[32], const u8* sig64, u8 recid, const u8* msg32) {
    sc r, s, e;
    bool ovr, ovs;
    sc_set_b32(r, sig64, &ovr);
    sc_set_b32(s, sig64 + 32, &ovs);
    sc_set_b32(e, msg32, nullptr);
    bool ok = recid <= 3 && !ovr && !ovs && !sc_is_zero(r) && !sc_is_zero(s);
    // x = r, or r + n where r < p - n (recovery's main_impl.h: fe_cmp_var(x, p - n) >= 0 refuses)
    u32 x[8];
    for (int i = 0; i < 8; i++) x[i] = r.v[i];
    if (recid & 2) {
        ok = ok && ecdsa_r_plus_n_flag(r) != 0;
        u256_add(x, x, SC_N);
    }
    for (int i = 0; i < 8; i++) {
        u8* q = x32 + 28 - 4 * i;
        q[0] = (u8)(x[i] >> 24); q[1] = (u8)(x[i] >> 16); q[2] = (u8)(x[i] >> 8); q[3] = (u8)x[i];
    }
    if (!ok) {
        work_set_invalid(w);
        return false;
    }
    sc rinv, u1, u2;
    sc_inverse_var(rinv, r);
    sc_mul(u1, rinv, e);
    sc_negate(u1, u1);
    sc_mul(u2, rinv, s);
    if (recid & 1) sc_negate(u2, u2);
    for (int i = 0; i < 5; i++) w.pad[i] = 0;
    sc_prepare_u2(w, u2);
    sc_prepare_u1(w, u1);
    w.flags = SV_WF_VALID;
    return true;
}

// Q from the parked Jacobian result and its 1/Z: the 33-byte compressed key (secp256k1_ec_pubkey_serialize)
SV_HD void b11_compress(u8 out33[33], const sv_jac& j, const fe& zi) {
    gej R;
    fe_from_words(R.x, j.x);
    fe_from_words(R.y, j.y);
    ge a;
    ge_set_gej_zinv(a, R, zi);
    fe_normalize(a.y);
    out33[0] = fe_is_odd(a.y) ? 3 : 2;
    fe_get_b32(out33 + 1, a.x);
}

// status and key of cnt (<= SV_FINAL_BATCH) consecutive parked recoveries, one field inversion for all of them
// (Montgomery's trick); a result that is not usable (refused before the ladder, x off the curve, Q = infinity) gets 0
// and a zero key
SV_HD void b11_recover_final_batch(int* status, u8* key33, const sv_jac* jac, int cnt) {
    fe pre[SV_FINAL_BATCH];
    fe acc, one;
    fe_set_u32(one, 1);
    for (int i = 0; i < cnt; i++) {
        fe z;
        fe_from_words(z, jac[i].z);
        if (!(jac[i].ok && !jac[i].inf && !fe_is_zero(z))) z = one;
        if (i == 0) pre[0] = z; else fe_mul(pre[i], pre[i - 1], z);
    }
    fe_inv(acc, pre[cnt - 1]);
    for (int i = cnt - 1; i >= 0; i--) {
        fe z, zi;
        fe_from_words(z, jac[i].z);
        const bool usable = jac[i].ok && !jac[i].inf && !fe_is_zero(z);
        if (!usable) z = one;
        if (i > 0) {
            fe_mul(zi, acc, pre[i - 1]);
            fe_mul(acc, acc, z);
        } else {
            zi = acc;
        }
        status[i] = usable ? 1 : 0;
        if (usable) b11_compress(key33 + 33 * i, jac[i], zi);
        else for (int k = 0; k < 33; k++) key33[33 * i + k] = 0;
    }
}
