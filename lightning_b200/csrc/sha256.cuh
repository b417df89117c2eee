// sha256.cuh — SHA-256 for the two hashing jobs on the verification path:
//   * sha256_double over a variable-length span (reference: bitcoin/shadouble.c:7-11 on top of
//     ccan/ccan/crypto/sha256/sha256.c:87 Transform / :243 sha256) — gossip message tails, BIP143
//     preimages;
//   * the BIP-340 challenge hash from its fixed midstate (reference:
//     modules/schnorrsig/main_impl.h:103-127).
// Plain FIPS 180-4 code, one thread per message; 32-bit rotates map to SHF.R.W, the rest to
// LOP3/IADD3 — this is ALU-pipe work that runs beside the IMAD-bound EC arithmetic.
#pragma once
#include "common.cuh"

static SV_CDATA const u32 SHA256_K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

SV_HD u32 sha_rotr(u32 x, int n) { return (x >> n) | (x << (32 - n)); }

SV_HD void sha256_init(u32 st[8]) {
    st[0] = 0x6a09e667u; st[1] = 0xbb67ae85u; st[2] = 0x3c6ef372u; st[3] = 0xa54ff53au;
    st[4] = 0x510e527fu; st[5] = 0x9b05688cu; st[6] = 0x1f83d9abu; st[7] = 0x5be0cd19u;
}

// one compression of a 16-word big-endian block
SV_HD void sha256_compress(u32 st[8], const u32 blk[16]) {
    u32 w[16];
    SV_UNROLL
    for (int i = 0; i < 16; i++) w[i] = blk[i];
    u32 a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#if SV_DEVICE_CODE
#pragma unroll 1
#endif
    for (int r = 0; r < 64; r += 16) {
        SV_UNROLL
        for (int i = 0; i < 16; i++) {
            if (r) {
                u32 w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
                u32 s0 = sha_rotr(w15, 7) ^ sha_rotr(w15, 18) ^ (w15 >> 3);
                u32 s1 = sha_rotr(w2, 17) ^ sha_rotr(w2, 19) ^ (w2 >> 10);
                w[i] = w[i] + s0 + w[(i + 9) & 15] + s1;
            }
            u32 S1 = sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25);
            u32 ch = (e & f) ^ (~e & g);
            u32 t1 = h + S1 + ch + SHA256_K[r + i] + w[i];
            u32 S0 = sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22);
            u32 mj = (a & b) ^ (a & c) ^ (b & c);
            u32 t2 = S0 + mj;
            h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// SHA-256 of an arbitrary byte span (byte loads: spans are unaligned slices of wire messages).
SV_HD void sha256_bytes(u32 st[8], const u8* p, size_t len) {
    sha256_init(st);
    u32 blk[16];
    size_t off = 0;
    // full blocks
    while (len - off >= 64) {
        for (int i = 0; i < 16; i++) {
            const u8* q = p + off + 4 * i;
            blk[i] = ((u32)q[0] << 24) | ((u32)q[1] << 16) | ((u32)q[2] << 8) | (u32)q[3];
        }
        sha256_compress(st, blk);
        off += 64;
    }
    // tail + padding (one or two blocks)
    size_t rem = len - off;
    u8 tail[128];
    for (int i = 0; i < 128; i++) tail[i] = 0;
    for (size_t i = 0; i < rem; i++) tail[i] = p[off + i];
    tail[rem] = 0x80;
    int nblk = (rem + 9 > 64) ? 2 : 1;
    u64 bits = (u64)len * 8;
    for (int i = 0; i < 8; i++) tail[nblk * 64 - 1 - i] = (u8)(bits >> (8 * i));
    for (int b = 0; b < nblk; b++) {
        for (int i = 0; i < 16; i++) {
            const u8* q = tail + 64 * b + 4 * i;
            blk[i] = ((u32)q[0] << 24) | ((u32)q[1] << 16) | ((u32)q[2] << 8) | (u32)q[3];
        }
        sha256_compress(st, blk);
    }
}

// second pass of sha256_double: SHA-256 of the 32-byte digest held as 8 state words
SV_HD void sha256_of_digest(u32 out[8], const u32 dg[8]) {
    u32 blk[16];
    SV_UNROLL
    for (int i = 0; i < 8; i++) blk[i] = dg[i];
    blk[8] = 0x80000000u;
    SV_UNROLL
    for (int i = 9; i < 15; i++) blk[i] = 0;
    blk[15] = 256;
    sha256_init(out);
    sha256_compress(out, blk);
}

// out32 = SHA256(SHA256(p[0..len)))   reference: sha256_double (bitcoin/shadouble.c:7)
SV_HD void sha256d_bytes(u8 out32[32], const u8* p, size_t len) {
    u32 st[8], o[8];
    sha256_bytes(st, p, len);
    sha256_of_digest(o, st);
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (u8)(o[i] >> 24);
        out32[4 * i + 1] = (u8)(o[i] >> 16);
        out32[4 * i + 2] = (u8)(o[i] >> 8);
        out32[4 * i + 3] = (u8)o[i];
    }
}

// BIP-340 challenge: SHA256(tag||tag|| r32 || px32 || msg32) with tag = SHA256("BIP0340/challenge").
// The state after the 64-byte tag block is a constant (reference: main_impl.h:103-114).
SV_HD void sha256_bip340_challenge(u8 out32[32], const u8* r32, const u8* px32, const u8* msg32) {
    u32 st[8] = {0x9cecba11u, 0x23925381u, 0x11679112u, 0xd1627e0fu, 0x97c87550u, 0x003cc765u, 0x90f61164u, 0x33e9b66au};
    u32 blk[16];
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        blk[i] = ((u32)r32[4 * i] << 24) | ((u32)r32[4 * i + 1] << 16) | ((u32)r32[4 * i + 2] << 8) | r32[4 * i + 3];
        blk[8 + i] = ((u32)px32[4 * i] << 24) | ((u32)px32[4 * i + 1] << 16) | ((u32)px32[4 * i + 2] << 8) | px32[4 * i + 3];
    }
    sha256_compress(st, blk);
    SV_UNROLL
    for (int i = 0; i < 8; i++)
        blk[i] = ((u32)msg32[4 * i] << 24) | ((u32)msg32[4 * i + 1] << 16) | ((u32)msg32[4 * i + 2] << 8) | msg32[4 * i + 3];
    blk[8] = 0x80000000u;
    SV_UNROLL
    for (int i = 9; i < 15; i++) blk[i] = 0;
    blk[15] = (64 + 96) * 8;
    sha256_compress(st, blk);
    SV_UNROLL
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (u8)(st[i] >> 24);
        out32[4 * i + 1] = (u8)(st[i] >> 16);
        out32[4 * i + 2] = (u8)(st[i] >> 8);
        out32[4 * i + 3] = (u8)st[i];
    }
}

// ---- BIP143 sighash of one segwit-v0 input of a 1-output transaction (SURVEY.md §8f N2) ------------------------
// What bitcoin_tx_hash_for_sig (bitcoin/signature.c:120-151) obtains from libwally's bip143_signature_hash
// (external/libwally-core/src/tx_io.c:660-765) for the commitment/HTLC transactions channeld checks
// (common/htlc_tx.c:10-69: one input, one output).  The preimage is assembled by the device from the fields below
// and double-hashed; the script bytes live in a separate blob.
struct sv_tx_item {
    u32 version, locktime, sequence, sighash_type;
    u8 prev_txid[32];            // internal byte order, as serialised inside the transaction
    u32 prev_index;
    u32 script_off, script_len;  // scriptCode = the witness script (bitcoin/script.c:732,849 for HTLCs)
    u32 out_script_off, out_script_len;  // scriptPubKey of the single output
    u32 flags;                           // SV_TX_* (include/cln_sigverify.h)
    u64 input_amount, output_amount;     // satoshi
    u32 prevouts_off, prevouts_len;      // SV_TX_INPUTS_SERIALIZED: every outpoint / every nSequence of the transaction
    u32 sequences_off, sequences_len;
};
#ifndef SV_TX_OUTPUTS_SERIALIZED
#define SV_TX_OUTPUTS_SERIALIZED 1u
#define SV_TX_INPUTS_SERIALIZED 2u
#define SV_TX_OUTPUTS_ZERO 4u
#endif

// incremental SHA-256 (byte granular): lets the preimage stream through without a bound on the script length
struct sha256_stream {
    u32 st[8];
    u32 blk[16];
    u32 fill;  // bytes in blk
    u64 total;
};
SV_HD void sha_stream_init(sha256_stream& c) {
    sha256_init(c.st);
    c.fill = 0;
    c.total = 0;
    for (int i = 0; i < 16; i++) c.blk[i] = 0;
}
SV_HD void sha_stream_byte(sha256_stream& c, u8 b) {
    u32 w = c.fill >> 2, sh = 24 - 8 * (c.fill & 3);
    c.blk[w] |= (u32)b << sh;
    c.fill++;
    c.total++;
    if (c.fill == 64) {
        sha256_compress(c.st, c.blk);
        for (int i = 0; i < 16; i++) c.blk[i] = 0;
        c.fill = 0;
    }
}
SV_HD void sha_stream_put(sha256_stream& c, const u8* p, size_t n) {
    for (size_t i = 0; i < n; i++) sha_stream_byte(c, p[i]);
}
SV_HD void sha_stream_le(sha256_stream& c, u64 v, int n) {
    for (int i = 0; i < n; i++) sha_stream_byte(c, (u8)(v >> (8 * i)));
}
SV_HD void sha_stream_varint(sha256_stream& c, u64 v) {  // Bitcoin CompactSize
    if (v < 0xfd) { sha_stream_byte(c, (u8)v); return; }
    if (v <= 0xffff) { sha_stream_byte(c, 0xfd); sha_stream_le(c, v, 2); return; }
    sha_stream_byte(c, 0xfe);
    sha_stream_le(c, v, 4);
}
// finish with SHA-256 of the digest (sha256_double), big-endian bytes out
SV_HD void sha_stream_final_double(sha256_stream& c, u8 out32[32]) {
    u64 bits = c.total * 8;
    sha_stream_byte(c, 0x80);
    while (c.fill != 56) sha_stream_byte(c, 0);
    c.blk[14] = (u32)(bits >> 32);
    c.blk[15] = (u32)bits;
    sha256_compress(c.st, c.blk);
    u32 o[8];
    sha256_of_digest(o, c.st);
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (u8)(o[i] >> 24);
        out32[4 * i + 1] = (u8)(o[i] >> 16);
        out32[4 * i + 2] = (u8)(o[i] >> 8);
        out32[4 * i + 3] = (u8)o[i];
    }
}

// The sighash is built in three steps: bip143_prefix (the preimage up to and including nSequence), bip143_hash_outputs
// and bip143_tail.  bip143_sighash runs them in turn; onchaind's fee grind (k_grind) runs the prefix once and the other
// two once per candidate output amount, so both paths hash with the same code.
//
// Prefix: false if the sighash type is not one libwally hashes for a Bitcoin segwit-v0 input: 0 (hashed as ALL), ALL, NONE,
// SINGLE, each with or without ANYONECANPAY (wally_tx_get_input_signature_hash, tx_io.c:972-1009).  Every other value is
// WALLY_EINVAL there, bits above the low byte included, and ANYPREVOUT (0x40, FORKID for Bitcoin) with them.  There is no
// bound on script sizes.  With SV_TX_INPUTS_SERIALIZED hashPrevouts / hashSequence run over the supplied spans
// (multi-input transactions).
SV_HD bool bip143_sighash_type_ok(u32 t) { return t <= 3u || (t >= 0x81u && t <= 0x83u); }
SV_HD bool bip143_prefix(sha256_stream& c, const sv_tx_item& t, const u8* blob) {
    sha_stream_init(c);
    if (!bip143_sighash_type_ok(t.sighash_type)) return false;
    const bool acp = (t.sighash_type & 0x80u) != 0;
    const u32 base = t.sighash_type & 0x1fu;
    const bool sh_none = base == 2, sh_single = base == 3;
    u8 h_prev[32], h_seq[32];
    for (int i = 0; i < 32; i++) { h_prev[i] = 0; h_seq[i] = 0; }
    const bool multi_in = (t.flags & SV_TX_INPUTS_SERIALIZED) != 0;
    if (!acp) {  // hashPrevouts
        sha_stream_init(c);
        if (multi_in) sha_stream_put(c, blob + t.prevouts_off, t.prevouts_len);
        else {
            sha_stream_put(c, t.prev_txid, 32);
            sha_stream_le(c, t.prev_index, 4);
        }
        sha_stream_final_double(c, h_prev);
    }
    if (!(acp || sh_single || sh_none)) {  // hashSequence
        sha_stream_init(c);
        if (multi_in) sha_stream_put(c, blob + t.sequences_off, t.sequences_len);
        else sha_stream_le(c, t.sequence, 4);
        sha_stream_final_double(c, h_seq);
    }
    sha_stream_init(c);
    sha_stream_le(c, t.version, 4);
    sha_stream_put(c, h_prev, 32);
    sha_stream_put(c, h_seq, 32);
    sha_stream_put(c, t.prev_txid, 32);
    sha_stream_le(c, t.prev_index, 4);
    sha_stream_varint(c, t.script_len);
    sha_stream_put(c, blob + t.script_off, t.script_len);
    sha_stream_le(c, t.input_amount, 8);
    sha_stream_le(c, t.sequence, 4);
    return true;
}

// hashOutputs.  By default the transaction has ONE output (output_amount, scriptPubKey span) — the HTLC-transaction
// shape; with SV_TX_OUTPUTS_SERIALIZED the out_script span holds the serialised outputs to commit to (amount ||
// CompactSize || script, concatenated: all of them for SIGHASH_ALL, the one at the input's index for SIGHASH_SINGLE,
// tx_io.c:714-737) — what check_tx_sig's adapter passes for commitment transactions.  32 zero bytes for SIGHASH_NONE and
// SV_TX_OUTPUTS_ZERO.
SV_HD void bip143_hash_outputs(u8 h_out[32], const sv_tx_item& t, const u8* blob, u64 output_amount) {
    for (int i = 0; i < 32; i++) h_out[i] = 0;
    if ((t.sighash_type & 0x1fu) == 2 || (t.flags & SV_TX_OUTPUTS_ZERO)) return;
    sha256_stream c;
    sha_stream_init(c);
    if (t.flags & SV_TX_OUTPUTS_SERIALIZED) {
        sha_stream_put(c, blob + t.out_script_off, t.out_script_len);
    } else {
        sha_stream_le(c, output_amount, 8);
        sha_stream_varint(c, t.out_script_len);
        sha_stream_put(c, blob + t.out_script_off, t.out_script_len);
    }
    sha_stream_final_double(c, h_out);
}

// hashOutputs || nLocktime || sighash type appended to the prefix stream c (consumed), then the double hash
SV_HD void bip143_tail(u8 out32[32], sha256_stream& c, const u8 h_out[32], const sv_tx_item& t) {
    sha_stream_put(c, h_out, 32);
    sha_stream_le(c, t.locktime, 4);
    sha_stream_le(c, t.sighash_type, 4);
    sha_stream_final_double(c, out32);
}

SV_HD bool bip143_sighash(u8 out32[32], const sv_tx_item& t, const u8* blob) {
    sha256_stream c;
    if (!bip143_prefix(c, t, blob)) {
        for (int i = 0; i < 32; i++) out32[i] = 0;
        return false;
    }
    u8 h_out[32];
    bip143_hash_outputs(h_out, t, blob, t.output_amount);
    bip143_tail(out32, c, h_out, t);
    return true;
}
