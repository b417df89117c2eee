// bolt12.cuh — BOLT12 signature hashes: TLV stream parse, Merkle root and tagged sighash.
//
// Reference (paths relative to the Core Lightning tree):
//   parse        fromwire_tlv(..., types = NULL, 0, ..., FROMWIRE_TLV_ANY_TYPE, ...)   wire/tlvstream.c:144-300
//                bigsize_get                                                        common/bigsize.c
//   Merkle root  merkle_tlv                                                         common/bolt12_merkle.c:160-194
//   sighash      sighash_from_merkle -> bip340_sighash_init                         common/bolt12_merkle.c:210-220,
//                                                                                   bitcoin/signature.c:389-405
//
// The hashes run over the raw record bytes of the stream.  CLN re-serialises each field before hashing
// (sha256_update_tlvfield); the two agree because the parse only accepts minimal BigSize encodings.
//
// Every function here is SV_HD: the kernels in engine.cu call them per lane, tests/host_emul compiles the same
// code for the host.  Digests are kept as eight big-endian state words; comparing them word by word as unsigned
// integers orders them as memcmp orders the 32 digest bytes.
#pragma once
#include "sha256.cuh"

// a field of a parsed stream: its numeric type and where its raw record (type, length, value) lies in the stream
struct b12_field {
    u64 type;
    u32 off;  // record start, from the start of the stream
    u32 len;  // whole record: BigSize type + BigSize length + value
};

// tag midstates shared by every stream of a batch: SHA256(tag) || SHA256(tag) already compressed
struct b12_tags {
    u32 leaf[8];     // "LnLeaf"
    u32 branch[8];   // "LnBranch"
    u32 sighash[8];  // "lightning" || messagename || fieldname (one tag; the kernels keep a table of these, one per tag)
};

// bigsize_get (common/bigsize.c): bytes consumed, 0 if truncated or not minimally encoded
SV_HD u32 b12_bigsize(const u8* p, u64 max, u64* val) {
    if (max < 1) return 0;
    u8 b = p[0];
    if (b < 0xfd) { *val = b; return 1; }
    u32 n = b == 0xfd ? 2 : (b == 0xfe ? 4 : 8);
    if (max < 1 + (u64)n) return 0;
    u64 v = 0;
    for (u32 k = 0; k < n; k++) v = (v << 8) | p[1 + k];
    if (b == 0xfd ? v < 0xfd : (b == 0xfe ? (v >> 16) == 0 : (v >> 32) == 0)) return 0;
    *val = v;
    return 1 + n;
}

// One step of the header walk: the record at *pos.  Returns false where fromwire_tlv fails (truncated or non-minimal
// BigSize, type not above prev_type, length past the end).  Reads header bytes only.
SV_HD bool b12_next(const u8* p, u32 len, u32* pos, bool first, u64 prev_type, b12_field* f) {
    u64 t, l;
    u32 a = *pos;
    u32 tl = b12_bigsize(p + a, len - a, &t);
    if (!tl) return false;
    if (!first && t <= prev_type) return false;
    u32 ll = b12_bigsize(p + a + tl, len - a - tl, &l);
    if (!ll) return false;
    u32 rest = len - a - tl - ll;
    if (l > rest) return false;
    f->type = t;
    f->off = a;
    f->len = tl + ll + (u32)l;
    *pos = a + f->len;
    return true;
}

// number of fields of the stream, or -1 if fromwire_tlv refuses it or it is empty (merkle_tlv asserts on an empty
// stream, bolt12_merkle.c:73, so no CLN caller reaches one)
SV_HD long long b12_count(const u8* p, u32 len) {
    u32 pos = 0;
    u64 prev = 0;
    long long cnt = 0;
    b12_field f;
    while (pos < len) {
        if (!b12_next(p, len, &pos, cnt == 0, prev, &f)) return -1;
        prev = f.type;
        cnt++;
    }
    return cnt ? cnt : -1;
}

// BOLT #12: signature TLV elements are types 240 through 1000 inclusive; they stay out of the tree
SV_HD bool b12_is_signature(u64 type) { return type >= 240 && type <= 1000; }

// Continue SHA-256 from state st (which has absorbed `done` bytes, a multiple of 64) over pre[0..prelen) || p[0..len)
// and finish it (padding included).  Byte loads: records are unaligned slices of the stream.
SV_HD void b12_sha_finish(u32 st[8], u64 done, const u8* pre, u32 prelen, const u8* p, u64 len) {
    const u64 total = prelen + len;
    const u64 nblk = (total + 9 + 63) / 64;
    const u64 bits = (done + total) * 8;
    u32 blk[16];
    for (u64 b = 0; b < nblk; b++) {
        for (int w = 0; w < 16; w++) {
            u32 word = 0;
            for (int q = 0; q < 4; q++) {
                u64 k = 64 * b + 4 * w + q;
                u32 byte;
                if (k < total) byte = k < prelen ? pre[k] : p[k - prelen];
                else if (k == total) byte = 0x80;
                else if (k >= 64 * nblk - 8) byte = (u32)(bits >> (8 * (64 * nblk - 1 - k))) & 0xff;
                else byte = 0;
                word = (word << 8) | byte;
            }
            blk[w] = word;
        }
        sha256_compress(st, blk);
    }
}

// midstate of a tagged hash: SHA256(tag) || SHA256(tag) compressed, tag = pre || p
SV_HD void b12_tag_mid(u32 mid[8], const u8* pre, u32 prelen, const u8* p, u64 len) {
    u32 h[8], blk[16];
    sha256_init(h);
    b12_sha_finish(h, 0, pre, prelen, p, len);
    for (int i = 0; i < 8; i++) { blk[i] = h[i]; blk[8 + i] = h[i]; }
    sha256_init(mid);
    sha256_compress(mid, blk);
}

// the two tree midstates, the same for every sighash tag
SV_HD void b12_make_tree_tags(b12_tags* t) {
    const u8 leaf[6] = {'L', 'n', 'L', 'e', 'a', 'f'};
    const u8 branch[8] = {'L', 'n', 'B', 'r', 'a', 'n', 'c', 'h'};
    b12_tag_mid(t->leaf, leaf, 6, leaf, 0);
    b12_tag_mid(t->branch, branch, 8, branch, 0);
}

// the batch's three tag midstates; sigtag = "lightning" || messagename || fieldname (bip340_sighash_init)
SV_HD void b12_make_tags(b12_tags* t, const u8* sigtag, u32 sigtag_len) {
    b12_make_tree_tags(t);
    b12_tag_mid(t->sighash, sigtag, sigtag_len, sigtag, 0);
}

// nonce tag of a stream: "LnNonce" || its first record (fields[0], even when that is a signature field)
SV_HD void b12_nonce_mid(u32 mid[8], const u8* first_rec, u32 first_len) {
    const u8 nonce[7] = {'L', 'n', 'N', 'o', 'n', 'c', 'e'};
    b12_tag_mid(mid, nonce, 7, first_rec, first_len);
}

// H(tag, msg) from the tag's midstate
SV_HD void b12_tagged(u32 out[8], const u32 mid[8], const u8* msg, u64 len) {
    for (int i = 0; i < 8; i++) out[i] = mid[i];
    b12_sha_finish(out, 64, msg, 0, msg, len);
}

// H("LnBranch", lesser || greater)
SV_HD void b12_branch(u32 out[8], const u32 mid[8], const u32 a[8], const u32 b[8]) {
    bool swap = false, decided = false;
    for (int i = 0; i < 8; i++) {
        if (!decided && a[i] != b[i]) { swap = a[i] > b[i]; decided = true; }
    }
    u32 blk[16];
    for (int i = 0; i < 8; i++) { blk[i] = swap ? b[i] : a[i]; blk[8 + i] = swap ? a[i] : b[i]; }
    for (int i = 0; i < 8; i++) out[i] = mid[i];
    sha256_compress(out, blk);
    blk[0] = 0x80000000u;
    for (int i = 1; i < 15; i++) blk[i] = 0;
    blk[15] = (64 + 64) * 8;
    sha256_compress(out, blk);
}

// the leaf pair of one non-signature field: LnBranch(LnLeaf(record), LnNonce(type))
SV_HD void b12_leaf_pair(u32 out[8], const b12_tags* t, const u32 nonce_mid[8], const u8* stream, const b12_field& f) {
    u32 leaf[8], nonce[8];
    b12_tagged(leaf, t->leaf, stream + f.off, f.len);
    // the record starts with the type's (minimal) BigSize encoding: its first 1, 3, 5 or 9 bytes
    u8 b0 = stream[f.off];
    u32 tl = b0 < 0xfd ? 1 : (b0 == 0xfd ? 3 : (b0 == 0xfe ? 5 : 9));
    b12_tagged(nonce, nonce_mid, stream + f.off, tl);
    b12_branch(out, t->branch, leaf, nonce);
}

// sighash_from_merkle: H(sighash tag, root) from the tag's midstate, big-endian bytes out
SV_HD void b12_sighash_mid(u8 out32[32], const u32 mid[8], const u32 root[8]) {
    u32 st[8], blk[16];
    for (int i = 0; i < 8; i++) { st[i] = mid[i]; blk[i] = root[i]; }
    blk[8] = 0x80000000u;
    for (int i = 9; i < 15; i++) blk[i] = 0;
    blk[15] = (64 + 32) * 8;
    sha256_compress(st, blk);
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (u8)(st[i] >> 24); out32[4 * i + 1] = (u8)(st[i] >> 16);
        out32[4 * i + 2] = (u8)(st[i] >> 8); out32[4 * i + 3] = (u8)st[i];
    }
}
SV_HD void b12_sighash(u8 out32[32], const b12_tags* t, const u32 root[8]) { b12_sighash_mid(out32, t->sighash, root); }
