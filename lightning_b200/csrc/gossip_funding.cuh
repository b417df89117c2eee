// gossip_funding.cuh — would gossipd have let a store's channel_announcement in, by lightningd's funding outputs?
//
// gossipd only writes a channel_announcement after lightningd has answered its txout request, and only when the output
// is unspent and is the P2WSH of the announcement's two bitcoin keys; it then writes a channel_amount record with the
// output's amount right after it.  The verdict below makes the same decision from lightningd's own tables.
//
// Reference (paths relative to the Core Lightning tree):
//   txout decision   get_txout: wallet_outpoint_for_scid, else wallet_have_block, else bitcoind  lightningd/gossip_control.c:78-115
//   reply handling   no output: ignore the announcement  gossipd/gossmap_manage.c:791-810
//                    script other than p2wsh(2-of-2):     :696-699, :812-819
//                    the amount record it writes:         :850-852
//   the script       bitcoin_redeem_2of2 (keys ordered by pubkey_cmp)  bitcoin/script.c:151-167, bitcoin/pubkey.c:84-90
//                    scriptpubkey_p2wsh: OP_0 PUSH32 SHA-256(script)
//   dying channels   GOSSIP_STORE_DYING_BIT on the announcement's header   gossipd/gossmap_manage.c:1420-1433
//   capacity         the record right after the announcement, read whatever its flags   common/gossmap.c:1473-1499
//
// gf_verdict is SV_HD: k_store_funding in engine.cu runs it per candidate announcement, tests/host_emul compiles it for
// the host.
#pragma once
#include "common.cuh"
#include "gossip_store.cuh"
#include "sha256.cuh"

// verdicts (include/cln_sigverify.h SV_GF_*)
#define GF_NONE 0
#define GF_FUNDED 1
#define GF_UNCHECKED 2
#define GF_DYING 3
#define GF_NO_TXOUT 4
#define GF_SCRIPT 5
#define GF_AMOUNT 6
#define GS_DYING 0x0800u
// the verdicts gossipd would have refused the announcement for: the prune deletes them
SV_HD bool gf_refused(u32 v) { return v >= GF_NO_TXOUT; }

// st = SHA-256(OP_2 PUSH33 ka PUSH33 kb OP_2 OP_CHECKMULTISIG), ka the key that memcmp orders first.  The 71-byte script
// and its padding are exactly two compression blocks, built word by word at fixed byte positions (unrolled on the
// device, so the script lives in registers).
SV_HD void gf_2of2_hash(const u8* k1, const u8* k2, u32 st[8]) {
    int c = 0;
    for (int b = 0; b < 33 && c == 0; b++) c = (int)k1[b] - (int)k2[b];
    const u8 *a = c < 0 ? k1 : k2, *z = c < 0 ? k2 : k1;
    u32 w[32];
    SV_UNROLL
    for (int i = 0; i < 32; i++) w[i] = 0;
    SV_UNROLL
    for (int i = 0; i < 72; i++) {
        const u32 v = i == 0 || i == 69 ? 0x52u : i == 1 || i == 35 ? 33u : i < 35 ? a[i - 2] : i < 69 ? z[i - 36]
                      : i == 70 ? 0xAEu : 0x80u;
        w[i >> 2] |= v << (24 - 8 * (i & 3));
    }
    w[31] = 71 * 8;  // the message length in bits
    sha256_init(st);
    sha256_compress(st, w);
    sha256_compress(st, w + 16);
}

// out34 = OP_0 PUSH32 SHA-256(script): scriptpubkey_p2wsh of the 2-of-2
SV_HD void gf_p2wsh_2of2(const u8* k1, const u8* k2, u8 out34[34]) {
    u32 st[8];
    gf_2of2_hash(k1, k2, st);
    out34[0] = 0x00;
    out34[1] = 0x20;
    for (int i = 0; i < 32; i++) out34[2 + i] = (u8)(st[i >> 2] >> (24 - 8 * (i & 3)));
}

// the lowest index i < n with a[i] >= x (n if none), a ascending
template <typename T>
SV_HD u64 gf_lower_bound(const T* a, u64 n, T x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = lo + (hi - lo) / 2;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The funding table, sorted: out_scid ascending (unique), out_idx[i] the caller's entry of out_scid[i], whose amount is
// sats[out_idx[i]] and whose script is script34[34 * out_idx[i]]; blocks ascending.
struct gf_table {
    const u64* out_scid;
    const u32* out_idx;
    const u64* sats;
    const u8* script34;
    u64 n_out;
    const u32* blocks;
    u64 n_blocks;
};

// The verdict of the channel_announcement whose record header is at hdr_off of a store of len bytes (its message parsed,
// so its fields lie inside the store).  The bitcoin keys and the scid are read at their fixed offsets after the
// features, as k_gossip_slice locates them.
SV_HD u32 gf_verdict(const u8* store, u64 len, u64 hdr_off, const gf_table& t) {
    const u8* h = store + hdr_off;
    if (gs_be16(h) & GS_DYING) return GF_DYING;
    const u8* m = h + GS_HDR;
    const u8* f = m + 260 + gs_be16(m + 258);  // chain_hash, scid, node_id_1, node_id_2, bitcoin_key_1, bitcoin_key_2
    u64 scid = 0;
    for (int b = 0; b < 8; b++) scid = (scid << 8) | f[32 + b];
    const u64 i = gf_lower_bound(t.out_scid, t.n_out, scid);
    if (i == t.n_out || t.out_scid[i] != scid) {
        const u32 block = (u32)(scid >> 40);
        const u64 j = gf_lower_bound(t.blocks, t.n_blocks, block);
        return j < t.n_blocks && t.blocks[j] == block ? GF_NO_TXOUT : GF_UNCHECKED;
    }
    const u64 e = t.out_idx ? t.out_idx[i] : i;
    u32 st[8];
    gf_2of2_hash(f + 106, f + 139, st);
    const u8* got = t.script34 + 34 * e;
    bool same = got[0] == 0x00 && got[1] == 0x20;
    SV_UNROLL
    for (int b = 0; b < 32; b++) same &= got[2 + b] == (u8)(st[b >> 2] >> (24 - 8 * (b & 3)));
    if (!same) return GF_SCRIPT;
    // the record directly after the announcement, by the header's length: a channel_amount holding the output's amount
    const u64 a = hdr_off + GS_HDR + gs_be16(h + 2);
    if (a + GS_HDR + 2 + 8 > len || gs_be16(store + a + GS_HDR) != GS_CHANNEL_AMOUNT) return GF_AMOUNT;
    u64 sat = 0;
    for (int b = 0; b < 8; b++) sat = (sat << 8) | store[a + GS_HDR + 2 + b];
    return sat == t.sats[e] ? GF_FUNDED : GF_AMOUNT;
}
