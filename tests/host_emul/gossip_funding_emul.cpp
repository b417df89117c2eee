// tests/host_emul/gossip_funding_emul.cpp — TEST-ONLY host build of lightning_b200/csrc/gossip_funding.cuh (linked into
// libemul.so): the per-announcement funding decision k_store_funding makes, and the 2-of-2 P2WSH script it builds.
// The table is passed already sorted, as the engine's CUB sorts leave it (out_idx NULL: entry i is out_scid[i]).
#include "../../lightning_b200/csrc/gossip_funding.cuh"

extern "C" void emul_gf_p2wsh_2of2(const u8* k1, const u8* k2, u8* out34) { gf_p2wsh_2of2(k1, k2, out34); }

// verdict[i] = gf_verdict of the announcement whose record header is at hdr_off[i]
extern "C" void emul_gf_verdict(const u8* store, u64 len, const u64* hdr_off, size_t n, const u64* out_scid,
                                const u64* sats, const u8* script34, u64 n_out, const u32* blocks, u64 n_blocks,
                                u8* verdict) {
    const gf_table t{out_scid, nullptr, sats, script34, n_out, blocks, n_blocks};
    for (size_t i = 0; i < n; i++) verdict[i] = (u8)gf_verdict(store, len, hdr_off[i], t);
}
