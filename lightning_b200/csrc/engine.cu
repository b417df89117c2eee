// engine.cu — kernels and C ABI of libcln_sigverify.so (sm_90a, H100).
//
// Kernels (SURVEY.md §2.3 naming):
//   K4  k_gtable_bases / k_gtable_fill   fixed-base comb table d * 2^(16 i) * G, built once per context
//   K3  k_sha256d                        SHA-256d of message spans (gossip tails, BIP143 preimages)
//   K1a k_prep_inv + k_prep_finish       scalar side of ECDSA (32 signatures per thread share one s^-1 exponentiation;
//                                        then one thread per signature: u1, u2, GLV split, recoding)
//   K2a k_prep_schnorr                   scalar side of BIP-340 (tagged challenge hash, -e, recoding)
//   K1b/K2b k_main<kind>                 curve side: thread per verification, persistent grid.  kind 3 / 4 = compressed /
//                                        x-only keys WITHOUT the square root (verify.cuh): the default for kinds 0 / 2
//       k_final_ecdsa33, k_final_schnorr_ns   batched division that settles the parked linear conditions of kinds 3 / 4
//       k_final_schnorr                  plain BIP-340 flow: affine R from the parked Jacobian R (batched inversion)
//       k_small<kind>                    one-launch latency path for small batches (5 warps per 32 verifications)
//       k_main_shared, k_dedup_*, k_sharedkey_build_many   one multiples table per distinct key (same-key / gossip batches)
//       k_gossip_slice / _status, k_bip143, k_mixed_*       callers' data formats on the device (rows N1, N2, C3)
//       k_b12_*                          BOLT12 streams: TLV parse, Merkle root (one warp per stream), tagged sighash
//       k_b11_*                          BOLT11 invoices: bech32, field walk, signing hash; public-key recovery around
//                                        k_main<SV_KIND_SCHNORR> (prep of u1, u2 and R.x, then affine Q compressed)
//       k_sb_* (batch.cu)                BIP-340 batch verification by random linear combination
//       k_pack_bitmap                    verdict bytes -> 1 bit per verification (ballot)
//       k_pubkey_parse                   batched pubkey_from_der
//       k_synth                          synthetic signed workload generator (benchmarks/tests)
//       k_probe_*                        integer-pipe microbenchmarks (roofline denominator)
//
// There is no host implementation of any of the arithmetic in this library: every entry point either
// runs the kernels or fails with an error code.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <stdio.h>
#include <chrono>
#include <memory>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>

#include "../../include/cln_sigverify.h"
#include "verify.cuh"
#include "bolt12.cuh"
#include "bolt11.cuh"
#include "gossip_store.cuh"
#include "gossip_salvage.cuh"
#include "gossip_funding.cuh"
#include "selftest.cuh"
#include "batch.cuh"  // constants and the host-testable stages; the kernels themselves are in batch.cu

#if !defined(SV_NO_SYNC_INLINE) && !defined(SV_FE_INLINE)
#error "compile with -DSV_FE_INLINE -DSV_MAIN_SYNC (default build) or -DSV_NO_SYNC_INLINE; see lightning_b200/build.py"
#endif
#ifdef SV_MAIN_SYNC
#define SV_MAIN_BLOCK 256
#else
#define SV_MAIN_BLOCK 128
#endif
#define SV_MAIN_MINB (512 / SV_MAIN_BLOCK)

// -------------------------------------------------------------------------------------------------
// kernels
// -------------------------------------------------------------------------------------------------
__global__ void k_gtable_bases(ge_mem* bases) {
    if (blockIdx.x == 0 && threadIdx.x == 0) gtable_make_bases(bases);
}
__global__ void __launch_bounds__(128) k_gtable_fill(ge_mem* table, const ge_mem* bases) {
    u32 e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < SV_GT_ENTRIES) gtable_make_entry(table, bases, e);
}

__global__ void __launch_bounds__(128) k_sha256d(const u8* data, const u64* off, const u32* len, size_t n, u8* out32) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) sha256d_bytes(out32 + 32 * i, data + off[i], len[i]);
}

// scalar side, ECDSA, in two kernels.
//   k_prep_inv    : each thread owns SV_PREP_BATCH (32) consecutive signatures: range checks and ONE Fermat
//                   exponentiation mod n amortised by Montgomery's trick (3 mults + 1/32 of ~330 per signature).  Few
//                   threads, long serial chains: latency bound, so it does nothing else.  Leaves s^-1 and the check
//                   flags in the (not yet used) work record.
//   k_prep_finish : one thread per signature: u1 = m/s, u2 = r/s, GLV split, window recoding -> work record.
__global__ void __launch_bounds__(64) k_prep_inv(const u8* msg, const u8* sig, size_t n, sv_work* work) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t base = t * SV_PREP_BATCH;
    if (base >= n) return;
    int cnt = (int)((n - base < SV_PREP_BATCH) ? (n - base) : SV_PREP_BATCH);
    sc sv[SV_PREP_BATCH];
    u32 okmask = 0, parsedmask = 0;
#pragma unroll 1
    for (int j = 0; j < SV_PREP_BATCH; j++) {
        sc r, s, m;
        bool ok = false, parsed = false;
        if (j < cnt) ok = ecdsa_parse(r, s, m, sig + 64 * (base + j), msg + 32 * (base + j), &parsed);
        parsedmask |= (parsed ? 1u : 0u) << j;
        if (!ok) {
#pragma unroll
            for (int k = 0; k < 8; k++) s.v[k] = (k == 0);
        }
        okmask |= (ok ? 1u : 0u) << j;
        sv[j] = s;
    }
    sc_batch_inverse(sv, SV_PREP_BATCH);
#pragma unroll 1
    for (int j = 0; j < cnt; j++) {
        u32* w = reinterpret_cast<u32*>(work + base + j);
        fe_to_words(w, *reinterpret_cast<const fe*>(&sv[j]));  // words 0..7: s^-1
        w[8] = ((okmask >> j) & 1u) | (((parsedmask >> j) & 1u) << 1);
    }
}
__global__ void __launch_bounds__(128) k_prep_finish(const u8* msg, const u8* sig, size_t n, sv_work* work) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32* wi = reinterpret_cast<const u32*>(work + i);
    sc sinv;
    fe tmp;
    fe_from_words(tmp, wi);
#pragma unroll
    for (int k = 0; k < 8; k++) sinv.v[k] = tmp.v[k];
    u32 f = wi[8];
    sc r, s, m;
    (void)ecdsa_parse(r, s, m, sig + 64 * i, msg + 32 * i);
    sv_work w;
    ecdsa_finish_prep(w, (f & 1u) != 0, r, m, sinv, (f & 2u) != 0);
    work[i] = w;
}

__global__ void __launch_bounds__(128) k_prep_schnorr(const u8* msg, const u8* key, const u8* sig, size_t n,
                                                      sv_work* work) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    sv_work w;
    schnorr_prep(w, sig + 64 * i, key + 32 * i, msg + 32 * i);
    work[i] = w;
}

// curve side: one thread per verification, persistent grid-stride loop.  Per-thread odd-multiples
// table lives in an HBM/L2-resident scratch slab (768 B per thread, 64-byte entries read with LDG.128).
// record used by lanes past the end of the batch: harmless scalars (k1 = k2 = 1, u1 = 0), never valid.
// (They must not alias a live record: the BIP-340 path overwrites records with the parked R.)
__device__ sv_work g_idle_work = {{1, 0, 0, 0, 0}, {1, 0, 0, 0, 0}, {0}, 0, {0}};

template <int KIND>
__global__ void __launch_bounds__(SV_MAIN_BLOCK, SV_MAIN_MINB)
    k_main(sv_work* work, const u8* __restrict__ key, const u8* __restrict__ sig, size_t n,
           const ge_mem* __restrict__ gtab, qtab_entry* scratch, u8* __restrict__ verdict, u8* keyok) {
    const size_t keylen = (KIND == SV_KIND_ECDSA33 || KIND == SV_KIND_ECDSA33_NS) ? 33 : (KIND == SV_KIND_ECDSA_XY ? 64 : 32);
    size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    qtab_entry* tab = scratch + tid * 8;
    // CTA-uniform trip count (lanes past the end redo dummy work and discard the result) so that every thread
    // reaches every SV_SYNC() of the barrier-synchronised build
    for (size_t base = (size_t)blockIdx.x * blockDim.x; base < n; base += stride) {
        size_t i = base + threadIdx.x;
        bool active = i < n;
        size_t j = active ? i : 0;
        const unsigned part = SV_MAIN_BLOCK;  // every thread of the CTA reaches every re-convergence barrier
        const sv_work* w = active ? (work + i) : &g_idle_work;
        if (KIND == SV_KIND_ECDSA33_NS) {
            // compressed-key ECDSA without the square root: D, B, c parked in the work record, k_final_ecdsa33 decides
            u32 code = ecdsa33_nosqrt_curve_side(w, key + keylen * j, sig + 64 * j, gtab, tab,
                                                 reinterpret_cast<sv_ns_park*>(work + j), active, part);
            if (active) verdict[i] = (u8)code;
        } else if (KIND == SV_KIND_SCHNORR_NS) {
            u32 code = schnorr_nosqrt_curve_side(w, key + keylen * j, sig + 64 * j, gtab, tab,
                                                 reinterpret_cast<sv_ns_park_schnorr*>(work + j), active, part);
            if (active) verdict[i] = (u8)code;
        } else if (KIND == SV_KIND_SCHNORR) {
            // park R in the work record; k_final_schnorr turns it into a verdict (batched inversion)
            bool ok = (w->flags & SV_WF_VALID) != 0;
            ge Q;
            ok = key_decode(Q, KIND, key + keylen * j) && ok;
            gej R;
            ecmult_uniform(R, w, Q, gtab, tab, part);
            if (active) schnorr_park(reinterpret_cast<sv_jac*>(work + i), R, ok);
        } else {
            bool kd;
            u32 v = verify_curve_side(KIND, w, key + keylen * j, sig + 64 * j, gtab, tab, &kd, part);
            if (active) {
                verdict[i] = (u8)v;
                // gossip ingest distinguishes "undecodable key" / "unparsable signature" (malformed message) from a bad signature
                if (keyok) keyok[i] = (u8)((kd ? 1u : 0u) | ((w->flags & SV_WF_PARSED) ? 2u : 0u));
            }
        }
    }
}

// ---- small-batch path (verify.cuh "small-batch path"): one CTA = 5 warps x up to 32 items.  The inputs may live in host-mapped pinned memory (zero-copy: the CTA pulls its items into shared memory
// with warp-coalesced loads) or in device memory.  aux (optional): bit 0 = key decoded, bit 1 = signature encoding parsed.
#define SV_SMALL_ITEMS 32
template <int KIND, bool NOSQRT>
__global__ void __launch_bounds__(160, 1)
    k_small(const u8* __restrict__ msg, const u8* __restrict__ key, const u8* __restrict__ sig, size_t n,
            const ge_mem* __restrict__ gtab, u8* __restrict__ verdict, u8* __restrict__ aux) {
    constexpr int keylen = (KIND == SV_KIND_ECDSA33) ? 33 : (KIND == SV_KIND_ECDSA_XY ? 64 : 32);
    __shared__ sv_small_item items[SV_SMALL_ITEMS];
    __shared__ __align__(16) u8 in_msg[SV_SMALL_ITEMS * 32];
    __shared__ __align__(16) u8 in_key[SV_SMALL_ITEMS * 64];
    __shared__ __align__(16) u8 in_sig[SV_SMALL_ITEMS * 64];
    const size_t base = (size_t)blockIdx.x * SV_SMALL_ITEMS;
    const int cnt = (int)((n - base < SV_SMALL_ITEMS) ? (n - base) : SV_SMALL_ITEMS);
    for (int t = threadIdx.x; t < cnt * 32; t += blockDim.x) in_msg[t] = msg[32 * base + t];
    for (int t = threadIdx.x; t < cnt * keylen; t += blockDim.x) in_key[t] = key[(size_t)keylen * base + t];
    for (int t = threadIdx.x; t < cnt * 64; t += blockDim.x) in_sig[t] = sig[64 * base + t];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // phase A (warps 0, 1) and the comb / finish: lane l works on item l; idle lanes redo item 0 into their own slot
    const bool active = lane < cnt;
    const int j = active ? lane : 0;
    sv_small_item* it = &items[lane];
    const u8* m = in_msg + 32 * j;
    const u8* k = in_key + keylen * j;
    const u8* sg = in_sig + 64 * j;
    if (warp == 0) {
        if (NOSQRT) small_key_side_ns(KIND, k, it); else small_key_side(KIND, k, it);
    } else if (warp == 1) small_scalar_side(KIND, m, k, sg, it);
    __syncthreads();
    // phase B: warps 0..3 run the half ladders on lane PAIRS (warp w: half w >> 1, items 16 (w & 1) + lane / 2), warp 4 the comb
    if (warp < 4) {
        pair_lane L;
        L.role = lane & 1;
        small_half_ladder_pair(L, &items[16 * (warp & 1) + (lane >> 1)], warp >> 1);
    } else {
        small_comb(it, gtab);
    }
    __syncthreads();
    if (warp == 0) {
        bool kd = false;
        u32 v = NOSQRT ? small_finish_ns(KIND, it, k, sg, gtab, aux ? &kd : nullptr) : small_finish(KIND, it, sg, &kd);
        if (active) {
            verdict[base + lane] = (u8)v;
            if (aux) aux[base + lane] = (u8)((kd ? 1u : 0u) | ((it->w.flags & SV_WF_PARSED) ? 2u : 0u));
        }
    }
}

// ---- mixed batches (config C3: interleaved ECDSA + BIP-340 with a 1-byte kind tag per item) ---------------------
// The curve kernels are specialised per kind (a warp must be homogeneous), so a mixed batch is split on the DEVICE:
// k_mixed_index appends every item to its kind's index list (warp-aggregated atomics), k_mixed_gather copies each kind's
// items into that kind's dense SoA region, the per-kind kernels run, k_mixed_scatter puts the verdicts back in item order.
__global__ void __launch_bounds__(256) k_mixed_index(const u8* __restrict__ kinds, size_t n, u32* __restrict__ count,
                                                     u32* __restrict__ idx) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    u32 k = (i < n) ? kinds[i] : 3u;
    if (k > 2u) k = 3u;  // unknown kind: no list (verdict stays 0)
    unsigned peers = __match_any_sync(0xFFFFFFFFu, k);
    if (k < 3u) {
        int leader = __ffs(peers) - 1;
        u32 base = 0;
        if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(&count[k], (u32)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        u32 rank = (u32)__popc(peers & ((1u << (threadIdx.x & 31)) - 1u));
        idx[(size_t)k * n + base + rank] = (u32)i;
    }
}
__global__ void __launch_bounds__(256) k_mixed_gather(const u32* __restrict__ idx, size_t c, int keylen,
                                                      const u8* __restrict__ msg, const u8* __restrict__ key64,
                                                      const u8* __restrict__ sig, u8* __restrict__ o_msg,
                                                      u8* __restrict__ o_key, u8* __restrict__ o_sig) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= c) return;
    size_t i = idx[j];
    const uint4* m = reinterpret_cast<const uint4*>(msg + 32 * i);
    const uint4* sg = reinterpret_cast<const uint4*>(sig + 64 * i);
    uint4* om = reinterpret_cast<uint4*>(o_msg + 32 * j);
    uint4* os = reinterpret_cast<uint4*>(o_sig + 64 * j);
    om[0] = m[0]; om[1] = m[1];
    os[0] = sg[0]; os[1] = sg[1]; os[2] = sg[2]; os[3] = sg[3];
    for (int b = 0; b < keylen; b++) o_key[(size_t)keylen * j + b] = key64[64 * i + b];
}
__global__ void __launch_bounds__(256) k_mixed_scatter(const u32* __restrict__ idx, size_t c, const u8* __restrict__ v,
                                                       u8* __restrict__ out) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < c) out[idx[j]] = v[j];
}

// ---- BIP-340 batch verification: the kernels live in batch.cu (compiled with fe_mul / fe_sqr as real functions) ----------
extern "C" int sv_batch_launch(const u8* d_msg, const u8* d_key, const u8* d_sig, size_t n, const u8* d_seed, void* d_pts,
                               signed char* d_dig, void* d_t, u8* d_ok, void* d_S, u8* d_gok, u8* d_out, const void* d_gtab,
                               cudaStream_t st, cudaEvent_t ev_mid);
__global__ void __launch_bounds__(256) k_sb_gather(const u32* __restrict__ idx, size_t c, const u8* __restrict__ msg, const u8* __restrict__ key32,
                                                   const u8* __restrict__ sig, u8* __restrict__ o_msg, u8* __restrict__ o_key, u8* __restrict__ o_sig) {
    size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= c) return;
    size_t i = idx[j];
    const uint4* m = reinterpret_cast<const uint4*>(msg + 32 * i);
    const uint4* k = reinterpret_cast<const uint4*>(key32 + 32 * i);
    const uint4* sg = reinterpret_cast<const uint4*>(sig + 64 * i);
    uint4* om = reinterpret_cast<uint4*>(o_msg + 32 * j);
    uint4* ok = reinterpret_cast<uint4*>(o_key + 32 * j);
    uint4* os = reinterpret_cast<uint4*>(o_sig + 64 * j);
    om[0] = m[0]; om[1] = m[1];
    ok[0] = k[0]; ok[1] = k[1];
    os[0] = sg[0]; os[1] = sg[1]; os[2] = sg[2]; os[3] = sg[3];
}

// ---- one key, many signatures (N3): build the key's table once, then a ladder-only curve kernel --------------
__global__ void k_sharedkey_build(int kind, const u8* key, sv_shared_key* out) {
    sharedkey_build(out, kind, key, blockDim.x);  // all 32 lanes compute the same values and store to the same addresses
}
__global__ void __launch_bounds__(SV_MAIN_BLOCK, SV_MAIN_MINB)
    k_main_shared(const sv_work* work, const u8* __restrict__ sig, size_t n, const ge_mem* __restrict__ gtab,
                  const sv_shared_key* sk, const u32* __restrict__ sk_index, u8* __restrict__ verdict, u8* __restrict__ aux) {
    // sk_index == nullptr: ONE key for the whole batch (channeld's HTLC loop); else item i uses table sk[sk_index[i]]
    // (key de-duplication inside a gossip batch: every distinct key is decoded and tabulated once)
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t base = (size_t)blockIdx.x * blockDim.x; base < n; base += stride) {
        size_t i = base + threadIdx.x;
        bool active = i < n;
        const sv_work* w = active ? (work + i) : &g_idle_work;
        const sv_shared_key* k = sk_index ? (sk + sk_index[active ? i : 0]) : sk;
        u32 v = verify_curve_side_shared(w, sig + 64 * (active ? i : 0), gtab, k, blockDim.x);
        if (active) {
            verdict[i] = (u8)v;
            if (aux) aux[i] = (u8)((k->ok ? 1u : 0u) | ((w->flags & SV_WF_PARSED) ? 2u : 0u));
        }
    }
}

// ---- key de-duplication (N3): exact (full 33-byte compare) open-addressing hash table keyed by the key bytes ----
__global__ void __launch_bounds__(256) k_dedup_insert(const u8* __restrict__ key, int keylen, size_t n, u32* slots, u32 mask,
                                                      u32* __restrict__ rep) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u8* k = key + (size_t)keylen * i;
    u32 h = 2166136261u;
    for (int b = 0; b < 12; b++) h = (h ^ k[b]) * 16777619u;  // FNV-1a over the prefix and the top of x
    u32 slot = (h ^ (h >> 15)) & mask;
    for (;;) {
        u32 old = atomicCAS(&slots[slot], 0xFFFFFFFFu, (u32)i);
        if (old == 0xFFFFFFFFu) { rep[i] = (u32)i; return; }
        const u8* o = key + (size_t)keylen * old;
        bool same = true;
        for (int b = 0; b < keylen; b++) same = same && (o[b] == k[b]);
        if (same) { rep[i] = old; return; }
        slot = (slot + 1) & mask;
    }
}
__global__ void __launch_bounds__(256) k_dedup_number(const u32* __restrict__ rep, size_t n, u32* counter, u32* __restrict__ tid,
                                                      u32* __restrict__ replist) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || rep[i] != (u32)i) return;
    u32 t = atomicAdd(counter, 1u);
    tid[i] = t;
    replist[t] = (u32)i;
}
__global__ void __launch_bounds__(256) k_dedup_resolve(const u32* __restrict__ rep, size_t n, u32* __restrict__ tid) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && rep[i] != (u32)i) tid[i] = tid[rep[i]];
}
__global__ void __launch_bounds__(128) k_sharedkey_build_many(int kind, const u8* __restrict__ key, int keylen,
                                                              const u32* __restrict__ replist, u32 distinct, sv_shared_key* out) {
    u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < distinct) sharedkey_build(out + t, kind, key + (size_t)keylen * replist[t]);
}

// ---- device-side BIP143 (SURVEY.md §8f N2): one thread per transaction input -> msg32 ----------------------
__global__ void __launch_bounds__(128) k_bip143(const sv_tx_item* txs, const u8* blob, size_t n, u8* msg32, u8* okout) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    okout[i] = bip143_sighash(msg32 + 32 * i, txs[i], blob) ? 1 : 0;
}
// force verdict 0 where the sighash could not be formed
__global__ void k_mask_verdicts(u8* verdict, const u8* ok, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && !ok[i]) verdict[i] = 0;
}

// ---- onchaind's HTLC fee grind (verify.cuh grind_*): one warp builds the shared state, then one thread per feerate ----
__global__ void k_grind_setup(int kind, const u8* key, const u8* sig, const sv_tx_item* tx, const u8* blob, qtab_entry* tab,
                              sv_grind_state* out) {
    sv_grind_state g;  // all 32 lanes compute the same values (the table stores coincide); lane 0 publishes the state
    grind_setup(&g, tab, kind, key, sig, *tx, blob, blockDim.x);
    if (threadIdx.x == 0) *out = g;
}
// feerates first .. first + count - 1; *best = the lowest feerate that verified so far (UINT64_MAX: none)
__global__ void __launch_bounds__(128) k_grind(const sv_grind_state* __restrict__ g, const sv_tx_item* __restrict__ tx,
                                               const u8* __restrict__ blob, const u8* __restrict__ sig,
                                               const ge_mem* __restrict__ gtab, u64 weight, u64 min_feerate, u64 first,
                                               u64 count, unsigned long long* best) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const u64 f = first + i;
    const sv_tx_item t = *tx;
    u64 fee;
    if (!grind_feerate_checked(f, weight, min_feerate, t.input_amount, &fee)) return;
    if (f > *(volatile unsigned long long*)best) return;  // a lower feerate of this chunk matched already
    if (grind_candidate(g, t, blob, sig, t.input_amount - fee, gtab)) atomicMin(best, (unsigned long long)f);
}

// ---- gossip ingest (SURVEY.md §8f N1): the device slices raw wire messages itself ----------------------------
// One thread per message.  Field offsets: wire/peer_wire.csv:340-377; signed regions and checking order:
// gossipd/sigcheck.c:9-43 (channel_update), 45-115 (channel_announcement), 118-164 (node_announcement).
// item_base[m] is the first item slot of message m (4 slots for a channel_announcement, 1 otherwise, host-computed
// from the 2-byte type).  Writes span (off,len), key33, sig64 per item; status[m] = -1 if malformed.
// Burst mode (chain32 != nullptr, sv_verify_gossip_burst_host): gossipd's gates after the parse
// (gossipd/gossmap_manage.c:659-670, :1048-1051) set status[m] = -4 (channel_announcement whose node_id_1 is not below
// node_id_2) or -3 (chain_hash other than chain32); the items are still sliced, because a signature encoding or
// bitcoin_key the wire parser refuses makes the message -1 first.  A channel_update takes signers33[m] only where
// kinds[m] == 1; the other updates get their key from k_gossip_resolve.
__global__ void __launch_bounds__(128) k_gossip_slice(const u8* blob, const u64* msg_off, const u32* msg_len,
                                                      const u32* item_base, const u8* signers33, size_t n_msgs,
                                                      u64* span_off, u32* span_len, u8* key33, u8* sig64, int* status,
                                                      const u8* chain32, const u8* kinds) {
    size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msgs) return;
    const u8* p = blob + msg_off[m];
    u32 len = msg_len[m];
    u32 type = len >= 2 ? (((u32)p[0] << 8) | p[1]) : 0;
    u32 base = item_base[m];
    int nitems = (type == 256) ? 4 : ((type == 257 || type == 258) ? 1 : 0);
    int st = 0;
    u32 hoff = (type == 256) ? 258 : 66;
    u32 keys = 0;
    if (type == 256) {
        if (len < 260) st = -1;
        else {
            u32 flen = ((u32)p[258] << 8) | p[259];
            keys = 260 + flen + 32 + 8;
            if (len < keys + 4 * 33) st = -1;
        }
    } else if (type == 257) {
        // signature(64) flen(2) features timestamp(4) node_id(33) rgb_color(3) alias(32) addrlen(2) addresses
        // (wire/peer_wire.csv:353-362): fromwire_node_announcement fails on any shorter message
        if (len < 68) st = -1;
        else {
            u32 flen = ((u32)p[66] << 8) | p[67];
            keys = 68 + flen + 4;
            if (len < keys + 33 + 3 + 32 + 2) st = -1;
            else {
                u32 alen = ((u32)p[keys + 68] << 8) | p[keys + 69];
                if (len < keys + 70 + alen) st = -1;
            }
        }
    } else if (type == 258) {
        // signature(64) chain_hash(32) short_channel_id(8) timestamp(4) message_flags(1) channel_flags(1)
        // cltv_expiry_delta(2) htlc_minimum_msat(8) fee_base_msat(4) fee_proportional_millionths(4)
        // htlc_maximum_msat(8) = 138 bytes with the type (wire/peer_wire.csv:366-377; htlc_maximum_msat is mandatory)
        if (len < 138 || (signers33 == nullptr && chain32 == nullptr)) st = -1;
    } else {
        st = -1;
    }
    int gate = 0;
    if (chain32 && st == 0 && type != 257) {
        const u8* ch = p + ((type == 256) ? keys - 40 : 66);
        for (int b = 0; b < 32; b++) gate |= ch[b] ^ chain32[b];
        gate = gate ? -3 : 0;
        if (type == 256) {
            int c = 0;  // node_id_cmp: memcmp of the 33 bytes
            for (int b = 0; b < 33 && c == 0; b++) c = (int)p[keys + b] - (int)p[keys + 33 + b];
            if (c >= 0) gate = -4;
        }
    }
    const bool cu_key = !chain32 || (kinds[m] == 1);
    for (int k = 0; k < nitems; k++) {
        u32 it = base + k;
        bool ok = (st == 0);
        span_off[it] = msg_off[m] + (ok ? hoff : 0);
        span_len[it] = ok ? (len - hoff) : 0;
        const u8* kp = (type == 258) ? (signers33 ? signers33 + 33 * m : p) : (p + keys + 33 * k);
        const bool kok = ok && (type != 258 || cu_key);
        for (int b = 0; b < 33; b++) key33[33 * (size_t)it + b] = kok ? kp[b] : 0;  // an all-zero key never verifies
        const u8* sp = p + 2 + 64 * k;
        for (int b = 0; b < 64; b++) sig64[64 * (size_t)it + b] = ok ? sp[b] : 0;
    }
    status[m] = st ? st : gate;
}

// ---- gossip bursts: a channel_update's signer found among the batch's own channel_announcements ------------------
// The scid table is exact open addressing keyed by the 8 scid bytes (k_dedup_insert's pattern): a slot holds a message
// index, the bytes are compared in the blob, and atomicMin keeps the LOWEST index of each scid (a slot only ever changes
// to another index of the same scid, so a concurrent probe still compares the right bytes).
#define SV_SCID_EMPTY 0xFFFFFFFFu
__device__ __forceinline__ const u8* gossip_scid(const u8* p) {
    // channel_announcement: after 4 signatures, features, chain_hash; channel_update: after signature and chain_hash
    return (p[1] == 0) ? p + 260 + (((u32)p[258] << 8) | p[259]) + 32 : p + 98;
}
__device__ __forceinline__ u32 scid_hash(const u8* s) {
    u32 h = 2166136261u;
    for (int b = 0; b < 8; b++) h = (h ^ s[b]) * 16777619u;
    return h ^ (h >> 15);
}
__device__ __forceinline__ bool scid_same(const u8* a, const u8* b) {
    bool same = true;
    for (int k = 0; k < 8; k++) same = same && (a[k] == b[k]);
    return same;
}
// every channel_announcement whose status is 0 goes in: after k_gossip_slice these are the well-formed, right-chain,
// ordered ones; after k_gossip_status the ones whose four signatures verify
__global__ void __launch_bounds__(256) k_scid_insert(const u8* blob, const u64* msg_off, const u32* msg_len, const int* status,
                                                     size_t n_msgs, u32* slots, u32 mask) {
    size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msgs || status[m] != 0 || msg_len[m] < 2) return;
    const u8* p = blob + msg_off[m];
    if (p[0] != 1 || p[1] != 0) return;
    const u8* s = gossip_scid(p);
    u32 slot = scid_hash(s) & mask;
    for (;;) {
        u32 old = atomicCAS(&slots[slot], SV_SCID_EMPTY, (u32)m);
        if (old == SV_SCID_EMPTY) return;
        if (scid_same(gossip_scid(blob + msg_off[old]), s)) { atomicMin(&slots[slot], (u32)m); return; }
        slot = (slot + 1) & mask;
    }
}
// One thread per channel_update that takes its signer from the batch (kinds 0 and 2, status 0 after the slice).  The
// candidate is the lowest-index announcement of the scid in the table; it counts only if it comes before the update.
// cand[m] = its index (the key is its node_id_1 or node_id_2 by channel_flags & 1, byte 111) or SV_SCID_EMPTY (the key
// is signers33[m] for kind 2, all zero otherwise).  list == nullptr: every message, item slot item_base[m].  list = the
// repair list ([count, m...]): update list[1 + t] moves to item slot tail + t, with its hash and signature.
__global__ void __launch_bounds__(128) k_gossip_resolve(const u8* blob, const u64* msg_off, const u32* msg_len, u32* item_base,
                                                        const int* status, const u8* kinds, const u8* signers33,
                                                        size_t n, const u32* slots, u32 mask, u32* cand, const u32* list,
                                                        u32 tail, u8* msg32, u8* key33, u8* sig64) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    size_t m = list ? list[1 + t] : t;
    if (!list) {
        if (status[m] != 0 || kinds[m] == 1 || msg_len[m] < 2) return;
        const u8* q = blob + msg_off[m];
        if (q[0] != 1 || q[1] != 2) return;
    }
    const u8* p = blob + msg_off[m];
    u32 it = item_base[m];
    if (list) {
        u32 to = tail + (u32)t;
        for (int b = 0; b < 32; b++) msg32[32 * (size_t)to + b] = msg32[32 * (size_t)it + b];
        for (int b = 0; b < 64; b++) sig64[64 * (size_t)to + b] = sig64[64 * (size_t)it + b];
        item_base[m] = it = to;
    }
    const u8* s = p + 98;
    u32 slot = scid_hash(s) & mask, j;
    for (;;) {
        j = slots[slot];
        if (j == SV_SCID_EMPTY || scid_same(gossip_scid(blob + msg_off[j]), s)) break;
        slot = (slot + 1) & mask;
    }
    const u8* kp = nullptr;
    if (j != SV_SCID_EMPTY && j < m) {
        const u8* a = blob + msg_off[j];
        kp = gossip_scid(a) + 8 + 33 * (p[111] & 1);
    } else {
        j = SV_SCID_EMPTY;
        if (kinds[m] == 2) kp = signers33 + 33 * m;
    }
    cand[m] = j;
    for (int b = 0; b < 33; b++) key33[33 * (size_t)it + b] = kp ? kp[b] : 0;
}
// status[m] = 1 + index of the first failing signature (the reference's order), 0 if all verify
// -1 also when CLN's wire parser would refuse the message: a signature with r >= n or s >= n
// (fromwire_secp256k1_ecdsa_signature, wire/fromwire.c:188-199) or an undecodable bitcoin_key (fromwire_pubkey,
// bitcoin/pubkey.c:102-113).  node_ids are raw bytes on the wire (common/node_id.c:54) and only fail the signature.
__device__ __forceinline__ int gossip_items_status(u32 type, u32 base, const u8* verdict, const u8* aux) {
    int nitems = (type == 256) ? 4 : 1;
    int st = 0;
    for (int k = nitems - 1; k >= 0; k--)
        if (!verdict[base + k]) st = k + 1;
    for (int k = 0; k < nitems; k++) {
        u32 it = base + k;
        if (!(aux[it] & 2u)) st = -1;                           // r or s >= n: the wire parser refuses the message
        if (type == 256 && k >= 2 && !(aux[it] & 1u)) st = -1;  // undecodable bitcoin_key
    }
    return st;
}
// Burst mode (kinds != nullptr): a gated message (-3, -4) keeps its gate unless the parse refuses it (-1).  A
// channel_update resolved from the batch (cand[m], k_gossip_resolve) is settled from its candidate's own item verdicts:
// if the candidate verifies, the update's own verdict stands; if not, the update goes on the repair list ([count, m...])
// and keeps status 0 for the repair round (which runs this kernel again with repair == nullptr).  No candidate: -2, or
// for kind 2 (the source peer's private-update check, gossmap_manage.c:1099-1110) 5 if it verifies under the peer.
__global__ void __launch_bounds__(128) k_gossip_status(const u8* blob, const u64* msg_off, const u32* msg_len,
                                                       const u32* item_base, size_t n_msgs, const u8* verdict,
                                                       const u8* aux, int* status, const u8* kinds, const u32* cand,
                                                       u32* repair) {
    size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_msgs) return;
    const int st0 = status[m];
    if (st0 != 0 && !(kinds && (st0 == -3 || st0 == -4))) return;
    const u8* p = blob + msg_off[m];
    u32 type = ((u32)p[0] << 8) | p[1];
    int st = gossip_items_status(type, item_base[m], verdict, aux);
    if (kinds && st != -1) {
        if (st0 != 0) return;
        if (type == 258 && kinds[m] != 1) {
            u32 j = cand[m];
            if (j == SV_SCID_EMPTY) {
                st = (kinds[m] == 2 && st == 0) ? 5 : -2;
            } else if (repair && gossip_items_status(256, item_base[j], verdict, aux) != 0) {
                repair[1 + atomicAdd(repair, 1u)] = (u32)m;
                return;
            }
        }
    }
    status[m] = st;
}

// ---- gossip_store (gossip_store.cuh): record checksums and the channel each update is signed for ---------------------
// k_store_crc_flags: one thread per record the host walk listed (header offsets), slice-by-8 tables in shared memory;
// bad[r] = 1 if its checksum fails
__global__ void __launch_bounds__(256) k_store_crc_flags(const u8* store, const u64* rec_off, size_t n, u8* bad) {
    __shared__ u32 tab[2048];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) gs_crc_fill(tab, i);
    __syncthreads();
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) bad[r] = !gs_record_crc_ok(tab, store, rec_off[r]);
}
// one thread per channel event (announcement, delete_chan, update, listed by the host in store order): its scid as the
// sort key and its own index as the value; an event whose reads would pass the end of the store (store_len) gets ok = 0
__global__ void __launch_bounds__(256) k_store_events(const u8* store, u64 store_len, const u64* ev_off, const u8* ev_kind,
                                                      size_t n, u64* key, u32* val, u8* ok) {
    size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const u8* p = store + ev_off[e];
    const bool good = gs_event_ok(ev_kind[e], p, store_len - ev_off[e]);
    key[e] = good ? gs_event_scid(ev_kind[e], p) : ~0ull;
    val[e] = (u32)e;
    ok[e] = good;
}
// After the stable sort by scid every scid's events are one run in store order.  The thread at the head of a run walks
// it with gs_event.  holder[m] = what message m saw (an update: the announcement it is signed for; an announcement: the
// one that already held its channel, i.e. it is redundant), GS_NONE otherwise; an update's signer (the holder's
// node_id_1 or node_id_2 by channel_flags & 1, byte 111) goes to signers33[m].
__global__ void __launch_bounds__(128) k_store_resolve(const u8* store, const u64* key, const u32* val, const u8* ok,
                                                       const u8* ev_kind, const u64* ev_off, const u32* ev_msg, size_t n,
                                                       const u64* msg_off, u32* holder, u8* signers33) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (i > 0 && key[i - 1] == key[i])) return;
    u32 held = GS_NONE;
    for (size_t j = i; j < n && key[j] == key[i]; j++) {
        const u32 e = val[j];
        if (!ok[e]) continue;
        const int kind = ev_kind[e];
        const u32 h = gs_event(&held, kind, ev_msg[e]);
        if (kind == GS_EV_DEL) continue;
        const u32 m = ev_msg[e];
        holder[m] = h;
        if (kind == GS_EV_UPD && h != GS_NONE) {
            const u8* a = store + msg_off[h];
            const u8* kp = a + 260 + gs_be16(a + 258) + 32 + 8 + 33 * (store[ev_off[e] + 111] & 1);
            for (int b = 0; b < 33; b++) signers33[33 * (size_t)m + b] = kp[b];
        }
    }
}
// an update whose scid holds no channel at its position: -2, once the parse (-1) and the chain gate (-3) have passed
__global__ void __launch_bounds__(256) k_store_finish(const u8* store, const u64* msg_off, const u32* holder, size_t n,
                                                      int* status) {
    size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n) return;
    const u8* p = store + msg_off[m];
    if (p[0] == 1 && p[1] == 2 && holder[m] == GS_NONE && (status[m] == 0 || status[m] == 1)) status[m] = -2;
}

// ---- gossip_store salvage (gossip_salvage.cuh): every byte offset that holds a sound record -------------------------
// k_salvage_filter: one thread per byte offset o = 1 + global thread index, 256 per block.  Without out, count[b] = the
// candidates (gs_salvage_candidate) of block b.  With out, count holds each block's exclusive prefix (cub's scan) and
// every candidate goes to out[count[b] + its rank in the block]: the list is in store order.
__global__ void __launch_bounds__(256) k_salvage_filter(const u8* store, u64 len, u64* count, u64* out) {
    __shared__ u32 warp_n[8];
    const u64 o = 1 + (u64)blockIdx.x * 256 + threadIdx.x;
    const bool c = gs_salvage_candidate(store, len, o);
    const unsigned m = __ballot_sync(~0u, c);
    const u32 w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) warp_n[w] = __popc(m);
    __syncthreads();
    if (!out) {
        if (threadIdx.x == 0) {
            u64 n = 0;
            for (int k = 0; k < 8; k++) n += warp_n[k];
            count[blockIdx.x] = n;
        }
        return;
    }
    if (!c) return;
    u64 r = count[blockIdx.x] + __popc(m & ((1u << lane) - 1));
    for (u32 k = 0; k < w; k++) r += warp_n[k];
    out[r] = o;
}
// k_salvage_crc: sound[i] = 1 if candidate i's checksum matches.  One thread per candidate; a candidate whose message is
// longer than GS_SV_LONG (up to 65,535 bytes, mostly random offsets) is checksummed by its whole warp, one slice per
// lane (gs_crc_lane), so it costs the warp about what a short candidate costs one thread.
__global__ void __launch_bounds__(256) k_salvage_crc(const u8* store, const u64* cand, size_t n, u8* sound) {
    __shared__ u32 tab[2048];
    __shared__ u32 x2n[32];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) gs_crc_fill(tab, i);
    if (threadIdx.x == 0) gs_crc_x2n(x2n);
    __syncthreads();
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const u32 lane = threadIdx.x & 31;
    const u64 o = i < n ? cand[i] : 0;
    const u32 ml = i < n ? gs_be16(store + o + 2) : 0;
    const bool lng = ml > GS_SV_LONG;
    if (i < n && !lng) sound[i] = gs_record_crc_ok(tab, store, o);
    for (unsigned m = __ballot_sync(~0u, lng); m; m &= m - 1) {
        const u32 src = __ffs(m) - 1;
        const u64 oo = __shfl_sync(~0u, o, src);
        const u32 L = __shfl_sync(~0u, ml, src);
        const u8* h = store + oo;
        u32 r = gs_crc_lane(tab, x2n, h + GS_HDR, L, lane);
        for (int d = 16; d; d >>= 1) r ^= __shfl_xor_sync(~0u, r, d);
        if (lane == src) sound[i] = (gs_crc_shift(x2n, gs_be32(h + 8), L) ^ r) == gs_be32(h + 4);
    }
}
// k_salvage_restore: one warp per break [t, q) the host walk found: restore[b] = 1 if the damaged header's checksum, with
// its timestamp, covers exactly store[t + 12, q) (at most 65,535 bytes)
__global__ void __launch_bounds__(256) k_salvage_restore(const u8* store, const u64* brk, size_t n, u8* restore) {
    __shared__ u32 tab[2048];
    __shared__ u32 x2n[32];
    for (u32 i = threadIdx.x; i < 256; i += blockDim.x) gs_crc_fill(tab, i);
    if (threadIdx.x == 0) gs_crc_x2n(x2n);
    __syncthreads();
    const size_t b = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
    const u32 lane = threadIdx.x & 31;
    if (b >= n) return;  // whole warps
    const u64 t = brk[2 * b], q = brk[2 * b + 1];
    if (!gs_restore_fits(t, q)) {
        if (lane == 0) restore[b] = 0;
        return;
    }
    const u8* h = store + t;
    const u32 L = (u32)(q - t - GS_HDR);
    u32 r = gs_crc_lane(tab, x2n, h + GS_HDR, L, lane);
    for (int d = 16; d; d >>= 1) r ^= __shfl_xor_sync(~0u, r, d);
    if (lane == 0) restore[b] = (gs_crc_shift(x2n, gs_be32(h + 8), L) ^ r) == gs_be32(h + 4);
}

// ---- gossip_store prune (sv_prune_gossip_store_host): the deletions, a second channel table and the flag writes ------
// k_prune_mark: thread i < n_msgs turns message i's first-round status into its deletion (an announcement that is not 0,
// an update that is -1 or -3: SV_GP_MESSAGE), and with a funding verdict per message (fund, else NULL) an announcement
// gossipd would have refused for its txout (SV_GP_FUNDING); thread i < nev masks event i out of the second round if it
// is the announcement of a deleted message
__global__ void __launch_bounds__(256) k_prune_mark(const u8* store, const u64* msg_off, const int* status, size_t n_msgs,
                                                    const u8* ev_kind, const u32* ev_msg, const u8* ok, size_t nev,
                                                    const u8* fund, u8* reason, u8* ok2) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_msgs) {
        const u8* p = store + msg_off[i];
        const int st = status[i];
        const bool upd = p[0] == 1 && p[1] == 2;
        reason[i] = (upd ? (st == -1 || st == -3) : st != 0) ? SV_GP_MESSAGE
                    : (fund && gf_refused(fund[i]))           ? SV_GP_FUNDING
                                                               : SV_GP_KEPT;
    }
    if (i < nev)
        ok2[i] = ok[i] && !(ev_kind[i] == GS_EV_ANN && (status[ev_msg[i]] != 0 || (fund && gf_refused(fund[ev_msg[i]]))));
}
// k_prune_select: one thread per message not yet deleted, after the second k_store_resolve (holder2, signers2).  An
// announcement that is redundant now: SV_GP_REDUNDANT.  An update without a channel: SV_GP_NO_CHANNEL; with the same
// holder as in the first round, its first verdict stands (SV_GP_SIGNATURE if it failed); with another holder it joins
// the compact list (list[0] = count, warp-aggregated), its digest and signature copied from its first-round item slot
// and the new signer's key written, in item slot tail + its list position.
__global__ void __launch_bounds__(128) k_prune_select(const u8* store, const u64* msg_off, const int* status, size_t n_msgs,
                                                      const u32* holder, const u32* holder2, const u32* item_base,
                                                      const u8* signers2, u8* reason, u32* list, u32 tail, u8* msg32,
                                                      u8* key33, u8* sig64) {
    size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool moved = false;
    if (m < n_msgs && reason[m] == SV_GP_KEPT) {
        const u8* p = store + msg_off[m];
        if (p[0] == 1 && p[1] == 0) {
            if (holder2[m] != GS_NONE) reason[m] = SV_GP_REDUNDANT;
        } else if (p[0] == 1 && p[1] == 2) {
            if (holder2[m] == GS_NONE) reason[m] = SV_GP_NO_CHANNEL;
            else if (holder2[m] != holder[m]) moved = true;
            else if (status[m] != 0) reason[m] = SV_GP_SIGNATURE;
        }
    }
    const unsigned mask = __ballot_sync(0xFFFFFFFFu, moved);
    if (!mask) return;
    const int lane = threadIdx.x & 31, leader = __ffs(mask) - 1;
    u32 first = 0;
    if (lane == leader) first = atomicAdd(list, (u32)__popc(mask));
    first = __shfl_sync(0xFFFFFFFFu, first, leader);
    if (!moved) return;
    const u32 t = first + (u32)__popc(mask & ((1u << lane) - 1u));
    list[1 + t] = (u32)m;
    const size_t from = item_base[m], to = (size_t)tail + t;
    for (int b = 0; b < 32; b++) msg32[32 * to + b] = msg32[32 * from + b];
    for (int b = 0; b < 64; b++) sig64[64 * to + b] = sig64[64 * from + b];
    for (int b = 0; b < 33; b++) key33[33 * to + b] = signers2[33 * (size_t)m + b];
}
// the compact list's verdicts (item slots tail + t): an update that fails under its new signer is SV_GP_SIGNATURE
__global__ void __launch_bounds__(256) k_prune_settle(const u32* list, const u8* verdict, u8* reason) {
    u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < list[0] && !verdict[t]) reason[list[1 + t]] = SV_GP_SIGNATURE;
}
// one thread per deleted record: sets GOSSIP_STORE_DELETED_BIT (the high byte of the be16 flags) in the device copy of
// the store and returns that byte, the only one that changes
__global__ void __launch_bounds__(256) k_prune_flags(u8* store, const u64* rec_off, size_t n, u8* flag_hi) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u8 v = store[rec_off[i]] | (u8)(GS_DELETED >> 8);
    store[rec_off[i]] = v;
    flag_hi[i] = v;
}

// ---- gossip_store funding (gossip_funding.cuh): lightningd's funding outputs against the announcements ---------------
// fills idx[i] = i: the values the table's scids carry through the sort
__global__ void __launch_bounds__(256) k_funding_iota(u32* idx, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) idx[i] = (u32)i;
}
// *dup = 1 if two neighbours of the sorted scids are equal
__global__ void __launch_bounds__(256) k_funding_dups(const u64* scid, size_t n, u32* dup) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > 0 && i < n && scid[i] == scid[i - 1]) *dup = 1;
}
// one thread per candidate announcement (message index cand[i]): fund[cand[i]] = its verdict (gf_verdict)
__global__ void __launch_bounds__(128) k_store_funding(const u8* store, u64 len, const u64* msg_off, const u32* cand, size_t n,
                                                       gf_table t, u8* fund) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 m = cand[i];
    fund[m] = (u8)gf_verdict(store, len, msg_off[m] - GS_HDR, t);
}

// ---- BOLT12 signatures (bolt12.cuh): the message hash of bolt12_check_signature on the device -----------------------
// k_b12_count: one thread per stream walks its BigSize headers (bytes only): field count, or 0 if the parse fails
__global__ void __launch_bounds__(128) k_b12_count(const u8* blob, const u64* off, const u32* len, size_t n, u32* cnt) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    long long c = b12_count(blob + off[i], len[i]);
    cnt[i] = c < 0 ? 0u : (u32)c;
}
// k_b12_tags: thread t < ntags computes the sighash midstate of tag t (tag bytes tagbytes[tagoff[t] .. +taglen[t])), thread
// ntags the leaf and branch midstates every tag shares
__global__ void k_b12_tags(const u8* tagbytes, const u64* tagoff, const u32* taglen, size_t ntags, b12_tags* tags,
                           u32* sigmid) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < ntags) b12_tag_mid(sigmid + 8 * t, tagbytes + tagoff[t], taglen[t], tagbytes, 0);
    else if (t == ntags) b12_make_tree_tags(tags);
}
// k_b12_merkle: one warp per stream.  Lane 0 walks the headers into the field records; the lanes hash one field each
// (leaf, nonce, leaf pair; strided past 32 fields); signature-range fields drop out by ballot / popc compaction; then the
// tree is reduced one level per step (neighbours paired, an odd last node carried up: merkle_tlv's power-of-two split);
// lane 0 hashes the root into the sighash under the stream's tag (sigmid[tag_of[i]]; tag_of NULL: tag 0).  Failed parses
// get a zero sighash (they are never verified as signed).
#define SV_B12_WARPS 4
__global__ void __launch_bounds__(32 * SV_B12_WARPS) k_b12_merkle(const u8* blob, const u64* off, const u32* len, size_t n,
                                                                  const u32* cnt, const u64* fbase, const b12_tags* tags,
                                                                  const u32* sigmid, const u32* tag_of,
                                                                  b12_field* recs, u32* nodes, u8* msg32) {
    const size_t i = (size_t)blockIdx.x * SV_B12_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;  // whole warps leave together
    const u32 F = cnt[i];
    if (F == 0) {
        msg32[32 * i + lane] = 0;
        return;
    }
    const u8* p = blob + off[i];
    const u32 L = len[i];
    b12_field* rec = recs + fbase[i];
    u32* node = nodes + 8 * fbase[i];
    __shared__ b12_tags s_tags[SV_B12_WARPS];  // one copy per warp: warps leave early, so no CTA-wide barrier
    u32 nm[8];
    if (lane == 0) {
        u32 pos = 0;
        u64 prev = 0;
        for (u32 j = 0; j < F; j++) {
            b12_field f;
            b12_next(p, L, &pos, j == 0, prev, &f);  // cannot fail: k_b12_count walked the same bytes
            prev = f.type;
            rec[j] = f;
        }
        b12_nonce_mid(nm, p + rec[0].off, rec[0].len);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) nm[k] = __shfl_sync(0xFFFFFFFFu, nm[k], 0);
    b12_tags& t = s_tags[threadIdx.x >> 5];
    if (lane < 16) reinterpret_cast<u32*>(&t)[lane] = reinterpret_cast<const u32*>(tags)[lane];  // leaf, branch
    __syncwarp();
    u32 m = 0;  // non-signature fields so far
    for (u32 j0 = 0; j0 < F; j0 += 32) {
        const u32 j = j0 + lane;
        b12_field f;
        bool leaf = false;
        if (j < F) {
            f = rec[j];
            leaf = !b12_is_signature(f.type);
        }
        u32 h[8];
        if (leaf) b12_leaf_pair(h, &t, nm, p, f);
        const unsigned b = __ballot_sync(0xFFFFFFFFu, leaf);
        if (leaf) {
            u32* d = node + 8 * (m + __popc(b & ((1u << lane) - 1u)));
#pragma unroll
            for (int k = 0; k < 8; k++) d[k] = h[k];
        }
        m += __popc(b);
    }
    __syncwarp();
    while (m > 1) {
        const u32 up = (m + 1) / 2;
        for (u32 k0 = 0; k0 < up; k0 += 32) {
            const u32 k = k0 + lane;
            u32 h[8];
            if (2 * k + 1 < m) b12_branch(h, t.branch, node + 16 * k, node + 16 * k + 8);
            else if (k < up) {
#pragma unroll
                for (int q = 0; q < 8; q++) h[q] = node[16 * k + q];
            }
            __syncwarp();  // every lane has read its pair before any lane of this round overwrites a slot
            if (k < up) {
#pragma unroll
                for (int q = 0; q < 8; q++) node[8 * k + q] = h[q];
            }
            __syncwarp();
        }
        m = up;
    }
    if (lane == 0) {
        u32 root[8];
#pragma unroll
        for (int q = 0; q < 8; q++) root[q] = m ? node[q] : 0u;  // no non-signature field: merkle_tlv's all-zero root
        b12_sighash_mid(msg32 + 32 * i, sigmid + 8 * (size_t)(tag_of ? tag_of[i] : 0u), root);
    }
}
// status[i] = verdict where the stream parsed, -1 where it did not
__global__ void __launch_bounds__(256) k_b12_status(const u32* cnt, const u8* verdict, size_t n, int* status) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) status[i] = cnt[i] ? (int)verdict[i] : -1;
}

// ---- BOLT11 invoices (bolt11.cuh): bolt11_decode's signature step ----------------------------------------------------
// k_b11_parse: one thread per invoice: bech32, the field walk, the `n` key, the signature bytes and the signing hash.
// is_n / is_r flag the invoices verified against their `n` key and the ones whose key is recovered (0 / 0: status -1).
__global__ void __launch_bounds__(128) k_b11_parse(const u8* blob, const u64* off, const u32* len, size_t n, u8* msg32,
                                                   u8* key33, u8* sig64, u8* recid, u32* is_n, u32* is_r) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u8* s = blob + off[i];
    b11_str b;
    b11_parsed p;
    const bool ok = b11_parse(s, len[i], &b, &p);
    if (ok) {
        b11_sighash(msg32 + 32 * i, s, b);
        for (int k = 0; k < 64; k++) sig64[64 * i + k] = p.sig[k];
        for (int k = 0; k < 33; k++) key33[33 * i + k] = p.key33[k];
        recid[i] = p.recid;
    } else {
        for (int k = 0; k < 32; k++) msg32[32 * i + k] = 0;
    }
    is_n[i] = ok && p.have_n;
    is_r[i] = ok && !p.have_n;
}
// the `n` invoices, packed (base_n: exclusive prefix sum of is_n) for the ordinary compressed-key ECDSA path
__global__ void __launch_bounds__(128) k_b11_gather_n(const u32* is_n, const u64* base_n, size_t n, const u8* msg32,
                                                      const u8* key33, const u8* sig64, u8* cmsg, u8* ckey, u8* csig) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !is_n[i]) return;
    const size_t j = base_n[i];
    for (int k = 0; k < 32; k++) cmsg[32 * j + k] = msg32[32 * i + k];
    for (int k = 0; k < 33; k++) ckey[33 * j + k] = key33[33 * i + k];
    for (int k = 0; k < 64; k++) csig[64 * j + k] = sig64[64 * i + k];
}
// the recovered invoices, packed: R's x (the ladder's x-only key) and the work record of u1 = -e / r, u2 = +-s / r
__global__ void __launch_bounds__(128) k_b11_rec_prep(const u32* is_r, const u64* base_r, size_t n, const u8* msg32,
                                                      const u8* sig64, const u8* recid, u8* x32, sv_work* work) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !is_r[i]) return;
    const size_t j = base_r[i];
    sv_work w;
    b11_recover_prep(w, x32 + 32 * j, sig64 + 64 * i, recid[i], msg32 + 32 * i);
    work[j] = w;
}
// Q = u1 G + u2 E as k_main<SV_KIND_SCHNORR> parked it: affine, checked, compressed (SV_FINAL_BATCH per thread)
__global__ void __launch_bounds__(64) k_b11_rec_final(const sv_work* work, size_t n, int* rstat, u8* rkey33) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t base = t * SV_FINAL_BATCH;
    if (base >= n) return;
    int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
    b11_recover_final_batch(rstat + base, rkey33 + 33 * base, reinterpret_cast<const sv_jac*>(work) + base, cnt);
}
// status and receiver_id of every invoice, from whichever path it took
__global__ void __launch_bounds__(256) k_b11_status(const u32* is_n, const u64* base_n, const u32* is_r, const u64* base_r,
                                                    size_t n, const u8* recid, const u8* key33, const u8* verdict_n,
                                                    const int* rstat, const u8* rkey33, int* status, u8* node33) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int st = -1;
    const u8* key = nullptr;
    if (is_n[i]) {
        st = (recid[i] <= 3 && verdict_n[base_n[i]]) ? 1 : 0;  // recid > 3 is refused before secp256k1_ecdsa_verify
        key = key33 + 33 * i;
    } else if (is_r[i]) {
        st = rstat[base_r[i]];
        key = rkey33 + 33 * base_r[i];
    }
    status[i] = st;
    for (int k = 0; k < 33; k++) node33[33 * i + k] = st == 1 ? key[k] : 0;
}

static_assert(sizeof(sv_jac) == sizeof(sv_work), "R is parked in place of the work record");
__global__ void __launch_bounds__(64) k_final_schnorr(const sv_work* work, const u8* sig, size_t n, u8* verdict) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t base = t * SV_FINAL_BATCH;
    if (base >= n) return;
    int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
    schnorr_final_batch(verdict + base, reinterpret_cast<const sv_jac*>(work) + base, sig + 64 * base, cnt);
}

static_assert(sizeof(sv_ns_park) == sizeof(sv_work), "D, B, c are parked in place of the work record");
__global__ void __launch_bounds__(64) k_final_ecdsa33(const sv_work* work, const u8* key33, const u8* sig, size_t n,
                                                       const ge_mem* gtab, u8* verdict, u8* aux) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t base = t * SV_FINAL_BATCH;
    if (base >= n) return;
    int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
    ecdsa33_nosqrt_final_batch(verdict + base, work + base, key33 + 33 * base, sig + 64 * base, gtab, cnt, aux ? aux + base : nullptr);
}

static_assert(sizeof(sv_ns_park_schnorr) == sizeof(sv_work), "D, B, N, CG are parked in place of the work record");
__global__ void __launch_bounds__(64) k_final_schnorr_ns(const sv_work* work, const u8* xonly32, const u8* sig, size_t n,
                                                          const ge_mem* gtab, u8* verdict) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t base = t * SV_FINAL_BATCH;
    if (base >= n) return;
    int cnt = (int)((n - base < SV_FINAL_BATCH) ? (n - base) : SV_FINAL_BATCH);
    schnorr_nosqrt_final_batch(verdict + base, work + base, xonly32 + 32 * base, sig + 64 * base, gtab, cnt);
}

__global__ void k_pack_bitmap(const u8* verdict, size_t n, u32* bitmap) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    u32 v = (i < n) ? (verdict[i] != 0) : 0u;
    u32 b = __ballot_sync(0xFFFFFFFFu, v);
    if ((threadIdx.x & 31) == 0 && i < n) bitmap[i >> 5] = b;
}

__global__ void __launch_bounds__(128) k_pubkey_parse(const u8* key33, size_t n, u8* xy64, u8* okout) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ge Q;
    bool ok = key_decode(Q, SV_KIND_ECDSA33, key33 + 33 * i);
    if (ok) {
        fe_get_b32(xy64 + 64 * i, Q.x);
        fe_get_b32(xy64 + 64 * i + 32, Q.y);
    } else {
        for (int k = 0; k < 64; k++) xy64[64 * i + k] = 0;
    }
    okout[i] = ok;
}

// ---- device-side self test of the arithmetic primitives (test support; body in selftest.cuh) -------
__global__ void __launch_bounds__(128) k_selftest(int op, const u32* __restrict__ a, const u32* __restrict__ b, size_t n,
                                                  u32* __restrict__ out, const ge_mem* __restrict__ gtab) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 A[8], B[8], R[16];
#pragma unroll
    for (int k = 0; k < 8; k++) { A[k] = a[8 * i + k]; B[k] = b[8 * i + k]; }
    selftest_item(op, A, B, R, gtab);
#pragma unroll
    for (int k = 0; k < 16; k++) out[16 * i + k] = R[k];
}
// ---- device-side self test of the group law and the multiplication schedules (test support; body in selftest.cuh) ---
__global__ void __launch_bounds__(128) k_selftest_group(int op, const u32* __restrict__ in, size_t n, u32* __restrict__ out,
                                                        const ge_mem* __restrict__ gtab) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    selftest_group_item(op, in + SV_STG_IN_WORDS * i, out + SV_STG_OUT_WORDS * i, gtab);
}

// ---- synthetic workload generator ---------------------------------------------------------------
SV_D void synth_hash(u8 out[32], u64 seed, u64 idx, u32 tag) {
    u8 buf[20];
    for (int k = 0; k < 8; k++) { buf[k] = (u8)(seed >> (8 * k)); buf[8 + k] = (u8)(idx >> (8 * k)); }
    for (int k = 0; k < 4; k++) buf[16 + k] = (u8)(tag >> (8 * k));
    u32 st[8];
    sha256_bytes(st, buf, 20);
    for (int k = 0; k < 8; k++) {
        out[4 * k] = (u8)(st[k] >> 24); out[4 * k + 1] = (u8)(st[k] >> 16);
        out[4 * k + 2] = (u8)(st[k] >> 8); out[4 * k + 3] = (u8)st[k];
    }
}
template <int KIND>
__global__ void __launch_bounds__(128) k_synth(u64 seed, size_t n, const ge_mem* gtab, u8* msg, u8* key, u8* sig) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u8 h[32];
    sc d, k, m, one;
#pragma unroll
    for (int q = 0; q < 8; q++) one.v[q] = (q == 0);
    synth_hash(h, seed, i, 1);
    sc_set_b32(d, h, nullptr);
    if (sc_is_zero(d)) d = one;
    synth_hash(h, seed, i, 2);
    sc_set_b32(k, h, nullptr);
    if (sc_is_zero(k)) k = one;
    synth_hash(h, seed, i, 3);
    for (int q = 0; q < 32; q++) msg[32 * i + q] = h[q];
    sc_set_b32(m, h, nullptr);
    ge P, R;
    ecmult_gen_comb(P, d, gtab);
    ecmult_gen_comb(R, k, gtab);
    if (KIND == SV_KIND_SCHNORR) {
        // BIP-340 signing equation with even-y P and R: s = k + e*d
        if (fe_is_odd(P.y)) sc_negate(d, d);
        if (fe_is_odd(R.y)) sc_negate(k, k);
        u8 rx[32], px[32], e32[32];
        fe_get_b32(rx, R.x);
        fe_get_b32(px, P.x);
        sha256_bip340_challenge(e32, rx, px, h);
        sc e, s;
        sc_set_b32(e, e32, nullptr);
        sc_mul(s, e, d);
        sc_add(s, s, k);
        for (int q = 0; q < 32; q++) { key[32 * i + q] = px[q]; sig[64 * i + q] = rx[q]; }
        sc_get_b32(sig + 64 * i + 32, s);
    } else {
        // ECDSA: r = x(kG) mod n, s = (m + r d)/k, normalised to low S
        u8 rx[32];
        fe_get_b32(rx, R.x);
        sc r, s, kinv;
        sc_set_b32(r, rx, nullptr);
        sc_inverse(kinv, k);
        sc_mul(s, r, d);
        sc_add(s, s, m);
        sc_mul(s, s, kinv);
        if (sc_is_high(s)) sc_negate(s, s);
        sc_get_b32(sig + 64 * i, r);
        sc_get_b32(sig + 64 * i + 32, s);
        if (KIND == SV_KIND_ECDSA33) {
            key[33 * i] = fe_is_odd(P.y) ? 3 : 2;
            fe_get_b32(key + 33 * i + 1, P.x);
        } else {
            fe_get_b32(key + 64 * i, P.x);
            fe_get_b32(key + 64 * i + 32, P.y);
        }
    }
}

// ---- integer-pipe probes ------------------------------------------------------------------------
// Each probe is its own kernel so that ncu reports them separately.  All run 256 threads x 8 CTAs/SM.
//   0 k_probe_imad_wide   independent IMAD.WIDE.U32 accumulations (no carries)      -> MAC/s (roofline peak)
//   1 k_probe_cmad4       4-deep IMAD.WIDE.U32(.X) carry chains as u256_mul_wide issues them -> MAC/s
//   2 k_probe_fe_mul      field multiplications/s          3 k_probe_fe_sqr   field squarings/s
//   4 k_probe_chain8      8-deep IMAD.WIDE.U32.X chains    -> MAC/s
//   5 k_probe_carry_save  IMAD.WIDE.U32 with carry-OUT only + one IADD3.X per product -> MAC/s
//   6 k_probe_imad32      separate 32-bit IMAD (lo) / IMAD.HI  -> instr/s
//   7 k_probe_addc        8-long IADD3(.X) carry chains -> adds/s
//   8 k_probe_dfma        independent FP64 FMA chains -> DFMA/s (the idle FP64 pipe; round-2 idea: DFMA-based products)
#define PROBE_PROLOGUE u32 t = blockIdx.x * blockDim.x + threadIdx.x
__global__ void __launch_bounds__(256) k_probe_imad_wide(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 lo[8], hi[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { lo[k] = t * 2654435761u + k; hi[k] = t ^ (k * 0x9E3779B9u); }
    u32 y = t | 3u;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            // acc_k += lo(acc_{k+1}) * y : eight independent 64-bit multiply-accumulates per step whose
            // multiplicands change every step (so ptxas cannot strength-reduce them to additions)
#pragma unroll
            for (int k = 0; k < 8; k++)
                asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.u32 %1, %2, %3, %1;"
                             : "+r"(lo[k]), "+r"(hi[k])
                             : "r"(lo[(k + 1) & 7]), "r"(y));
        }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= lo[k] ^ hi[k];
    if (s == 0x1234567u) sink[0] = s;
}
__global__ void __launch_bounds__(256) k_probe_cmad4(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 E[8], O[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { E[k] = t + k; O[k] = t * 3 + k; }
    u32 a0 = t | 1, a1 = t ^ 0xABCDEFu, a2 = t * 7 + 1, a3 = ~t, b = t * 2654435761u;
    u32 cs = 0;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            cs += sv_cmad4(E, a0, a1, a2, a3, b);
            cs += sv_cmad4(O, a1, a2, a3, a0, b);
        }
    }
    u32 s = cs;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= E[k] ^ O[k];
    if (s == 0x12345u) sink[0] = s;
}
template <int SQR>
__global__ void __launch_bounds__(256) k_probe_fe(int iters, u32* sink) {
    PROBE_PROLOGUE;
    fe a, b;
#pragma unroll
    for (int k = 0; k < 8; k++) { a.v[k] = t * 2654435761u + k; b.v[k] = (t ^ 0x5bd1e995u) * (k + 3); }
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
        if (!SQR) { fe_mul(a, a, b); fe_mul(b, b, a); }
        else { fe_sqr(a, a); fe_sqr(b, b); }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= a.v[k] ^ b.v[k];
    if (s == 0x12345u) sink[0] = s;
}
__global__ void __launch_bounds__(256) k_probe_chain8(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 A[16], B[16];
#pragma unroll
    for (int k = 0; k < 16; k++) { A[k] = t + k; B[k] = t * 5 + k; }
    u32 x0 = t | 1, x1 = t ^ 0xABCDEFu, x2 = t * 7 + 1, x3 = ~t, y = t * 2654435761u;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int k = 0; k < 2; k++) {
#define CHAIN8(ACC)                                                                                              \
    asm volatile("mad.lo.cc.u32 %0, %16, %20, %0;\n\tmadc.hi.cc.u32 %1, %16, %20, %1;\n\t"                         \
                 "madc.lo.cc.u32 %2, %17, %20, %2;\n\tmadc.hi.cc.u32 %3, %17, %20, %3;\n\t"                        \
                 "madc.lo.cc.u32 %4, %18, %20, %4;\n\tmadc.hi.cc.u32 %5, %18, %20, %5;\n\t"                        \
                 "madc.lo.cc.u32 %6, %19, %20, %6;\n\tmadc.hi.cc.u32 %7, %19, %20, %7;\n\t"                        \
                 "madc.lo.cc.u32 %8, %17, %20, %8;\n\tmadc.hi.cc.u32 %9, %17, %20, %9;\n\t"                        \
                 "madc.lo.cc.u32 %10, %18, %20, %10;\n\tmadc.hi.cc.u32 %11, %18, %20, %11;\n\t"                    \
                 "madc.lo.cc.u32 %12, %19, %20, %12;\n\tmadc.hi.cc.u32 %13, %19, %20, %13;\n\t"                    \
                 "madc.lo.cc.u32 %14, %16, %20, %14;\n\tmadc.hi.u32 %15, %16, %20, %15;"                           \
                 : "+r"(ACC[0]), "+r"(ACC[1]), "+r"(ACC[2]), "+r"(ACC[3]), "+r"(ACC[4]), "+r"(ACC[5]), "+r"(ACC[6]), \
                   "+r"(ACC[7]), "+r"(ACC[8]), "+r"(ACC[9]), "+r"(ACC[10]), "+r"(ACC[11]), "+r"(ACC[12]),           \
                   "+r"(ACC[13]), "+r"(ACC[14]), "+r"(ACC[15])                                                      \
                 : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(y))
            CHAIN8(A);
            CHAIN8(B);
        }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 16; k++) s ^= A[k] ^ B[k];
    if (s == 0x12345u) sink[0] = s;
}
__global__ void __launch_bounds__(256) k_probe_carry_save(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 lo[8], hi[8], c[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { lo[k] = t + k; hi[k] = t * 3 + k; c[k] = k; }
    u32 x = t * 2654435761u + 12345u, y = t ^ 0x9E3779B9u;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int k = 0; k < 8; k++)
                asm volatile("mad.lo.cc.u32 %0, %3, %4, %0;\n\tmadc.hi.cc.u32 %1, %3, %4, %1;\n\taddc.u32 %2, %2, 0;"
                             : "+r"(lo[k]), "+r"(hi[k]), "+r"(c[k])
                             : "r"(x), "r"(y));
        }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= lo[k] ^ hi[k] ^ c[k];
    if (s == 0x12345u) sink[0] = s;
}
__global__ void __launch_bounds__(256) k_probe_imad32(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 a[8];
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = t + k;
    u32 x = t * 2654435761u + 12345u, y = t ^ 0x9E3779B9u, z = t * 31 + 7;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int k = 0; k < 8; k += 2)
                asm volatile("mad.lo.u32 %0, %2, %3, %0;\n\tmad.hi.u32 %1, %2, %4, %1;"
                             : "+r"(a[k]), "+r"(a[k + 1])
                             : "r"(x), "r"(y), "r"(z));
        }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= a[k];
    if (s == 0x12345u) sink[0] = s;
}
__global__ void __launch_bounds__(256) k_probe_dfma(int iters, u32* sink) {
    PROBE_PROLOGUE;
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = 1.0 + (double)(t + k) * 1e-9;
    double x = 1.0000001 + (double)t * 1e-12, y = 0.9999999;
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int k = 0; k < 8; k++) a[k] = fma(a[k], x, y);
        }
    }
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s += a[k];
    if (s == 1234.5) sink[0] = 1;
}
__global__ void __launch_bounds__(256) k_probe_addc(int iters, u32* sink) {
    PROBE_PROLOGUE;
    u32 a[8], b[8], c[8], d[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { a[k] = t + k; b[k] = t * 3 + k; c[k] = t ^ k; d[k] = ~t + k; }
#pragma unroll 1
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int r = 0; r < 2; r++) {
            u256_add(a, a, b);
            u256_add(c, c, d);
            u256_add(b, b, c);
            u256_add(d, d, a);
        }
    }
    u32 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= a[k] ^ b[k] ^ c[k] ^ d[k];
    if (s == 0x12345u) sink[0] = s;
}

// -------------------------------------------------------------------------------------------------
// context
// -------------------------------------------------------------------------------------------------
#define SV_NSLOTS 2
#define SV_SMALL_CAP 8192           // items the pinned small-batch staging block holds
#ifndef SV_SMALL_MAX_DEFAULT
// largest batch sent down the small-batch path (SV_SMALL_MAX overrides; 0 disables); tools/latency_table.py times both
// paths at the sizes around it
#define SV_SMALL_MAX_DEFAULT 8192
#endif
// smallest sizes of the grow-only context buffers (dev_buf::reserve)
#define SV_ITEMS_FLOOR ((size_t)4096)        // staging, span arrays and launch-slot records, in items
#define SV_GBUF_FLOOR ((size_t)1 << 16)      // g_buf and d_data, in bytes
#define SV_SCRATCH_FLOOR ((size_t)1 << 20)   // dd_buf, sk_buf and b12_buf, in bytes
struct sv_queue_item {
    int kind;
    u8 msg[32];
    u8 key[64];
    u8 sig[64];
};

struct sv_ctx;

// A device allocation owned by the context or by one call, freed when its owner goes.  It converts to its pointer, so it
// is used like one.  reserve() is the one place a buffer grows: see its definition below.
template <typename T = u8>
struct dev_buf {
    T* p = nullptr;
    size_t cap = 0;  // bytes
    dev_buf() = default;
    dev_buf(const dev_buf&) = delete;
    dev_buf& operator=(const dev_buf&) = delete;
    ~dev_buf() { if (p) cudaFree(p); }
    operator T*() const { return p; }
    template <typename U> U* at(size_t off) const { return reinterpret_cast<U*>(reinterpret_cast<u8*>(p) + off); }  // a slab piece
    int reserve(sv_ctx* ctx, size_t bytes, size_t floor, cudaEvent_t wait = nullptr);
};

// Offsets of the pieces of one scratch slab, in the order they are taken; size is the slab's length so far.
struct slab_layout {
    size_t size = 0;
    size_t take(size_t bytes, size_t align = 16) {
        const size_t at = (size + align - 1) / align * align;
        size = at + bytes;
        return at;
    }
};

// The marks of the profiling mode, one timing event each.  Every verification launch records MK_PREP, MK_MAIN and MK_END
// (sv_get_last_timing reads them).  A synchronous entry point records its stage marks as well and turns its marks into
// its splits before it returns.  Calls on one context are issued one at a time, so the entry points share stage slots.
enum sv_mark {
    MK_PREP, MK_MAIN, MK_END,
    // BOLT12, BOLT11
    MK_B12_PARSE = 3, MK_B12_SIGHASH,
    MK_B11_PARSE = 3, MK_B11_PACKED, MK_B11_CURVE, MK_B11_DONE,
    // the gossip_store audit and prune, and their funding step
    MK_STORE_COPY = 3, MK_STORE_COPIED, MK_STORE_CRC, MK_STORE_PASS, MK_PRUNE_ROUND2, MK_PRUNE_FLAGS,
    MK_FUND_STAGE, MK_FUND_STAGED, MK_FUND_KERNEL, MK_FUND_DONE,
    // the salvage
    MK_SALVAGE_COUNT = 3, MK_SALVAGE_SCANNED, MK_SALVAGE_EMIT, MK_SALVAGE_CRC, MK_SALVAGE_DONE,
    MK_COUNT = MK_FUND_DONE + 1
};

struct sv_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;      // second compute stream: consecutive slices of a large host batch alternate
                                         // streams, so the thin last wave of one slice's curve kernel overlaps the next
                                         // slice's kernels
    cudaStream_t copy_stream = nullptr;  // H2D of the next slice overlaps the kernels of the current one (sv_verify_host)
    cudaEvent_t h2d_ev[8] = {};
    ge_mem* d_gtab = nullptr;
    dev_buf<> d_hot;    // [slot 0 table slab | G comb table | slot 1 table slab]
    size_t l2_persist = 0, l2_max_persist = 0, hot_slab = 0, hot_gt = 0;
    cudaStream_t policy_streams[4] = {};  // (stream, slab) pairs whose access-policy window is already set
    const void* policy_slabs[4] = {};
    int l2_policy = 1;  // sv_set_l2_policy (default on)
    dev_buf<ge_mem> d_bases;
    size_t scratch_bytes = 0;
    int main_grid = 0;
    // Launch slots: the scalar-side work records and the per-thread Q-table slab of one prep+main launch pair.  Two slots,
    // used round-robin, let launches issued on DIFFERENT streams overlap (the partially filled last wave of one batch's
    // curve kernel runs beside the next batch's kernels); a slot is re-used only after the event recorded behind its
    // previous use, so calls on one context can never corrupt each other whatever streams the caller picks.
    struct slot_t {
        dev_buf<sv_work> d_work;
        qtab_entry* d_scratch = nullptr;
        cudaEvent_t done = nullptr;
        cudaStream_t last_stream = nullptr;
        int used = 0;
    } slot[SV_NSLOTS];
    unsigned next_slot = 0;
    // small-batch path: calls of up to small_max signatures run as ONE launch of k_small reading their inputs straight
    // from this pinned, device-mapped staging block (no H2D/D2H copy commands, no allocation)
    size_t small_max = SV_SMALL_MAX_DEFAULT, small_cap = SV_SMALL_CAP;
    u8* h_small = nullptr;
    // key de-duplication scratch (hash table + index lists; also the BIP-340 batch scratch) and the table array of the
    // distinct keys
    dev_buf<> dd_buf, sk_buf;
    int dedup = 1;   // gossip batches: look for repeated keys (sv_set_dedup; default on)
    int nosqrt = 1;  // compressed-key ECDSA through the flow without the square root (default on; env SV_NOSQRT=0: measurement aid)
    u32 last_distinct = 0;
    u32 last_repair = 0;  // updates the last gossip burst re-resolved in its repair round
    // device staging for the host-buffer entry points (ensure_staging)
    dev_buf<> d_msg, d_key, d_sig, d_verdict;
    // raw-span staging
    dev_buf<> d_data;
    dev_buf<u64> d_off;
    dev_buf<u32> d_len;
    dev_buf<u32> d_sink;
    // per-call scratch of the gossip, transaction, mixed, BOLT12 and fee-grind entry points (ensure_gbuf)
    dev_buf<> g_buf;
    // BOLT12 field records and tree nodes, sized by the counting pass
    dev_buf<> b12_buf;
    int profiling = 0;
    cudaEvent_t mark_ev[MK_COUNT] = {};  // one timing event per mark (sv_set_profiling)
    float b12_ms[2] = {};        // last sv_verify_bolt12_host: parse / Merkle / sighash kernels, verification kernels
    float b11_ms[2] = {};        // last sv_verify_bolt11_host: parse stage, curve stage
    float gs_ms[4] = {};         // last sv_verify_gossip_store_host: header walk, H2D, checksums, verification (profiling mode)
    float gp_ms[4] = {};         // last sv_prune_gossip_store_host: header walk, first round, second round, flag write
    float gf_ms[2] = {};         // last funding call: table staging and sort, k_store_funding
    float gv_ms[3] = {};         // last sv_salvage_gossip_store_host: filter, checksums, host walk
    unsigned long long launches = 0;
    std::vector<sv_queue_item> queue;
    std::string err;
};

static std::string g_create_err;

// every entry point runs on the context's device and puts the caller's current device back on return
struct dev_guard {
    int prev = -1;
    cudaError_t enter(int dev) {
        cudaError_t e = cudaGetDevice(&prev);
        if (e != cudaSuccess) { prev = -1; return e; }
        if (prev == dev) { prev = -1; return cudaSuccess; }
        return cudaSetDevice(dev);
    }
    ~dev_guard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int fail(sv_ctx* ctx, int code, const char* what, cudaError_t e) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s", what, e == cudaSuccess ? "" : cudaGetErrorString(e));
    if (ctx) ctx->err = buf; else g_create_err = buf;
    return code;
}
#define CK(call)                                                                   \
    do {                                                                           \
        cudaError_t e__ = (call);                                                  \
        if (e__ != cudaSuccess) return fail(ctx, e__ == cudaErrorMemoryAllocation ? SV_ERR_NOMEM : SV_ERR_CUDA, #call, e__); \
    } while (0)

// profiling mode: mark k recorded on st (nothing otherwise), and the milliseconds from mark a to mark b
static cudaError_t mark(const sv_ctx* ctx, sv_mark k, cudaStream_t st) {
    return ctx->profiling ? cudaEventRecord(ctx->mark_ev[k], st) : cudaSuccess;
}
static cudaError_t mark_ms(const sv_ctx* ctx, sv_mark a, sv_mark b, float* ms) {
    return cudaEventElapsedTime(ms, ctx->mark_ev[a], ctx->mark_ev[b]);
}

// Grow-only: nothing happens while the buffer holds `bytes`.  Otherwise it waits until no launch can still read the old
// allocation (the whole device, or only the event `wait` when the caller knows the last user), frees it and allocates the
// smallest power-of-two multiple of `floor` that holds `bytes`; a failure leaves the buffer empty.  floor == bytes is an
// exact fit, for the fixed allocations and the per-call ones.  A successful reserve always leaves an allocation, even for
// 0 bytes (floor 0 counts as 1), so the pointer handed to a copy or a kernel is never null.
template <typename T>
int dev_buf<T>::reserve(sv_ctx* ctx, size_t bytes, size_t floor, cudaEvent_t wait) {
    if (p && bytes <= cap) return SV_OK;
    if (bytes > ((size_t)-1) / 2) return fail(ctx, SV_ERR_NOMEM, "device buffer size", cudaSuccess);
    if (p) {
        CK(wait ? cudaEventSynchronize(wait) : cudaDeviceSynchronize());
        cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    size_t want = floor ? floor : 1;
    while (want < bytes) want *= 2;
    T* q = nullptr;
    CK(cudaMalloc(&q, want));
    p = q;
    cap = want;
    return SV_OK;
}

extern "C" size_t sv_key_size(int kind) {
    return kind == SV_KIND_ECDSA33 ? 33 : kind == SV_KIND_ECDSA_XY ? 64 : kind == SV_KIND_SCHNORR ? 32 : 0;
}
extern "C" const char* sv_last_error(const sv_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

// Pick the next launch slot for n work records on stream st: waits (on the device, not the host) for the slot's previous
// user if that ran on another stream, grows the record array geometrically when needed (the only host-synchronising case).
static int acquire_slot(sv_ctx* ctx, size_t n, cudaStream_t st, sv_ctx::slot_t** out) {
    sv_ctx::slot_t* sl = &ctx->slot[ctx->next_slot++ % SV_NSLOTS];
    if (sl->used && sl->last_stream != st) CK(cudaStreamWaitEvent(st, sl->done, 0));
    // only this slot's previous launch reads its records: the other slot's launch may go on running meanwhile
    int rc = sl->d_work.reserve(ctx, n * sizeof(sv_work), SV_ITEMS_FLOOR * sizeof(sv_work), sl->done);
    if (rc) return rc;
    *out = sl;
    return SV_OK;
}
static int release_slot(sv_ctx* ctx, sv_ctx::slot_t* sl, cudaStream_t st) {
    CK(cudaEventRecord(sl->done, st));
    sl->last_stream = st;
    sl->used = 1;
    return SV_OK;
}
static int ensure_staging(sv_ctx* ctx, size_t n) {
    int rc = ctx->d_msg.reserve(ctx, n * 32, SV_ITEMS_FLOOR * 32);
    if (!rc) rc = ctx->d_key.reserve(ctx, n * 64, SV_ITEMS_FLOOR * 64);
    if (!rc) rc = ctx->d_sig.reserve(ctx, n * 64, SV_ITEMS_FLOOR * 64);
    if (!rc) rc = ctx->d_verdict.reserve(ctx, n, SV_ITEMS_FLOOR);
    return rc;
}
static int ensure_spans(sv_ctx* ctx, size_t n) {
    int rc = ctx->d_off.reserve(ctx, n * sizeof(u64), SV_ITEMS_FLOOR * sizeof(u64));
    return rc ? rc : ctx->d_len.reserve(ctx, n * sizeof(u32), SV_ITEMS_FLOOR * sizeof(u32));
}
static int ensure_gbuf(sv_ctx* ctx, size_t bytes) { return ctx->g_buf.reserve(ctx, bytes, SV_GBUF_FLOOR); }

// everything sv_create sets up after the defaults, on the context's device
static int ctx_init(sv_ctx* ctx) {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, ctx->device));
    ctx->sm_count = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : ctx->h2d_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (sv_ctx::slot_t& sl : ctx->slot) CK(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
    int rc = ctx->d_bases.reserve(ctx, 16 * sizeof(ge_mem), 16 * sizeof(ge_mem));
    if (!rc) rc = ctx->d_sink.reserve(ctx, 64, 64);
    if (rc) return rc;
    CK(cudaHostAlloc((void**)&ctx->h_small, (size_t)SV_SMALL_CAP * (32 + 64 + 64 + 2), cudaHostAllocMapped | cudaHostAllocPortable));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_main<SV_KIND_ECDSA33>, SV_MAIN_BLOCK, 0));
    if (occ < 1) occ = 1;
    ctx->main_grid = ctx->sm_count * occ;
    // deployment knob: leave a few CTA slots of the persistent curve kernel free for a collective's kernel that becomes
    // ready while the grid is resident (bench.py sets 2 when it gathers verdict bitmaps over NCCL)
    if (const char* e = getenv("SV_MAIN_GRID_RESERVE")) {
        int r = atoi(e);
        if (r > 0 && r < ctx->main_grid) ctx->main_grid -= r;
    }
    ctx->scratch_bytes = (size_t)ctx->main_grid * SV_MAIN_BLOCK * 8 * sizeof(qtab_entry);
    // G table and the launch slots' per-thread table slabs live in ONE allocation: a single L2 access-policy window
    // then covers everything the curve kernel reads more than once (see apply_l2_policy).  Layout [slab 0 | G table |
    // slab 1]: each slot's slab is contiguous with the G table, so one window covers both.
    static_assert(SV_NSLOTS == 2, "the hot-region layout below is for two launch slots");
    slab_layout hot;
    hot.take(ctx->scratch_bytes, 256);
    const size_t o_gt = hot.take((size_t)SV_GT_ENTRIES * sizeof(ge_mem), 256), o_slab1 = hot.take(ctx->scratch_bytes, 256);
    rc = ctx->d_hot.reserve(ctx, hot.size, hot.size);
    if (rc) return rc;
    ctx->slot[0].d_scratch = reinterpret_cast<qtab_entry*>(ctx->d_hot.p);
    ctx->d_gtab = reinterpret_cast<ge_mem*>(ctx->d_hot + o_gt);
    ctx->slot[1].d_scratch = reinterpret_cast<qtab_entry*>(ctx->d_hot + o_slab1);
    const size_t sb = o_gt, gt = o_slab1 - o_gt;
    ctx->hot_slab = sb;
    ctx->hot_gt = gt;
    // persisting L2 carve-out (as much as the device allows); failure is not an error: the hint is then simply absent
    int maxp = 0;
    if (cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, ctx->device) == cudaSuccess && maxp > 0 &&
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)maxp < sb + gt ? (size_t)maxp : sb + gt) == cudaSuccess)
        ctx->l2_persist = (size_t)maxp < sb + gt ? (size_t)maxp : sb + gt;  // one slab + the G table; the rest of L2 stays ordinary
    else (void)cudaGetLastError();
    ctx->l2_max_persist = maxp > 0 ? (size_t)maxp : 0;
    k_gtable_bases<<<1, 32, 0, ctx->stream>>>(ctx->d_bases);
    k_gtable_fill<<<(SV_GT_ENTRIES + 127) / 128, 128, 0, ctx->stream>>>(ctx->d_gtab, ctx->d_bases);
    ctx->launches += 2;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));
    return SV_OK;
}

extern "C" int sv_create(sv_ctx** out, int device) {
    sv_ctx* ctx = nullptr;
    if (!out) return SV_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail(nullptr, SV_ERR_NO_DEVICE, "no CUDA device (this engine has no CPU fallback)", e);
    if (device < 0 || device >= ndev) return fail(nullptr, SV_ERR_ARG, "bad device ordinal", cudaSuccess);
    dev_guard dg__;
    CK(dg__.enter(device));
    ctx = new sv_ctx();
    ctx->device = device;
    if (const char* e = getenv("SV_L2_POLICY")) ctx->l2_policy = atoi(e) != 0;  // measurement aid
    if (const char* e = getenv("SV_NOSQRT")) ctx->nosqrt = atoi(e) != 0;
    if (const char* e = getenv("SV_SMALL_MAX")) ctx->small_max = (size_t)strtoull(e, nullptr, 10);
    if (ctx->small_max > ctx->small_cap) ctx->small_max = ctx->small_cap;
    int rc = ctx_init(ctx);
    if (rc) {
        g_create_err = ctx->err;
        sv_destroy(ctx);
        return rc;
    }
    *out = ctx;
    return SV_OK;
}

extern "C" void sv_destroy(sv_ctx* ctx) {
    if (!ctx) return;
    dev_guard dg__;
    dg__.enter(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->h_small) cudaFreeHost(ctx->h_small);
    for (sv_ctx::slot_t& sl : ctx->slot)
        if (sl.done) cudaEventDestroy(sl.done);
    for (cudaEvent_t e : ctx->mark_ev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ctx->h2d_ev) if (e) cudaEventDestroy(e);
    for (cudaStream_t s : {ctx->copy_stream, ctx->stream2, ctx->stream}) if (s) cudaStreamDestroy(s);
    delete ctx;  // the device buffers free themselves
}

extern "C" int sv_get_info(const sv_ctx* ctx, sv_info* info) {
    if (!ctx || !info) return SV_ERR_ARG;
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, k_main<SV_KIND_ECDSA33>);
    info->device = ctx->device;
    info->sm_count = ctx->sm_count;
    info->main_block = SV_MAIN_BLOCK;
    info->main_grid = ctx->main_grid;
    info->main_regs = fa.numRegs;
    info->gtable_bytes = (size_t)SV_GT_ENTRIES * sizeof(ge_mem);
    info->scratch_bytes = ctx->scratch_bytes;
    info->l2_persist_bytes = ctx->l2_policy ? ctx->l2_persist : 0;
    info->l2_max_persist_bytes = ctx->l2_max_persist;
    info->launches = ctx->launches;
    return SV_OK;
}

// the ECDSA scalar side of n signatures into the work records (two launches)
static void launch_ecdsa_prep(sv_ctx* ctx, const u8* d_msg, const u8* d_sig, size_t n, sv_work* work, cudaStream_t st) {
    size_t threads = (n + SV_PREP_BATCH - 1) / SV_PREP_BATCH;
    k_prep_inv<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(d_msg, d_sig, n, work);
    k_prep_finish<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_msg, d_sig, n, work);
    ctx->launches += 2;
}
// grid of a curve kernel over n items: one thread per item, at most the persistent grid
static unsigned main_grid_for(const sv_ctx* ctx, size_t n) {
    size_t want = (n + SV_MAIN_BLOCK - 1) / SV_MAIN_BLOCK;
    return (unsigned)(want < (size_t)ctx->main_grid ? want : (size_t)ctx->main_grid);
}

// ECDSA batch with repeated keys: returns 1 if it handled the batch (enough repetition to pay), 0 if the caller should take
// the ordinary path, < 0 on error.  Synchronises the stream once (the number of distinct keys sizes the table array).
static int launch_verify_dedup(sv_ctx* ctx, int kind, const u8* d_msg, const u8* d_key, const u8* d_sig, size_t n,
                               u8* d_verdict, cudaStream_t st, u8* d_aux, u32* distinct_out) {
    // batches the small-batch kernel takes are faster there than through the search (one launch, ~0.5 ms)
    if (kind == SV_KIND_SCHNORR || n < 4096 || n <= ctx->small_max || n > 0x7FFFFFFFu) return 0;
    const int keylen = (int)sv_key_size(kind);
    u32 cap = 1;
    while (cap < 2 * n) cap <<= 1;
    slab_layout head;  // [slots cap][rep n][tid n][replist n][counter]
    const size_t o_slots = head.take(4 * (size_t)cap), o_rep = head.take(4 * n), o_tid = head.take(4 * n),
                 o_replist = head.take(4 * n), o_counter = head.take(4);
    int rc = ctx->dd_buf.reserve(ctx, head.size, SV_SCRATCH_FLOOR);
    if (rc) return rc;
    const dev_buf<>& B = ctx->dd_buf;
    u32 *slots = B.at<u32>(o_slots), *rep = B.at<u32>(o_rep), *tid = B.at<u32>(o_tid), *replist = B.at<u32>(o_replist),
        *counter = B.at<u32>(o_counter);
    CK(cudaMemsetAsync(slots, 0xFF, (size_t)cap * 4, st));
    CK(cudaMemsetAsync(counter, 0, 4, st));
    unsigned gb = (unsigned)((n + 255) / 256);
    k_dedup_insert<<<gb, 256, 0, st>>>(d_key, keylen, n, slots, cap - 1, rep);
    k_dedup_number<<<gb, 256, 0, st>>>(rep, n, counter, tid, replist);
    k_dedup_resolve<<<gb, 256, 0, st>>>(rep, n, tid);
    ctx->launches += 3;
    u32 distinct = 0;
    CK(cudaMemcpyAsync(&distinct, counter, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (distinct_out) *distinct_out = distinct;
    if ((size_t)distinct * 10 > n * 6) return 0;  // fewer than 40 % repeats: the per-thread tables are as cheap
    rc = ctx->sk_buf.reserve(ctx, (size_t)distinct * sizeof(sv_shared_key), SV_SCRATCH_FLOOR);
    if (rc) return rc;
    sv_shared_key* sk = ctx->sk_buf.at<sv_shared_key>(0);
    sv_ctx::slot_t* sl = nullptr;
    rc = acquire_slot(ctx, n, st, &sl);
    if (rc) return rc;
    CK(mark(ctx, MK_PREP, st));
    launch_ecdsa_prep(ctx, d_msg, d_sig, n, sl->d_work, st);
    CK(mark(ctx, MK_MAIN, st));
    k_sharedkey_build_many<<<(distinct + 127) / 128, 128, 0, st>>>(kind, d_key, keylen, replist, distinct, sk);
    k_main_shared<<<main_grid_for(ctx, n), SV_MAIN_BLOCK, 0, st>>>(sl->d_work, d_sig, n, ctx->d_gtab, sk, tid, d_verdict, d_aux);
    CK(mark(ctx, MK_END, st));
    ctx->launches += 2;
    CK(cudaGetLastError());
    rc = release_slot(ctx, sl, st);
    return rc ? rc : 1;
}

// L2 residency: the curve kernel re-reads the G comb table (34 MiB) and its own per-thread multiples tables (52 MiB per
// launch slot on an H100) ~70 times per verification, while inputs, work records and verdicts stream through once;
// without a policy the slabs cycle through L2 to DRAM.  The window
// marks [G table | slabs] as persisting (as many of its lines as the carve-out holds) and everything else on the stream
// as streaming.
static void apply_l2_policy(sv_ctx* ctx, cudaStream_t st, const void* slab) {
    if (!ctx->l2_policy || !ctx->l2_persist) return;
    // one window per stream: the table slab of the launch slot this stream is about to use (52 MiB on an H100, written once
    // and re-read ~70 times per verification) plus the G comb table next to it (34 MiB): the part the persisting carve-out
    // holds (32 MB on an H100) stays in L2 while inputs, work records and verdicts stream past.  (One window over G table +
    // both slabs at hit ratio carve-out/window raises DRAM traffic instead: the lines that lose the draw are treated as
    // streaming.)
    for (int i = 0; i < 4; i++)
        if (ctx->policy_streams[i] == st && ctx->policy_slabs[i] == slab) return;
    cudaStreamAttrValue v;
    memset(&v, 0, sizeof v);
    // slot 0: [slab 0 | G table], slot 1: [G table | slab 1] — the slab and the comb table, the two things a verification re-reads
    const bool first = slab == (const void*)ctx->slot[0].d_scratch;
    v.accessPolicyWindow.base_ptr = first ? (void*)ctx->d_hot.p : (void*)ctx->d_gtab;
    v.accessPolicyWindow.num_bytes = ctx->hot_slab + ctx->hot_gt;
    double ratio = 0.95 * (double)ctx->l2_persist / (double)(ctx->hot_slab + ctx->hot_gt);
    v.accessPolicyWindow.hitRatio = (float)(ratio > 1.0 ? 1.0 : ratio);
    v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    if (cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v) != cudaSuccess) { (void)cudaGetLastError(); return; }
    for (int i = 3; i > 0; i--) { ctx->policy_streams[i] = ctx->policy_streams[i - 1]; ctx->policy_slabs[i] = ctx->policy_slabs[i - 1]; }
    ctx->policy_streams[0] = st;
    ctx->policy_slabs[0] = slab;
}

static int launch_small(sv_ctx* ctx, int kind, const u8* d_msg, const u8* d_key, const u8* d_sig, size_t n,
                        u8* d_verdict, u8* d_aux, cudaStream_t st) {
    unsigned grid = (unsigned)((n + SV_SMALL_ITEMS - 1) / SV_SMALL_ITEMS);
    CK(mark(ctx, MK_PREP, st));
    CK(mark(ctx, MK_MAIN, st));
    // x-only keys: without the square root unless switched off (verify.cuh).  BIP-340 needs a field inversion at the end
    // either way, so dropping the square root is pure gain.  For compressed-key ECDSA the division
    // D/B would be an inversion the plain flow does not have, as long as the square root it replaces and divergent across
    // lanes: measured slower, so kind 0 stays on the plain flow.
    if (kind == SV_KIND_ECDSA33) k_small<SV_KIND_ECDSA33, false><<<grid, 160, 0, st>>>(d_msg, d_key, d_sig, n, ctx->d_gtab, d_verdict, d_aux);
    else if (kind == SV_KIND_ECDSA_XY) k_small<SV_KIND_ECDSA_XY, false><<<grid, 160, 0, st>>>(d_msg, d_key, d_sig, n, ctx->d_gtab, d_verdict, d_aux);
    else if (ctx->nosqrt) k_small<SV_KIND_SCHNORR, true><<<grid, 160, 0, st>>>(d_msg, d_key, d_sig, n, ctx->d_gtab, d_verdict, d_aux);
    else k_small<SV_KIND_SCHNORR, false><<<grid, 160, 0, st>>>(d_msg, d_key, d_sig, n, ctx->d_gtab, d_verdict, d_aux);
    CK(mark(ctx, MK_END, st));
    ctx->launches += 1;
    CK(cudaGetLastError());
    return SV_OK;
}

static int launch_verify(sv_ctx* ctx, int kind, const u8* d_msg, const u8* d_key, const u8* d_sig, size_t n,
                         u8* d_verdict, u32* d_bitmap, cudaStream_t st, u8* d_keyok = nullptr) {
    if (n == 0) return SV_OK;
    if (n <= ctx->small_max) {  // few signatures: the latency-oriented kernel (one launch, three warps per verification)
        int rc = launch_small(ctx, kind, d_msg, d_key, d_sig, n, d_verdict, d_keyok, st);
        if (rc) return rc;
        if (d_bitmap) {
            k_pack_bitmap<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_verdict, n, d_bitmap);
            ctx->launches += 1;
            CK(cudaGetLastError());
        }
        return SV_OK;
    }
    sv_ctx::slot_t* sl = nullptr;
    int rc = acquire_slot(ctx, n, st, &sl);
    if (rc) return rc;
    apply_l2_policy(ctx, st, sl->d_scratch);
    sv_work* work = sl->d_work;
    CK(mark(ctx, MK_PREP, st));
    if (kind == SV_KIND_SCHNORR) {
        k_prep_schnorr<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_msg, d_key, d_sig, n, work);
        ctx->launches += 1;
    } else {
        launch_ecdsa_prep(ctx, d_msg, d_sig, n, work, st);
    }
    CK(mark(ctx, MK_MAIN, st));
    const unsigned grid = main_grid_for(ctx, n);
    if (kind == SV_KIND_ECDSA33 && ctx->nosqrt) {
        // compressed keys: the flow that skips the square root (verify.cuh "without the square root")
        k_main<SV_KIND_ECDSA33_NS><<<grid, SV_MAIN_BLOCK, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, sl->d_scratch, d_verdict, nullptr);
        size_t threads = (n + SV_FINAL_BATCH - 1) / SV_FINAL_BATCH;
        k_final_ecdsa33<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, d_verdict, d_keyok);
        ctx->launches += 1;
    } else if (kind == SV_KIND_ECDSA33)
        k_main<SV_KIND_ECDSA33><<<grid, SV_MAIN_BLOCK, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, sl->d_scratch, d_verdict, d_keyok);
    else if (kind == SV_KIND_ECDSA_XY)
        k_main<SV_KIND_ECDSA_XY><<<grid, SV_MAIN_BLOCK, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, sl->d_scratch, d_verdict, d_keyok);
    else if (ctx->nosqrt) {
        k_main<SV_KIND_SCHNORR_NS><<<grid, SV_MAIN_BLOCK, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, sl->d_scratch, d_verdict, nullptr);
        size_t threads = (n + SV_FINAL_BATCH - 1) / SV_FINAL_BATCH;
        k_final_schnorr_ns<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, d_verdict);
        ctx->launches += 1;
    } else {
        k_main<SV_KIND_SCHNORR><<<grid, SV_MAIN_BLOCK, 0, st>>>(work, d_key, d_sig, n, ctx->d_gtab, sl->d_scratch, d_verdict, d_keyok);
        size_t threads = (n + SV_FINAL_BATCH - 1) / SV_FINAL_BATCH;
        k_final_schnorr<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(work, d_sig, n, d_verdict);
        ctx->launches += 1;
    }
    CK(mark(ctx, MK_END, st));
    ctx->launches += 1;
    if (d_bitmap) {
        size_t nb = (n + 255) / 256;
        k_pack_bitmap<<<(unsigned)nb, 256, 0, st>>>(d_verdict, n, d_bitmap);
        ctx->launches += 1;
    }
    CK(cudaGetLastError());
    return release_slot(ctx, sl, st);
}

extern "C" int sv_verify_device(sv_ctx* ctx, int kind, const void* d_msg32, const void* d_key, const void* d_sig64,
                                size_t n, void* d_verdicts, void* d_bitmap, void* stream) {
    if (!ctx || sv_key_size(kind) == 0 || (n && (!d_msg32 || !d_key || !d_sig64 || !d_verdicts))) return SV_ERR_ARG;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    return launch_verify(ctx, kind, (const u8*)d_msg32, (const u8*)d_key, (const u8*)d_sig64, n, (u8*)d_verdicts,
                         (u32*)d_bitmap, st);
}

extern "C" int sv_set_l2_policy(sv_ctx* ctx, int on) {
    if (!ctx) return SV_ERR_ARG;
    ctx->l2_policy = on ? 1 : 0;
    return SV_OK;
}
extern "C" int sv_set_dedup(sv_ctx* ctx, int on) {
    if (!ctx) return SV_ERR_ARG;
    ctx->dedup = on ? 1 : 0;
    return SV_OK;
}
extern "C" int sv_set_nosqrt(sv_ctx* ctx, int on) {
    if (!ctx) return SV_ERR_ARG;
    ctx->nosqrt = on ? 1 : 0;
    return SV_OK;
}
extern "C" unsigned sv_last_distinct_keys(const sv_ctx* ctx) { return ctx ? ctx->last_distinct : 0; }
extern "C" int sv_set_small_max(sv_ctx* ctx, size_t n) {
    if (!ctx) return SV_ERR_ARG;
    ctx->small_max = n < ctx->small_cap ? n : ctx->small_cap;
    return SV_OK;
}
extern "C" size_t sv_get_small_max(const sv_ctx* ctx) { return ctx ? ctx->small_max : 0; }

extern "C" int sv_set_profiling(sv_ctx* ctx, int on) {
    if (!ctx) return SV_ERR_ARG;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    if (on && !ctx->mark_ev[0])
        for (cudaEvent_t& e : ctx->mark_ev) CK(cudaEventCreate(&e));
    ctx->profiling = on ? 1 : 0;
    return SV_OK;
}
// device time of the last sv_verify_bolt12_host call: parse + Merkle + sighash kernels, then the verification kernels
extern "C" int sv_get_last_bolt12_timing(sv_ctx* ctx, float* merkle_ms, float* verify_ms) {
    if (!ctx || !ctx->profiling || !merkle_ms || !verify_ms) return SV_ERR_ARG;
    *merkle_ms = ctx->b12_ms[0];
    *verify_ms = ctx->b12_ms[1];
    return SV_OK;
}
// device time of the last sv_verify_bolt11_host call: parse and hash stage, then the verification and recovery stage
extern "C" int sv_get_last_bolt11_timing(sv_ctx* ctx, float* parse_ms, float* curve_ms) {
    if (!ctx || !ctx->profiling || !parse_ms || !curve_ms) return SV_ERR_ARG;
    *parse_ms = ctx->b11_ms[0];
    *curve_ms = ctx->b11_ms[1];
    return SV_OK;
}
// device time of the last sv_verify_* launch pair (call after the stream has been synchronised)
extern "C" int sv_get_last_timing(sv_ctx* ctx, float* prep_ms, float* main_ms) {
    if (!ctx || !ctx->profiling || !prep_ms || !main_ms) return SV_ERR_ARG;
    CK(mark_ms(ctx, MK_PREP, MK_MAIN, prep_ms));
    CK(mark_ms(ctx, MK_MAIN, MK_END, main_ms));
    return SV_OK;
}

extern "C" void* sv_get_stream(const sv_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

extern "C" int sv_sync(sv_ctx* ctx, void* stream) {
    if (!ctx) return SV_ERR_ARG;
    CK(cudaStreamSynchronize(stream ? (cudaStream_t)stream : ctx->stream));
    return SV_OK;
}

#ifndef SV_HOST_CHUNK
#define SV_HOST_CHUNK (1u << 21)
#endif

// Small batch (n <= small_max): inputs go through the pinned staging block, the kernel reads them over the bus itself and
// writes the verdict bytes back the same way: one launch and one stream synchronisation, nothing else.  same_key: `key` is
// one key, repeated for every item.
static int verify_small_host(sv_ctx* ctx, int kind, const u8* msg32, const u8* key, bool same_key, const u8* sig64, size_t n,
                             u8* verdicts) {
    const size_t ks = sv_key_size(kind);
    u8 *hm = ctx->h_small, *hk = hm + 32 * ctx->small_cap, *hs = hk + 64 * ctx->small_cap, *hv = hs + 64 * ctx->small_cap;
    memcpy(hm, msg32, 32 * n);
    if (same_key)
        for (size_t i = 0; i < n; i++) memcpy(hk + ks * i, key, ks);
    else
        memcpy(hk, key, ks * n);
    memcpy(hs, sig64, 64 * n);
    int rc = launch_small(ctx, kind, hm, hk, hs, n, hv, nullptr, ctx->stream);
    if (rc) return rc;
    CK(cudaStreamSynchronize(ctx->stream));
    memcpy(verdicts, hv, n);
    return SV_OK;
}

extern "C" int sv_verify_host(sv_ctx* ctx, int kind, const uint8_t* msg32, const uint8_t* key, const uint8_t* sig64,
                              size_t n, uint8_t* verdicts) {
    size_t ks_ = sv_key_size(kind);
    if (!ctx || ks_ == 0 || (n && (!msg32 || !key || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    if (n <= ctx->small_max) return verify_small_host(ctx, kind, msg32, key, false, sig64, n, verdicts);
    size_t chunk = n < SV_HOST_CHUNK ? n : SV_HOST_CHUNK;
    int rc = ensure_staging(ctx, chunk);
    if (rc) return rc;
    // Software pipeline inside a chunk: slices sized in whole waves of the persistent grid; slice k+1 is copied on
    // the copy stream while slice k runs; consecutive slices alternate between the two compute streams (each has its own
    // launch slot), so the partially filled last wave of one slice overlaps the next slice.  First slice small so the
    // kernels start early — and it also takes the odd remainder of the chunk: its thin last wave is covered by the second
    // slice, and the LAST slice (whose tail nothing can cover: the call is synchronous) ends on a full wave.
    const size_t wave = (size_t)ctx->main_grid * SV_MAIN_BLOCK;
    for (size_t off = 0; off < n; off += chunk) {
        size_t c = (n - off < chunk) ? (n - off) : chunk;
        size_t done = 0;
        int k = 0;
        const bool piped = c > 2 * wave;
        while (done < c) {
            size_t want = (k == 0) ? wave + c % wave : 6 * wave;
            size_t s = (c - done <= want + 2 * wave) ? (c - done) : want;  // do not leave a sliver behind
            if (k >= 7) s = c - done;
            cudaStream_t cs = piped ? ctx->copy_stream : ctx->stream;
            cudaStream_t ks = (piped && (k & 1)) ? ctx->stream2 : ctx->stream;
            CK(cudaMemcpyAsync(ctx->d_msg + 32 * done, msg32 + 32 * (off + done), 32 * s, cudaMemcpyHostToDevice, cs));
            CK(cudaMemcpyAsync(ctx->d_key + ks_ * done, key + ks_ * (off + done), ks_ * s, cudaMemcpyHostToDevice, cs));
            CK(cudaMemcpyAsync(ctx->d_sig + 64 * done, sig64 + 64 * (off + done), 64 * s, cudaMemcpyHostToDevice, cs));
            if (cs != ks) {
                CK(cudaEventRecord(ctx->h2d_ev[k], cs));
                CK(cudaStreamWaitEvent(ks, ctx->h2d_ev[k], 0));
            }
            rc = launch_verify(ctx, kind, ctx->d_msg + 32 * done, ctx->d_key + ks_ * done, ctx->d_sig + 64 * done, s,
                               ctx->d_verdict + done, nullptr, ks);
            if (rc) return rc;
            CK(cudaMemcpyAsync(verdicts + off + done, ctx->d_verdict + done, s, cudaMemcpyDeviceToHost, ks));
            done += s;
            k++;
        }
        // the next chunk reuses the staging buffers: its copies must not overtake this chunk's kernels
        CK(cudaStreamSynchronize(ctx->stream));
        if (piped) CK(cudaStreamSynchronize(ctx->stream2));
    }
    return SV_OK;
}

static int stage_spans(sv_ctx* ctx, const uint8_t* data, size_t data_len, const uint64_t* off, const uint32_t* len,
                       size_t n) {
    for (size_t i = 0; i < n; i++)
        if (off[i] > data_len || (size_t)len[i] > data_len - off[i]) return fail(ctx, SV_ERR_ARG, "span out of range", cudaSuccess);
    int rc = ctx->d_data.reserve(ctx, data_len, SV_GBUF_FLOOR);
    if (!rc) rc = ensure_spans(ctx, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_data, data, data_len, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_off, off, n * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_len, len, n * sizeof(u32), cudaMemcpyHostToDevice, ctx->stream));
    return SV_OK;
}

extern "C" int sv_verify_host_raw(sv_ctx* ctx, int kind, const uint8_t* data, size_t data_len, const uint64_t* off,
                                  const uint32_t* len, const uint8_t* key, const uint8_t* sig64, size_t n,
                                  uint8_t* verdicts) {
    size_t ks = sv_key_size(kind);
    if (!ctx || ks == 0 || (n && (!data || !off || !len || !key || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    rc = stage_spans(ctx, data, data_len, off, len, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_key, key, ks * n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_sig, sig64, 64 * n, cudaMemcpyHostToDevice, ctx->stream));
    k_sha256d<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(ctx->d_data, ctx->d_off, ctx->d_len, n, ctx->d_msg);
    ctx->launches += 1;
    rc = launch_verify(ctx, kind, ctx->d_msg, ctx->d_key, ctx->d_sig, n, ctx->d_verdict, nullptr, ctx->stream);
    if (rc) return rc;
    CK(cudaMemcpyAsync(verdicts, ctx->d_verdict, n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SV_OK;
}

extern "C" int sv_sha256d_host(sv_ctx* ctx, const uint8_t* data, size_t data_len, const uint64_t* off,
                               const uint32_t* len, size_t n, uint8_t* out32) {
    if (!ctx || (n && (!data || !off || !len || !out32))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    rc = stage_spans(ctx, data, data_len, off, len, n);
    if (rc) return rc;
    k_sha256d<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(ctx->d_data, ctx->d_off, ctx->d_len, n, ctx->d_msg);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out32, ctx->d_msg, 32 * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SV_OK;
}

extern "C" int sv_pubkey_parse_host(sv_ctx* ctx, const uint8_t* key33, size_t n, uint8_t* xy64, uint8_t* ok) {
    if (!ctx || (n && (!key33 || !xy64 || !ok))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    CK(cudaMemcpyAsync(ctx->d_key, key33, 33 * n, cudaMemcpyHostToDevice, ctx->stream));
    k_pubkey_parse<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(ctx->d_key, n, ctx->d_sig, ctx->d_verdict);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(xy64, ctx->d_sig, 64 * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(ok, ctx->d_verdict, n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return SV_OK;
}

// the ECDSA33 verification of a gossip batch's items: with key de-duplication when it is on and pays
static int gossip_verify_items(sv_ctx* ctx, u8* d_msg, u8* d_key, u8* d_sig, size_t n, u8* d_verdict, cudaStream_t st,
                               u8* d_keyok, u32* distinct_out) {
    // node keys repeat heavily inside a gossip batch (every channel of a node, its updates, its announcement)
    int rc = ctx->dedup ? launch_verify_dedup(ctx, SV_KIND_ECDSA33, d_msg, d_key, d_sig, n, d_verdict, st, d_keyok, distinct_out) : 0;
    if (rc == 0) rc = launch_verify(ctx, SV_KIND_ECDSA33, d_msg, d_key, d_sig, n, d_verdict, nullptr, st, d_keyok);
    else if (rc == 1) rc = SV_OK;
    return rc;
}

// gossip ingest with device-side slicing: blob = concatenated wire messages, msg_off/msg_len locate them.
// chain32 == nullptr: sv_verify_gossip_host (signers from the caller).  Otherwise sv_verify_gossip_burst_host: kinds
// (n_msgs bytes, or nullptr for all 0) says where each channel_update's signer comes from.
static int gossip_run(sv_ctx* ctx, const uint8_t* chain32, const uint8_t* blob, size_t blob_len, const uint64_t* msg_off,
                      const uint32_t* msg_len, size_t n_msgs, const uint8_t* kinds, const uint8_t* cu_signers33, int* status) {
    if (!ctx || (n_msgs && (!blob || !msg_off || !msg_len || !status))) return SV_ERR_ARG;
    if (n_msgs == 0) return SV_OK;
    const bool burst = chain32 != nullptr;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    // the host only reads the 2-byte type of each message to lay out the item slots
    std::vector<u32> base(n_msgs);
    size_t items = 0, n_ca = 0, n_cu = 0;
    for (size_t m = 0; m < n_msgs; m++) {
        if (msg_off[m] > blob_len || msg_len[m] > blob_len - msg_off[m]) return fail(ctx, SV_ERR_ARG, "message out of range", cudaSuccess);
        u32 type = msg_len[m] >= 2 ? (((u32)blob[msg_off[m]] << 8) | blob[msg_off[m] + 1]) : 0;
        base[m] = (u32)items;
        items += (type == 256) ? 4 : ((type == 257 || type == 258) ? 1 : 0);
        if (burst) {
            u8 k = kinds ? kinds[m] : 0;
            if (k > 2) return fail(ctx, SV_ERR_ARG, "signer_kind above 2", cudaSuccess);
            if (type == 258 && k != 0 && !cu_signers33) return fail(ctx, SV_ERR_ARG, "signer_kind 1 or 2 without signers33", cudaSuccess);
            n_ca += type == 256;
            n_cu += type == 258;
        }
    }
    if (items + n_cu > 0xFFFFFFFFu) return fail(ctx, SV_ERR_ARG, "too many signatures in one gossip batch", cudaSuccess);
    // burst: item slots [items, items + n_cu) take the updates of a repair round
    size_t cap = items + n_cu ? items + n_cu : 1;
    int rc = ensure_staging(ctx, cap);
    if (!rc) rc = ctx->d_data.reserve(ctx, blob_len, SV_GBUF_FLOOR);
    if (!rc) rc = ensure_spans(ctx, cap > n_msgs ? cap : n_msgs);
    if (rc) return rc;
    // one slab: [msg_off u64][msg_len u32][item_base u32][status int][signers 33B][keyok 1B per item], and for a burst
    // [kinds 1B][cand u32][repair list u32 (count, then indices)][chain_hash 32B][scid table u32]
    u32 tcap = 64;
    while (tcap < 2 * n_ca) tcap <<= 1;
    slab_layout L;
    const size_t o_moff = L.take(8 * n_msgs), o_mlen = L.take(4 * n_msgs), o_base = L.take(4 * n_msgs),
                 o_status = L.take(4 * n_msgs), o_signers = L.take(33 * n_msgs), o_keyok = L.take(cap),
                 o_kinds = L.take(burst ? n_msgs : 0), o_cand = L.take(burst ? 4 * n_msgs : 0),
                 o_rep = L.take(burst ? 4 * (n_msgs + 1) : 0), o_chain = L.take(burst ? 32 : 0),
                 o_slots = L.take(burst ? 4 * (size_t)tcap : 0);
    rc = ensure_gbuf(ctx, L.size + 64);
    if (rc) return rc;
    const dev_buf<>& G = ctx->g_buf;
    u64* d_moff = G.at<u64>(o_moff);
    u32 *d_mlen = G.at<u32>(o_mlen), *d_base = G.at<u32>(o_base);
    int* d_status = G.at<int>(o_status);
    u8* d_signers = cu_signers33 ? G.at<u8>(o_signers) : nullptr;
    u8* d_keyok = G.at<u8>(o_keyok);
    u8* d_kinds = burst ? G.at<u8>(o_kinds) : nullptr;
    u32* d_cand = burst ? G.at<u32>(o_cand) : nullptr;
    u32* d_repair = burst ? G.at<u32>(o_rep) : nullptr;
    u8* d_chain = burst ? G.at<u8>(o_chain) : nullptr;
    u32* d_slots = burst ? G.at<u32>(o_slots) : nullptr;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ctx->d_data, blob, blob_len, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_moff, msg_off, n_msgs * sizeof(u64), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_mlen, msg_len, n_msgs * sizeof(u32), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_base, base.data(), n_msgs * sizeof(u32), cudaMemcpyHostToDevice, st));
    if (cu_signers33) CK(cudaMemcpyAsync(d_signers, cu_signers33, n_msgs * 33, cudaMemcpyHostToDevice, st));
    if (burst) {
        if (kinds) CK(cudaMemcpyAsync(d_kinds, kinds, n_msgs, cudaMemcpyHostToDevice, st));
        else CK(cudaMemsetAsync(d_kinds, 0, n_msgs, st));
        CK(cudaMemcpyAsync(d_chain, chain32, 32, cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_repair, 0, 4, st));
    }
    unsigned gm = (unsigned)((n_msgs + 127) / 128);
    k_gossip_slice<<<gm, 128, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_base, d_signers, n_msgs, ctx->d_off, ctx->d_len,
                                       ctx->d_key, ctx->d_sig, d_status, d_chain, d_kinds);
    ctx->launches += 1;
    if (burst && n_cu) {
        // each update's signer from the first gated announcement of its scid, written into its item slot before hashing
        CK(cudaMemsetAsync(d_slots, 0xFF, (size_t)tcap * 4, st));
        k_scid_insert<<<(unsigned)((n_msgs + 255) / 256), 256, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_status, n_msgs, d_slots, tcap - 1);
        k_gossip_resolve<<<gm, 128, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_base, d_status, d_kinds, d_signers, n_msgs, d_slots,
                                             tcap - 1, d_cand, nullptr, 0, ctx->d_msg, ctx->d_key, ctx->d_sig);
        ctx->launches += 2;
    }
    if (items) {
        k_sha256d<<<(unsigned)((items + 127) / 128), 128, 0, st>>>(ctx->d_data, ctx->d_off, ctx->d_len, items, ctx->d_msg);
        ctx->launches += 1;
        rc = gossip_verify_items(ctx, ctx->d_msg, ctx->d_key, ctx->d_sig, items, ctx->d_verdict, st, d_keyok, &ctx->last_distinct);
        if (rc == SV_OK) {
            k_gossip_status<<<gm, 128, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_base, n_msgs, ctx->d_verdict, d_keyok, d_status,
                                                d_kinds, d_cand, burst ? d_repair : nullptr);
            ctx->launches += 1;
        }
    }
    u32 n_repair = 0;
    cudaError_t ce = cudaMemcpyAsync(status, d_status, n_msgs * sizeof(int), cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess && burst) ce = cudaMemcpyAsync(&n_repair, d_repair, 4, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (rc) return rc;
    if (ce != cudaSuccess) return fail(ctx, SV_ERR_CUDA, "gossip ingest", ce);
    if (n_repair) {
        // Repair round: some updates resolved to an announcement whose own signatures fail.  The right one is the first
        // announcement before the update whose status is 0 (every such status is final now), else the source peer (kind
        // 2), else none.  The table is rebuilt from those announcements only, the updates move to the spare item slots
        // [items, items + n_repair) and are verified again; k_gossip_status then settles them (and recomputes the rest
        // to the same values).  Nothing it resolves to can fail, so one round is enough.
        CK(cudaMemsetAsync(d_slots, 0xFF, (size_t)tcap * 4, st));
        k_scid_insert<<<(unsigned)((n_msgs + 255) / 256), 256, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_status, n_msgs, d_slots, tcap - 1);
        k_gossip_resolve<<<(n_repair + 127) / 128, 128, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_base, d_status, d_kinds, d_signers,
                                                                 n_repair, d_slots, tcap - 1, d_cand, d_repair, (u32)items,
                                                                 ctx->d_msg, ctx->d_key, ctx->d_sig);
        ctx->launches += 2;
        rc = gossip_verify_items(ctx, ctx->d_msg + 32 * items, ctx->d_key + 33 * items, ctx->d_sig + 64 * items, n_repair,
                                 ctx->d_verdict + items, st, d_keyok + items, nullptr);
        if (rc) return rc;
        k_gossip_status<<<gm, 128, 0, st>>>(ctx->d_data, d_moff, d_mlen, d_base, n_msgs, ctx->d_verdict, d_keyok, d_status,
                                            d_kinds, d_cand, nullptr);
        ctx->launches += 1;
        CK(cudaMemcpyAsync(status, d_status, n_msgs * sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    ctx->last_repair = n_repair;
    return SV_OK;
}

extern "C" int sv_verify_gossip_host(sv_ctx* ctx, const uint8_t* blob, size_t blob_len, const uint64_t* msg_off,
                                     const uint32_t* msg_len, size_t n_msgs, const uint8_t* cu_signers33, int* status) {
    return gossip_run(ctx, nullptr, blob, blob_len, msg_off, msg_len, n_msgs, nullptr, cu_signers33, status);
}

extern "C" int sv_verify_gossip_burst_host(sv_ctx* ctx, const uint8_t chain_hash32[32], const uint8_t* blob, size_t blob_len,
                                           const uint64_t* msg_off, const uint32_t* msg_len, size_t n_msgs,
                                           const uint8_t* signer_kind, const uint8_t* signers33, int* status) {
    if (!chain_hash32) return SV_ERR_ARG;
    return gossip_run(ctx, chain_hash32, blob, blob_len, msg_off, msg_len, n_msgs, signer_kind, signers33, status);
}
extern "C" unsigned sv_last_gossip_repairs(const sv_ctx* ctx) { return ctx ? ctx->last_repair : 0; }

// ---- a whole gossip_store: gossmap's record walk (host, headers only), every checksum, and every signature with the
// signer gossmap's channel table gives, on the device (see cln_sigverify.h) --------------------------------------------
extern "C" size_t sv_gossip_store_count(const uint8_t* store, size_t len) {
    if (!store || len < 1) return 0;
    gs_walk_end we;
    return (size_t)gs_walk(store, len, [](const gs_rec&) {}, &we);
}

static_assert(GS_ST_DELETED == SV_GS_DELETED && GS_ST_STORE_RECORD == SV_GS_STORE_RECORD && GS_ST_UNKNOWN == SV_GS_UNKNOWN &&
                  GS_ST_NOT_REACHED == SV_GS_NOT_REACHED && GS_ST_INCOMPLETE == SV_GS_INCOMPLETE &&
                  GS_ST_PARTIAL == SV_GS_PARTIAL && GS_ST_TRUNCATED == SV_GS_TRUNCATED && GS_ST_BAD_CRC == SV_GS_BAD_CRC &&
                  GS_ST_ENDED == SV_GS_ENDED && GS_ST_NO_AMOUNT == SV_GS_NO_AMOUNT,
              "gossip_store.cuh and cln_sigverify.h must agree on the record statuses");

// One pass over a staged store: the messages (item slots laid out from the 2-byte type) and channel events of the live
// records before `cut` (skip[r] != 0 leaves record r out as well), sliced, resolved, hashed and verified on the device.
// The slab stays allocated with the pass, so the prune's second round reuses the sorted events, the first holders and
// the digests (item slots of ctx->d_msg / d_sig; ctx's staging holds extra_items more slots after them).  MK_STORE_PASS
// (profiling mode) follows the last status.
struct store_pass {
    std::vector<u64> moff, eoff;
    std::vector<u32> mlen, base, mrec, emsg, msg_of;
    std::vector<u8> ekind;
    size_t items = 0, n_msgs = 0, nev = 0;
    std::vector<int> mstatus;  // per message: the statuses of sv_verify_gossip_store_host
    std::vector<u32> holder;   // per message: the message index of the holder the event saw, or GS_NONE
    dev_buf<> s;
    u64 *d_moff = nullptr, *d_eoff = nullptr, *d_key2 = nullptr;
    u32 *d_base = nullptr, *d_holder = nullptr, *d_emsg = nullptr, *d_val2 = nullptr;
    int* d_status = nullptr;
    u8 *d_ekind = nullptr, *d_ok = nullptr;
};
static int store_pass_run(sv_ctx* ctx, const u8* d_store, size_t len, const uint8_t* chain_hash32,
                          const std::vector<gs_rec>& rec, size_t cut, const u8* skip, size_t extra_items, store_pass& P) {
    cudaStream_t st = ctx->stream;
    P.msg_of.assign(rec.size(), GS_NONE);
    size_t& items = P.items;
    for (size_t r = 0; r < cut; r++) {
        if (rec[r].status != GS_LIVE || (skip && skip[r])) continue;
        const u32 t = rec[r].type, m = (u32)P.moff.size();
        if (t == 256 || t == 257 || t == 258) {
            P.msg_of[r] = m;
            P.moff.push_back(rec[r].off + GS_HDR); P.mlen.push_back(rec[r].len); P.base.push_back((u32)items);
            P.mrec.push_back((u32)r);
            items += t == 256 ? 4 : 1;
        }
        const int k = t == 256 ? GS_EV_ANN : t == 258 ? GS_EV_UPD : t == GS_DELETE_CHAN ? GS_EV_DEL : -1;
        if (k >= 0) {
            P.eoff.push_back(rec[r].off + GS_HDR); P.ekind.push_back((u8)k);
            P.emsg.push_back(k == GS_EV_DEL ? GS_NONE : m);
        }
    }
    const size_t n_msgs = P.n_msgs = P.moff.size(), nev = P.nev = P.eoff.size();
    if (items + extra_items >= 0xFFFFFFFFu || nev >= 0x7FFFFFFFu)
        return fail(ctx, SV_ERR_ARG, "too many signatures in one store", cudaSuccess);
    P.mstatus.assign(n_msgs, 0);
    P.holder.assign(n_msgs, GS_NONE);
    if (!n_msgs) {
        CK(mark(ctx, MK_STORE_PASS, st));
        CK(cudaStreamSynchronize(st));
        return SV_OK;
    }
    int rc = ensure_staging(ctx, items + extra_items);
    if (!rc) rc = ensure_spans(ctx, items);
    if (rc) return rc;
    size_t cub_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const u64*)nullptr, (u64*)nullptr, (const u32*)nullptr,
                                       (u32*)nullptr, (int)nev, 0, 64, st));
    // one slab: per message [off u64][len u32][item base u32][status int][holder u32][signer 33B][kind 1B], per item
    // [keyok 1B], per event [off u64][key u64 x2][msg u32][value u32 x2][kind 1B][ok 1B], chain hash, sort scratch
    slab_layout L;
    const size_t o_moff = L.take(8 * n_msgs), o_mlen = L.take(4 * n_msgs), o_base = L.take(4 * n_msgs),
                 o_status = L.take(4 * n_msgs), o_holder = L.take(4 * n_msgs), o_sig = L.take(33 * n_msgs),
                 o_kinds = L.take(n_msgs), o_keyok = L.take(items), o_eoff = L.take(8 * nev), o_key = L.take(8 * nev),
                 o_key2 = L.take(8 * nev), o_emsg = L.take(4 * nev), o_val = L.take(4 * nev),
                 o_val2 = L.take(4 * nev), o_ekind = L.take(nev), o_ok = L.take(nev), o_chain = L.take(32),
                 o_cub = L.take(cub_bytes);
    dev_buf<>& s = P.s;
    rc = s.reserve(ctx, L.size, L.size);
    if (rc) return rc;
    u64 *d_moff = P.d_moff = s.at<u64>(o_moff), *d_eoff = P.d_eoff = s.at<u64>(o_eoff), *d_key = s.at<u64>(o_key),
        *d_key2 = P.d_key2 = s.at<u64>(o_key2);
    u32 *d_mlen = s.at<u32>(o_mlen), *d_base = P.d_base = s.at<u32>(o_base), *d_holder = P.d_holder = s.at<u32>(o_holder),
        *d_emsg = P.d_emsg = s.at<u32>(o_emsg), *d_val = s.at<u32>(o_val), *d_val2 = P.d_val2 = s.at<u32>(o_val2);
    int* d_status = P.d_status = s.at<int>(o_status);
    u8 *d_signers = s + o_sig, *d_kinds = chain_hash32 ? s + o_kinds : nullptr, *d_keyok = s + o_keyok,
       *d_ekind = P.d_ekind = s + o_ekind, *d_ok = P.d_ok = s + o_ok, *d_chain = chain_hash32 ? s + o_chain : nullptr;
    CK(cudaMemcpyAsync(d_moff, P.moff.data(), 8 * n_msgs, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_mlen, P.mlen.data(), 4 * n_msgs, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_base, P.base.data(), 4 * n_msgs, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_holder, 0xFF, 4 * n_msgs, st));
    CK(cudaMemsetAsync(d_signers, 0, 33 * n_msgs, st));  // an update without a channel keeps the all-zero key
    if (chain_hash32) {
        // with a chain hash, k_gossip_slice applies gossipd's gates (burst mode); every update's signer is given
        CK(cudaMemsetAsync(d_kinds, 1, n_msgs, st));
        CK(cudaMemcpyAsync(d_chain, chain_hash32, 32, cudaMemcpyHostToDevice, st));
    }
    if (nev) {
        CK(cudaMemcpyAsync(d_eoff, P.eoff.data(), 8 * nev, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_emsg, P.emsg.data(), 4 * nev, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_ekind, P.ekind.data(), nev, cudaMemcpyHostToDevice, st));
        k_store_events<<<(unsigned)((nev + 255) / 256), 256, 0, st>>>(d_store, len, d_eoff, d_ekind, nev, d_key, d_val, d_ok);
        CK(cub::DeviceRadixSort::SortPairs(s + o_cub, cub_bytes, d_key, d_key2, d_val, d_val2, (int)nev, 0, 64, st));
        k_store_resolve<<<(unsigned)((nev + 127) / 128), 128, 0, st>>>(d_store, d_key2, d_val2, d_ok, d_ekind, d_eoff, d_emsg,
                                                                        nev, d_moff, d_holder, d_signers);
        ctx->launches += 2;
    }
    unsigned gm = (unsigned)((n_msgs + 127) / 128);
    k_gossip_slice<<<gm, 128, 0, st>>>(d_store, d_moff, d_mlen, d_base, d_signers, n_msgs, ctx->d_off, ctx->d_len,
                                       ctx->d_key, ctx->d_sig, d_status, d_chain, d_kinds);
    k_sha256d<<<(unsigned)((items + 127) / 128), 128, 0, st>>>(d_store, ctx->d_off, ctx->d_len, items, ctx->d_msg);
    ctx->launches += 2;
    rc = gossip_verify_items(ctx, ctx->d_msg, ctx->d_key, ctx->d_sig, items, ctx->d_verdict, st, d_keyok, &ctx->last_distinct);
    if (rc) return rc;
    k_gossip_status<<<gm, 128, 0, st>>>(d_store, d_moff, d_mlen, d_base, n_msgs, ctx->d_verdict, d_keyok, d_status,
                                        d_kinds, nullptr, nullptr);
    k_store_finish<<<(unsigned)((n_msgs + 255) / 256), 256, 0, st>>>(d_store, d_moff, d_holder, n_msgs, d_status);
    ctx->launches += 2;
    CK(mark(ctx, MK_STORE_PASS, st));
    CK(cudaMemcpyAsync(P.mstatus.data(), d_status, 4 * n_msgs, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(P.holder.data(), d_holder, 4 * n_msgs, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}

// The funding table staged on the device for one call and sorted there: the outputs by scid (their entries carried as
// values), the heights ascending.  A duplicate scid is SV_ERR_ARG.  MK_FUND_STAGE, MK_FUND_STAGED around the staging.
struct funding_stage {
    dev_buf<> s;
    gf_table t{};
};
static int funding_stage_run(sv_ctx* ctx, const sv_funding_table* tb, funding_stage& F) {
    cudaStream_t st = ctx->stream;
    const size_t n = tb->n_outputs, nb = tb->n_blocks;
    if (n >= 0x7FFFFFFFu || nb >= 0x7FFFFFFFu) return fail(ctx, SV_ERR_ARG, "funding table too large", cudaSuccess);
    size_t cub_pairs = 0, cub_keys = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, cub_pairs, (const u64*)nullptr, (u64*)nullptr, (const u32*)nullptr,
                                       (u32*)nullptr, (int)n, 0, 64, st));
    CK(cub::DeviceRadixSort::SortKeys(nullptr, cub_keys, (const u32*)nullptr, (u32*)nullptr, (int)nb, 0, 32, st));
    // one slab: per output [scid u64 x2][entry u32 x2][amount u64][script 34B], per height [u32 x2], the duplicate
    // flag, sort scratch
    slab_layout L;
    const size_t o_key = L.take(8 * n), o_key2 = L.take(8 * n), o_idx = L.take(4 * n), o_idx2 = L.take(4 * n),
                 o_sat = L.take(8 * n), o_script = L.take(34 * n), o_blk = L.take(4 * nb), o_blk2 = L.take(4 * nb),
                 o_dup = L.take(4), o_cub = L.take(cub_pairs > cub_keys ? cub_pairs : cub_keys);
    int rc = F.s.reserve(ctx, L.size, L.size);
    if (rc) return rc;
    dev_buf<>& s = F.s;
    u32* d_dup = s.at<u32>(o_dup);
    CK(mark(ctx, MK_FUND_STAGE, st));
    CK(cudaMemsetAsync(d_dup, 0, 4, st));
    if (n) {
        CK(cudaMemcpyAsync(s.at<u64>(o_key), tb->scid, 8 * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(s.at<u64>(o_sat), tb->satoshis, 8 * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(s + o_script, tb->script34, 34 * n, cudaMemcpyHostToDevice, st));
        k_funding_iota<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.at<u32>(o_idx), n);
        CK(cub::DeviceRadixSort::SortPairs(s + o_cub, cub_pairs, s.at<u64>(o_key), s.at<u64>(o_key2), s.at<u32>(o_idx),
                                           s.at<u32>(o_idx2), (int)n, 0, 64, st));
        k_funding_dups<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.at<u64>(o_key2), n, d_dup);
        ctx->launches += 2;
    }
    if (nb) {
        CK(cudaMemcpyAsync(s.at<u32>(o_blk), tb->blocks, 4 * nb, cudaMemcpyHostToDevice, st));
        CK(cub::DeviceRadixSort::SortKeys(s + o_cub, cub_keys, s.at<u32>(o_blk), s.at<u32>(o_blk2), (int)nb, 0, 32, st));
    }
    CK(mark(ctx, MK_FUND_STAGED, st));
    u32 dup = 0;
    CK(cudaMemcpyAsync(&dup, d_dup, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (dup) return fail(ctx, SV_ERR_ARG, "funding table: a scid appears twice", cudaSuccess);
    F.t = gf_table{s.at<u64>(o_key2), s.at<u32>(o_idx2), s.at<u64>(o_sat), s + o_script, (u64)n, s.at<u32>(o_blk2), (u64)nb};
    return SV_OK;
}
static bool funding_table_ok(const sv_funding_table* t) {
    return t && (!t->n_outputs || (t->scid && t->satoshis && t->script34)) && (!t->n_blocks || t->blocks);
}
static void funding_count(sv_gossip_funding_summary& F, u8 v) {
    uint64_t* per[7] = {nullptr, &F.funded, &F.unchecked, &F.dying, &F.no_txout, &F.script, &F.amount};
    if (v == GF_NONE) return;
    F.checked++;
    (*per[v])++;
}

static_assert(GF_NONE == SV_GF_NONE && GF_FUNDED == SV_GF_FUNDED && GF_UNCHECKED == SV_GF_UNCHECKED &&
                  GF_DYING == SV_GF_DYING && GF_NO_TXOUT == SV_GF_NO_TXOUT && GF_SCRIPT == SV_GF_SCRIPT &&
                  GF_AMOUNT == SV_GF_AMOUNT,
              "gossip_funding.cuh and cln_sigverify.h must agree on the funding verdicts");

// What the audit and the prune share: gossmap's header walk (past_truncated: the prune's), the funding table staged
// (with a table), the store staged in a buffer of its own (a store can be hundreds of MB) and the checksum of every live
// record and of the ENDED record tested on the device.  Marks: MK_STORE_COPY before the store's copy, MK_STORE_COPIED
// after it, MK_STORE_CRC after the checksums.
struct store_front {
    dev_guard dg;  // the first member: the buffers below are freed on the context's device
    std::vector<gs_rec> rec;
    gs_walk_end we;
    float walk_ms = 0;
    funding_stage F;
    dev_buf<> d_store, d_crc;
    std::vector<u8> bad;  // per record: 1 if its checksum was tested and failed
};
static int store_front_run(sv_ctx* ctx, const uint8_t* store, size_t len, const sv_funding_table* table,
                           size_t rec_capacity, bool past_truncated, store_front& G) {
    if (store[0] >> 5) return fail(ctx, SV_ERR_ARG, "gossip_store major version is not 0", cudaSuccess);
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<gs_rec>& rec = G.rec;
    rec.reserve(len / 256 + 16);
    const size_t nrec = gs_walk(store, len, [&rec](const gs_rec& r) { rec.push_back(r); }, &G.we, past_truncated);
    if (nrec > rec_capacity) return fail(ctx, SV_ERR_ARG, "rec_capacity is below the store's record count", cudaSuccess);
    if (nrec >= 0xFFFFFFFFu) return fail(ctx, SV_ERR_ARG, "too many records", cudaSuccess);
    // the records whose checksum map_catchup tests: every live one the walk reached, the ENDED record included
    std::vector<u64> crc_off;
    std::vector<u32> crc_rec;
    for (size_t r = 0; r < nrec; r++)
        if (rec[r].status == GS_LIVE || rec[r].status == GS_ST_ENDED) { crc_off.push_back(rec[r].off); crc_rec.push_back((u32)r); }
    G.walk_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    CK(G.dg.enter(ctx->device));
    cudaStream_t st = ctx->stream;
    if (table) {
        int rc = funding_stage_run(ctx, table, G.F);
        if (rc) return rc;
    }
    const size_t n = crc_off.size(), crc_bytes = n * 9 + 16;
    int rc = G.d_store.reserve(ctx, len, len);
    if (!rc) rc = G.d_crc.reserve(ctx, crc_bytes, crc_bytes);
    if (rc) return rc;
    u64* d_off = G.d_crc.at<u64>(0);
    u8* d_bad = G.d_crc.at<u8>(n * 8);
    CK(mark(ctx, MK_STORE_COPY, st));
    CK(cudaMemcpyAsync(G.d_store, store, len, cudaMemcpyHostToDevice, st));
    if (n) CK(cudaMemcpyAsync(d_off, crc_off.data(), n * 8, cudaMemcpyHostToDevice, st));
    CK(mark(ctx, MK_STORE_COPIED, st));
    if (n) {
        k_store_crc_flags<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(G.d_store, d_off, n, d_bad);
        ctx->launches += 1;
    }
    CK(mark(ctx, MK_STORE_CRC, st));
    std::vector<u8> bad(n);
    if (n) CK(cudaMemcpyAsync(bad.data(), d_bad, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    G.bad.assign(nrec, 0);
    for (size_t k = 0; k < n; k++) G.bad[crc_rec[k]] = bad[k];
    return SV_OK;
}

// The funding verdicts of P's announcements whose status is 0 and whose record lies before cut, GF_NONE for every other
// message: in d_fund on the device (n_msgs bytes at its start, which k_prune_mark reads) and in fund on the host once the
// stream is synchronised.  MK_FUND_KERNEL, MK_FUND_DONE around the kernel.
static int store_funding_run(sv_ctx* ctx, const store_front& G, size_t len, const store_pass& P, size_t cut,
                             dev_buf<>& d_fund, std::vector<u8>& fund) {
    cudaStream_t st = ctx->stream;
    const size_t n = P.n_msgs;
    std::vector<u32> cand;
    for (size_t m = 0; m < n; m++)
        if (P.mrec[m] < cut && G.rec[P.mrec[m]].type == 256 && P.mstatus[m] == 0) cand.push_back((u32)m);
    slab_layout L;
    L.take(n);
    const size_t o_cand = L.take(4 * cand.size());
    int rc = d_fund.reserve(ctx, L.size, L.size);
    if (rc) return rc;
    u32* d_cand = d_fund.at<u32>(o_cand);
    CK(cudaMemsetAsync(d_fund, GF_NONE, n, st));
    CK(mark(ctx, MK_FUND_KERNEL, st));
    if (!cand.empty()) {
        CK(cudaMemcpyAsync(d_cand, cand.data(), 4 * cand.size(), cudaMemcpyHostToDevice, st));
        k_store_funding<<<(unsigned)((cand.size() + 127) / 128), 128, 0, st>>>(G.d_store, len, P.d_moff, d_cand, cand.size(),
                                                                               G.F.t, d_fund);
        ctx->launches += 1;
    }
    CK(mark(ctx, MK_FUND_DONE, st));
    fund.resize(n);
    if (n) CK(cudaMemcpyAsync(fund.data(), d_fund, n, cudaMemcpyDeviceToHost, st));
    return SV_OK;
}

// gossmap's store-only records: a load passes over them; a record of any other type it does not know is unknown
static bool gs_store_record(u32 t) {
    return t == GS_CHANNEL_AMOUNT || t == GS_DELETE_CHAN || t == GS_CHAN_DYING || t == GS_UUID;
}
// a reached record's status: the walk's if it is not live, else GS_ST_BAD_CRC if its checksum failed, else its message's
// status (m: its message in P), else GS_ST_STORE_RECORD or GS_ST_UNKNOWN
static int store_status(const gs_rec& r, u8 bad, u32 m, const store_pass& P) {
    if (r.status != GS_LIVE) return r.status;
    if (bad) return GS_ST_BAD_CRC;
    if (m != GS_NONE) return P.mstatus[m];
    return gs_store_record(r.type) ? GS_ST_STORE_RECORD : GS_ST_UNKNOWN;
}

// sv_verify_gossip_store_host, and with a table (else NULL) sv_verify_gossip_store_funding_host
static int store_audit(sv_ctx* ctx, const uint8_t* store, size_t len, const uint8_t* chain_hash32,
                       const sv_funding_table* table, uint64_t* rec_off, uint16_t* rec_type, int* rec_status,
                       uint64_t* rec_holder, uint8_t* rec_funding, size_t rec_capacity, sv_gossip_store_summary* sum,
                       sv_gossip_funding_summary* fsum) {
    store_front G;
    int rc = store_front_run(ctx, store, len, table, rec_capacity, false, G);
    if (rc) return rc;
    const std::vector<gs_rec>& rec = G.rec;
    const size_t nrec = rec.size();
    const gs_walk_end& we = G.we;
    // the walk ends at the first bad checksum: only the records before it are verified
    size_t cut = 0;
    while (cut < nrec && !G.bad[cut]) cut++;
    int cut_status = cut < nrec ? GS_ST_BAD_CRC : 0;
    store_pass P;
    rc = store_pass_run(ctx, G.d_store, len, chain_hash32, rec, cut, nullptr, 0, P);
    if (rc) return rc;
    const std::vector<u32>&msg_of = P.msg_of, &mrec = P.mrec, &holder = P.holder;
    // an announcement without room for its amount record stops the walk unless it is redundant (add_channel returns the
    // channel that already holds the scid before it looks for the amount)
    if (we.no_amount < cut && holder[msg_of[we.no_amount]] == GS_NONE) {
        cut = we.no_amount;
        cut_status = GS_ST_NO_AMOUNT;
    }
    // the funding verdicts of the reached announcements whose status is 0
    dev_buf<> d_fund;
    std::vector<u8> fund;
    if (table) {
        rc = store_funding_run(ctx, G, len, P, cut, d_fund, fund);
        if (rc) return rc;
        CK(cudaStreamSynchronize(ctx->stream));
    }
    sv_gossip_store_summary S;
    memset(&S, 0, sizeof S);
    sv_gossip_funding_summary FS;
    memset(&FS, 0, sizeof FS);
    S.version = store[0];
    S.stop = cut_status ? cut_status : we.stop;
    S.end_offset = cut_status ? rec[cut].off : we.end;
    S.records = nrec;
    for (size_t r = 0; r < nrec; r++) {
        const u32 t = rec[r].type, m = msg_of[r];
        const bool reached = !(cut_status && r >= cut);
        const int s = reached ? store_status(rec[r], G.bad[r], m, P) : r == cut ? cut_status : GS_ST_NOT_REACHED;
        u64 h = ~(u64)0;
        if (reached && m != GS_NONE) {
            if (holder[m] != GS_NONE) h = rec[mrec[holder[m]]].off;
            S.redundant_announcements += t == 256 && holder[m] != GS_NONE;
            S.updates_without_channel += t == 258 && len - rec[r].off - GS_HDR >= GS_UPD_READ && holder[m] == GS_NONE;
            S.good += s == 0; S.bad_signature += s >= 1 && s <= 4; S.malformed += s == -1; S.no_channel += s == -2;
            S.wrong_chain += s == -3; S.bad_order += s == -4;
        }
        if (s == GS_ST_ENDED && rec[r].len >= 10)
            for (int b = 0; b < 8; b++) S.ended_equivalent_offset = (S.ended_equivalent_offset << 8) | store[rec[r].off + GS_HDR + 2 + b];
        rec_off[r] = rec[r].off;
        rec_type[r] = (uint16_t)t;
        rec_status[r] = s;
        if (rec_holder) rec_holder[r] = h;
        if (table) {
            const u8 v = reached && m != GS_NONE ? fund[m] : (u8)GF_NONE;
            rec_funding[r] = v;
            funding_count(FS, v);
        }
        S.deleted += s == GS_ST_DELETED; S.store_records += s == GS_ST_STORE_RECORD; S.unknown += s == GS_ST_UNKNOWN;
        S.not_reached += s == GS_ST_NOT_REACHED;
    }
    *sum = S;
    if (table) *fsum = FS;
    ctx->gs_ms[0] = G.walk_ms;
    if (ctx->profiling) {
        CK(mark_ms(ctx, MK_STORE_COPY, MK_STORE_COPIED, &ctx->gs_ms[1]));
        CK(mark_ms(ctx, MK_STORE_COPIED, MK_STORE_CRC, &ctx->gs_ms[2]));
        CK(mark_ms(ctx, MK_STORE_CRC, MK_STORE_PASS, &ctx->gs_ms[3]));
        if (table) {
            CK(mark_ms(ctx, MK_FUND_STAGE, MK_FUND_STAGED, &ctx->gf_ms[0]));
            CK(mark_ms(ctx, MK_FUND_KERNEL, MK_FUND_DONE, &ctx->gf_ms[1]));
        }
    }
    return SV_OK;
}
extern "C" int sv_verify_gossip_store_host(sv_ctx* ctx, const uint8_t* store, size_t len, const uint8_t* chain_hash32,
                                           uint64_t* rec_off, uint16_t* rec_type, int* rec_status, uint64_t* rec_holder,
                                           size_t rec_capacity, sv_gossip_store_summary* sum) {
    if (!ctx || !store || len < 1 || !sum || (rec_capacity && (!rec_off || !rec_type || !rec_status))) return SV_ERR_ARG;
    return store_audit(ctx, store, len, chain_hash32, nullptr, rec_off, rec_type, rec_status, rec_holder, nullptr,
                       rec_capacity, sum, nullptr);
}
extern "C" int sv_verify_gossip_store_funding_host(sv_ctx* ctx, const uint8_t* store, size_t len,
                                                   const uint8_t* chain_hash32, const sv_funding_table* table,
                                                   uint64_t* rec_off, uint16_t* rec_type, int* rec_status,
                                                   uint64_t* rec_holder, uint8_t* rec_funding, size_t rec_capacity,
                                                   sv_gossip_store_summary* sum, sv_gossip_funding_summary* fsum) {
    if (!ctx || !store || len < 1 || !sum || !fsum || !funding_table_ok(table) ||
        (rec_capacity && (!rec_off || !rec_type || !rec_status || !rec_funding)))
        return SV_ERR_ARG;
    return store_audit(ctx, store, len, chain_hash32, table, rec_off, rec_type, rec_status, rec_holder, rec_funding,
                       rec_capacity, sum, fsum);
}
extern "C" int sv_get_last_gossip_funding_timing(sv_ctx* ctx, float* ms2) {
    if (!ctx || !ctx->profiling || !ms2) return SV_ERR_ARG;
    for (int i = 0; i < 2; i++) ms2[i] = ctx->gf_ms[i];
    return SV_OK;
}
// where the last sv_verify_gossip_store_host call spent its time (profiling mode): host header walk, H2D copy of the store,
// checksum kernel, then slicing, resolution, hashing and verification to the last status (device events)
extern "C" int sv_get_last_gossip_store_timing(sv_ctx* ctx, float* ms4) {
    if (!ctx || !ctx->profiling || !ms4) return SV_ERR_ARG;
    for (int i = 0; i < 4; i++) ms4[i] = ctx->gs_ms[i];
    return SV_OK;
}

// ---- pruning a gossip_store: the records gossmap should not trust marked deleted (see cln_sigverify.h) --------------
extern "C" size_t sv_gossip_prune_count(const uint8_t* store, size_t len) {
    if (!store || len < 1) return 0;
    gs_walk_end we;
    return (size_t)gs_walk(store, len, [](const gs_rec&) {}, &we, true);
}

// sv_prune_gossip_store_host, and with a table (else NULL) sv_prune_gossip_store_funding_host
static int store_prune(sv_ctx* ctx, const uint8_t* store, size_t len, const uint8_t* chain_hash32,
                       const sv_funding_table* table, uint8_t* out, uint64_t* rec_off, uint16_t* rec_type, int* rec_status,
                       uint8_t* rec_pruned, uint8_t* rec_funding, size_t rec_capacity, sv_gossip_prune_summary* sum,
                       sv_gossip_funding_summary* fsum) {
    store_front G;
    int rc = store_front_run(ctx, store, len, table, rec_capacity, true, G);
    if (rc) return rc;
    const std::vector<gs_rec>& rec = G.rec;
    const std::vector<u8>& skip = G.bad;  // a live record whose checksum fails is deleted and left out of both rounds
    const size_t nrec = rec.size();
    const gs_walk_end& we = G.we;
    u8* d_store = G.d_store;
    cudaStream_t st = ctx->stream;
    size_t n_upd = 0;
    for (const gs_rec& r : rec) n_upd += r.status == GS_LIVE && r.type == 258;
    // first round: the audit's statuses and channel table over the records with good checksums
    store_pass P;
    rc = store_pass_run(ctx, d_store, len, chain_hash32, rec, nrec, skip.data(), n_upd, P);
    if (rc) return rc;
    const size_t n_msgs = P.n_msgs, nev = P.nev, items = P.items;
    // the funding verdicts of the announcements whose first-round status is 0: the refused ones join rule 2.  Without a
    // table d_fund stays empty, and k_prune_mark reads no verdicts.
    dev_buf<> d_fund;
    std::vector<u8> fund;
    if (table) {
        rc = store_funding_run(ctx, G, len, P, nrec, d_fund, fund);
        if (rc) return rc;
    }
    std::vector<u8> reason(n_msgs, SV_GP_KEPT);
    u32 n_moved = 0;
    if (n_msgs) {
        // second round: the deletions of the first, the table again over the sorted events with those announcements
        // masked out, and the updates whose holder changed verified again under their new signer
        slab_layout L;
        const size_t o_reason = L.take(n_msgs), o_holder2 = L.take(4 * n_msgs), o_sig2 = L.take(33 * n_msgs),
                     o_ok2 = L.take(nev), o_list = L.take(4 * (n_upd + 1)), o_keyok = L.take(n_upd);
        dev_buf<> s2;
        rc = s2.reserve(ctx, L.size, L.size);
        if (rc) return rc;
        u8 *d_reason = s2 + o_reason, *d_sig2 = s2 + o_sig2, *d_ok2 = s2 + o_ok2, *d_keyok = s2 + o_keyok;
        u32 *d_holder2 = s2.at<u32>(o_holder2), *d_list = s2.at<u32>(o_list);
        CK(cudaMemsetAsync(d_holder2, 0xFF, 4 * n_msgs, st));
        CK(cudaMemsetAsync(d_list, 0, 4, st));
        const size_t nmark = n_msgs > nev ? n_msgs : nev;
        k_prune_mark<<<(unsigned)((nmark + 255) / 256), 256, 0, st>>>(d_store, P.d_moff, P.d_status, n_msgs, P.d_ekind,
                                                                     P.d_emsg, P.d_ok, nev, d_fund, d_reason, d_ok2);
        ctx->launches += 1;
        if (nev) {
            k_store_resolve<<<(unsigned)((nev + 127) / 128), 128, 0, st>>>(d_store, P.d_key2, P.d_val2, d_ok2, P.d_ekind,
                                                                            P.d_eoff, P.d_emsg, nev, P.d_moff, d_holder2,
                                                                            d_sig2);
            ctx->launches += 1;
        }
        k_prune_select<<<(unsigned)((n_msgs + 127) / 128), 128, 0, st>>>(d_store, P.d_moff, P.d_status, n_msgs, P.d_holder,
                                                                        d_holder2, P.d_base, d_sig2, d_reason, d_list,
                                                                        (u32)items, ctx->d_msg, ctx->d_key, ctx->d_sig);
        ctx->launches += 1;
        CK(cudaMemcpyAsync(&n_moved, d_list, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (n_moved) {
            rc = gossip_verify_items(ctx, ctx->d_msg + 32 * items, ctx->d_key + 33 * items, ctx->d_sig + 64 * items, n_moved,
                                     ctx->d_verdict + items, st, d_keyok, nullptr);
            if (rc) return rc;
            k_prune_settle<<<(n_moved + 255) / 256, 256, 0, st>>>(d_list, ctx->d_verdict + items, d_reason);
            ctx->launches += 1;
        }
        CK(mark(ctx, MK_PRUNE_ROUND2, st));
        CK(cudaMemcpyAsync(reason.data(), d_reason, n_msgs, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    } else {
        CK(mark(ctx, MK_PRUNE_ROUND2, st));
    }
    // every record's reason, in store order
    std::vector<u8> pr(nrec, SV_GP_KEPT);
    for (size_t r = 0; r < nrec; r++) {
        const u32 t = rec[r].type, m = P.msg_of[r];
        if (rec[r].status == GS_ST_TRUNCATED) pr[r] = SV_GP_TRUNCATED;
        else if (rec[r].status != GS_LIVE) continue;
        else if (skip[r]) pr[r] = SV_GP_BAD_CRC;
        else if (m != GS_NONE) pr[r] = reason[m];
        else if (!gs_store_record(t)) pr[r] = SV_GP_UNKNOWN;
        // the amount record right after a deleted announcement goes with it (gossip_store_del)
        if (r > 0 && pr[r] == SV_GP_KEPT && t == GS_CHANNEL_AMOUNT && pr[r - 1] != SV_GP_KEPT && rec[r - 1].type == 256)
            pr[r] = SV_GP_AMOUNT;
    }
    // an announcement kept without room for its amount record stops the walk: it and the records after it stay
    size_t cut = nrec;
    if (we.no_amount < nrec && pr[we.no_amount] == SV_GP_KEPT) cut = we.no_amount;
    std::vector<u64> doff;
    for (size_t r = 0; r < cut; r++)
        if (pr[r] != SV_GP_KEPT) doff.push_back(rec[r].off);
    // the flag writes on the device; only the changed flag bytes come back
    const size_t nd = doff.size();
    std::vector<u8> flag_hi(nd);
    if (nd) {
        dev_buf<> t_del;
        rc = t_del.reserve(ctx, nd * 9, nd * 9);
        if (rc) return rc;
        u64* d_doff = t_del.at<u64>(0);
        u8* d_hi = t_del.at<u8>(nd * 8);
        CK(cudaMemcpyAsync(d_doff, doff.data(), nd * 8, cudaMemcpyHostToDevice, st));
        k_prune_flags<<<(unsigned)((nd + 255) / 256), 256, 0, st>>>(d_store, d_doff, nd, d_hi);
        ctx->launches += 1;
        CK(cudaMemcpyAsync(flag_hi.data(), d_hi, nd, cudaMemcpyDeviceToHost, st));
    }
    CK(mark(ctx, MK_PRUNE_FLAGS, st));
    CK(cudaStreamSynchronize(st));
    if (out != store) memcpy(out, store, len);
    for (size_t i = 0; i < nd; i++) out[doff[i]] = flag_hi[i];
    sv_gossip_prune_summary S;
    memset(&S, 0, sizeof S);
    S.version = store[0];
    S.stop = cut < nrec ? GS_ST_NO_AMOUNT : we.stop;
    S.end_offset = cut < nrec ? rec[cut].off : we.end;
    S.records = nrec;
    S.reverified = n_moved;
    sv_gossip_funding_summary FS;
    memset(&FS, 0, sizeof FS);
    uint64_t* per_reason[10] = {nullptr, &S.bad_crc, &S.truncated, &S.message, &S.redundant, &S.no_channel,
                                &S.signature, &S.amount, &S.unknown, &FS.deleted};
    for (size_t r = 0; r < nrec; r++) {
        const u32 t = rec[r].type, m = P.msg_of[r];
        const int s = r < cut ? store_status(rec[r], skip[r], m, P) : r == cut ? GS_ST_NO_AMOUNT : GS_ST_NOT_REACHED;
        const u8 why = r < cut ? pr[r] : (u8)SV_GP_KEPT;
        rec_off[r] = rec[r].off;
        rec_type[r] = (uint16_t)t;
        rec_status[r] = s;
        rec_pruned[r] = why;
        if (why) { S.pruned++; (*per_reason[why])++; }
        if (table) {
            const u8 v = r < cut && m != GS_NONE ? fund[m] : (u8)GF_NONE;
            rec_funding[r] = v;
            funding_count(FS, v);
        }
    }
    *sum = S;
    if (table) *fsum = FS;
    ctx->gp_ms[0] = G.walk_ms;
    if (ctx->profiling) {
        CK(mark_ms(ctx, MK_STORE_COPY, MK_STORE_PASS, &ctx->gp_ms[1]));
        CK(mark_ms(ctx, MK_STORE_PASS, MK_PRUNE_ROUND2, &ctx->gp_ms[2]));
        CK(mark_ms(ctx, MK_PRUNE_ROUND2, MK_PRUNE_FLAGS, &ctx->gp_ms[3]));
        if (table) {
            CK(mark_ms(ctx, MK_FUND_STAGE, MK_FUND_STAGED, &ctx->gf_ms[0]));
            CK(mark_ms(ctx, MK_FUND_KERNEL, MK_FUND_DONE, &ctx->gf_ms[1]));
        }
    }
    return SV_OK;
}
extern "C" int sv_prune_gossip_store_host(sv_ctx* ctx, const uint8_t* store, size_t len, const uint8_t* chain_hash32,
                                          uint8_t* out, uint64_t* rec_off, uint16_t* rec_type, int* rec_status,
                                          uint8_t* rec_pruned, size_t rec_capacity, sv_gossip_prune_summary* sum) {
    if (!ctx || !store || !out || len < 1 || !sum || (rec_capacity && (!rec_off || !rec_type || !rec_status || !rec_pruned)))
        return SV_ERR_ARG;
    return store_prune(ctx, store, len, chain_hash32, nullptr, out, rec_off, rec_type, rec_status, rec_pruned, nullptr,
                       rec_capacity, sum, nullptr);
}
extern "C" int sv_prune_gossip_store_funding_host(sv_ctx* ctx, const uint8_t* store, size_t len,
                                                  const uint8_t* chain_hash32, const sv_funding_table* table, uint8_t* out,
                                                  uint64_t* rec_off, uint16_t* rec_type, int* rec_status,
                                                  uint8_t* rec_pruned, uint8_t* rec_funding, size_t rec_capacity,
                                                  sv_gossip_prune_summary* sum, sv_gossip_funding_summary* fsum) {
    if (!ctx || !store || !out || len < 1 || !sum || !fsum || !funding_table_ok(table) ||
        (rec_capacity && (!rec_off || !rec_type || !rec_status || !rec_pruned || !rec_funding)))
        return SV_ERR_ARG;
    return store_prune(ctx, store, len, chain_hash32, table, out, rec_off, rec_type, rec_status, rec_pruned, rec_funding,
                       rec_capacity, sum, fsum);
}
extern "C" int sv_get_last_gossip_prune_timing(sv_ctx* ctx, float* ms4) {
    if (!ctx || !ctx->profiling || !ms4) return SV_ERR_ARG;
    for (int i = 0; i < 4; i++) ms4[i] = ctx->gp_ms[i];
    return SV_OK;
}

// ---- salvaging a gossip_store past damaged record headers (see cln_sigverify.h) -----------------------------------
// The store staged once: the sorted sound offsets (the filter twice around the scan of its per-block counts, then the
// checksums), the host walk's breaks, and the restore check of each.  gv_ms (profiling mode): the two filter passes and
// the scan (device marks around the kernels only, without the count's copy back and the candidate buffer's allocation
// between them), the checksums, the host walk.
static int salvage_run(sv_ctx* ctx, const uint8_t* store, size_t len, std::vector<u64>& sound, std::vector<u64>& brk,
                       std::vector<u8>& restore) {
    for (float& ms : ctx->gv_ms) ms = 0;
    if (len < 1 + GS_HDR + 2) return SV_OK;  // no record fits
    cudaStream_t st = ctx->stream;
    const u64 nb = (len - 1 + 255) / 256;
    size_t scan_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (u64*)nullptr, nb + 1, st));
    // [per-block counts u64 nb + 1][scan scratch]
    slab_layout L;
    L.take(8 * (nb + 1));
    const size_t o_scan = L.take(scan_bytes);
    dev_buf<> d_store, d_cnt, d_cand, d_brk;
    int rc = d_store.reserve(ctx, len, len);
    if (!rc) rc = d_cnt.reserve(ctx, L.size, L.size);
    if (rc) return rc;
    u64* cnt = d_cnt.at<u64>(0);
    CK(cudaMemcpyAsync(d_store, store, len, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(cnt + nb, 0, 8, st));  // count[0, nb) exclusive, count[nb] the total
    CK(mark(ctx, MK_SALVAGE_COUNT, st));
    k_salvage_filter<<<(unsigned)nb, 256, 0, st>>>(d_store, len, cnt, nullptr);
    CK(cub::DeviceScan::ExclusiveSum(d_cnt + o_scan, scan_bytes, cnt, nb + 1, st));
    ctx->launches += 1;
    CK(mark(ctx, MK_SALVAGE_SCANNED, st));
    u64 n = 0;
    CK(cudaMemcpyAsync(&n, cnt + nb, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (n) {
        rc = d_cand.reserve(ctx, 9 * n, 9 * n);
        if (rc) return rc;
        u64* cand = d_cand.at<u64>(0);
        u8* ok = d_cand.at<u8>(8 * n);
        CK(mark(ctx, MK_SALVAGE_EMIT, st));
        k_salvage_filter<<<(unsigned)nb, 256, 0, st>>>(d_store, len, cnt, cand);
        CK(mark(ctx, MK_SALVAGE_CRC, st));
        k_salvage_crc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_store, cand, n, ok);
        ctx->launches += 2;
        CK(mark(ctx, MK_SALVAGE_DONE, st));
        std::vector<u64> c(n);
        std::vector<u8> good(n);
        CK(cudaMemcpyAsync(c.data(), cand, 8 * n, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(good.data(), ok, n, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (u64 k = 0; k < n; k++)
            if (good[k]) sound.push_back(c[k]);
    } else if (ctx->profiling) {
        CK(mark(ctx, MK_SALVAGE_EMIT, st));
        CK(mark(ctx, MK_SALVAGE_CRC, st));
        CK(mark(ctx, MK_SALVAGE_DONE, st));
        CK(cudaStreamSynchronize(st));
    }
    if (ctx->profiling) {
        float a, b;
        CK(mark_ms(ctx, MK_SALVAGE_COUNT, MK_SALVAGE_SCANNED, &a));
        CK(mark_ms(ctx, MK_SALVAGE_EMIT, MK_SALVAGE_CRC, &b));
        ctx->gv_ms[0] = a + b;
        CK(mark_ms(ctx, MK_SALVAGE_CRC, MK_SALVAGE_DONE, &ctx->gv_ms[1]));
    }
    const auto t0 = std::chrono::steady_clock::now();
    gs_salvage_breaks(store, len, sound.data(), sound.size(), [&brk](u64 t, u64 q) { brk.push_back(t); brk.push_back(q); });
    ctx->gv_ms[2] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const size_t nbrk = brk.size() / 2;
    restore.assign(nbrk, 0);
    if (!nbrk) return SV_OK;
    rc = d_brk.reserve(ctx, 17 * nbrk, 17 * nbrk);
    if (rc) return rc;
    CK(cudaMemcpyAsync(d_brk, brk.data(), 16 * nbrk, cudaMemcpyHostToDevice, st));
    k_salvage_restore<<<(unsigned)((nbrk + 7) / 8), 256, 0, st>>>(d_store, d_brk.at<u64>(0), nbrk, d_brk + 16 * nbrk);
    ctx->launches += 1;
    CK(cudaMemcpyAsync(restore.data(), d_brk + 16 * nbrk, nbrk, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}
extern "C" int sv_salvage_gossip_store_host(sv_ctx* ctx, const uint8_t* store, size_t len, uint8_t* out, uint64_t* act_off,
                                            uint64_t* act_resume, uint8_t* act_kind, size_t act_capacity,
                                            sv_gossip_salvage_summary* sum) {
    if (!ctx || !store || !out || len < 1 || !sum || (act_capacity && (!act_off || !act_resume || !act_kind)))
        return SV_ERR_ARG;
    if (store[0] >> 5) return fail(ctx, SV_ERR_ARG, "gossip_store major version is not 0", cudaSuccess);
    dev_guard dg;
    CK(dg.enter(ctx->device));
    std::vector<u64> sound, brk;
    std::vector<u8> restore;
    int rc = salvage_run(ctx, store, len, sound, brk, restore);
    if (rc) return rc;
    const size_t n = restore.size();
    std::vector<u64> t(n), q(n);
    for (size_t i = 0; i < n; i++) {
        t[i] = brk[2 * i];
        q[i] = brk[2 * i + 1];
        if (i < act_capacity) {
            act_off[i] = t[i];
            act_resume[i] = q[i];
            act_kind[i] = restore[i] ? SV_SALVAGE_RESTORED : SV_SALVAGE_BRIDGED;
        }
    }
    if (out != store) memcpy(out, store, len);
    const gs_salvage_count c = gs_salvage_apply(out, t.data(), q.data(), restore.data(), n);
    *sum = sv_gossip_salvage_summary{c.breaks, c.restored, c.bridged, c.bridged_bytes, c.fillers, (uint64_t)sound.size()};
    return SV_OK;
}
extern "C" int sv_get_last_gossip_salvage_timing(sv_ctx* ctx, float* ms3) {
    if (!ctx || !ctx->profiling || !ms3) return SV_ERR_ARG;
    for (int i = 0; i < 3; i++) ms3[i] = ctx->gv_ms[i];
    return SV_OK;
}

// n ECDSA signatures by ONE key (channeld's HTLC loop): table of the key built once, ladder-only kernel
extern "C" int sv_verify_samekey_host(sv_ctx* ctx, int kind, const uint8_t* key, const uint8_t* msg32, const uint8_t* sig64,
                                      size_t n, uint8_t* verdicts) {
    size_t ks = sv_key_size(kind);
    if (!ctx || ks == 0 || kind == SV_KIND_SCHNORR || (n && (!key || !msg32 || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    // a commitment_signed carries at most 483 HTLC signatures: latency matters more than the 18 % of work a shared table
    // saves, so small same-key batches take the small-batch path with the key repeated per item
    if (n <= ctx->small_max) return verify_small_host(ctx, kind, msg32, key, true, sig64, n, verdicts);
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    sv_ctx::slot_t* sl = nullptr;
    rc = acquire_slot(ctx, n, st, &sl);
    if (rc) return rc;
    // the shared key's table lives at the head of the slot's (otherwise unused) per-thread table slab
    sv_shared_key* d_sk = reinterpret_cast<sv_shared_key*>(sl->d_scratch);
    CK(cudaMemcpyAsync(ctx->d_key, key, ks, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_msg, msg32, 32 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_sig, sig64, 64 * n, cudaMemcpyHostToDevice, st));
    k_sharedkey_build<<<1, 32, 0, st>>>(kind, ctx->d_key, d_sk);
    launch_ecdsa_prep(ctx, ctx->d_msg, ctx->d_sig, n, sl->d_work, st);
    k_main_shared<<<main_grid_for(ctx, n), SV_MAIN_BLOCK, 0, st>>>(sl->d_work, ctx->d_sig, n, ctx->d_gtab, d_sk, nullptr,
                                                                   ctx->d_verdict, nullptr);
    ctx->launches += 2;
    CK(cudaGetLastError());
    rc = release_slot(ctx, sl, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(verdicts, ctx->d_verdict, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}

// check_tx_sig with the BIP143 sighash computed on the device (channeld's per-HTLC loop as one launch)
static_assert(sizeof(sv_tx_item) == sizeof(sv_tx), "host and device views of the transaction item must agree");
extern "C" int sv_verify_tx_host(sv_ctx* ctx, int kind, const sv_tx* txs, const uint8_t* scripts, size_t scripts_len,
                                 const uint8_t* key, const uint8_t* sig64, size_t n, uint8_t* verdicts,
                                 uint8_t* sighash32_out) {
    size_t ks = sv_key_size(kind);
    if (!ctx || ks == 0 || kind == SV_KIND_SCHNORR || (n && (!txs || !key || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    for (size_t i = 0; i < n; i++)
        if ((size_t)txs[i].script_off + txs[i].script_len > scripts_len ||
            (size_t)txs[i].out_script_off + txs[i].out_script_len > scripts_len ||
            ((txs[i].flags & SV_TX_INPUTS_SERIALIZED) &&
             ((size_t)txs[i].prevouts_off + txs[i].prevouts_len > scripts_len ||
              (size_t)txs[i].sequences_off + txs[i].sequences_len > scripts_len)))
            return fail(ctx, SV_ERR_ARG, "script span out of range", cudaSuccess);
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    // transaction records + sighash-ok flags in the auxiliary slab (no allocation on the steady-state call path)
    slab_layout L;
    const size_t o_txs = L.take(n * sizeof(sv_tx_item)), o_ok = L.take(n);
    int rc = ensure_staging(ctx, n);
    if (!rc) rc = ctx->d_data.reserve(ctx, scripts_len + 1, SV_GBUF_FLOOR);
    if (!rc) rc = ensure_gbuf(ctx, L.size + 64);
    if (rc) return rc;
    sv_tx_item* d_txs = ctx->g_buf.at<sv_tx_item>(o_txs);
    u8* d_ok = ctx->g_buf + o_ok;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(d_txs, txs, n * sizeof(sv_tx_item), cudaMemcpyHostToDevice, st));
    if (scripts_len) CK(cudaMemcpyAsync(ctx->d_data, scripts, scripts_len, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_key, key, ks * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_sig, sig64, 64 * n, cudaMemcpyHostToDevice, st));
    k_bip143<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_txs, ctx->d_data, n, ctx->d_msg, d_ok);
    ctx->launches += 1;
    rc = launch_verify(ctx, kind, ctx->d_msg, ctx->d_key, ctx->d_sig, n, ctx->d_verdict, nullptr, st);
    cudaError_t ce = cudaSuccess;
    if (rc == SV_OK) {
        k_mask_verdicts<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ctx->d_verdict, d_ok, n);
        ctx->launches += 1;
        ce = cudaMemcpyAsync(verdicts, ctx->d_verdict, n, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess && sighash32_out) ce = cudaMemcpyAsync(sighash32_out, ctx->d_msg, 32 * n, cudaMemcpyDeviceToHost, st);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    }
    if (rc) return rc;
    if (ce != cudaSuccess) return fail(ctx, SV_ERR_CUDA, "sv_verify_tx_host", ce);
    return SV_OK;
}

// ---- mixed batches: kinds[n] tags, keys in 64-byte slots (the first 33 / 64 / 32 bytes used) ----------------------
// inputs already on the device; scratch = [count u32 x4][idx u32 x 3n]; staging = the context's SoA staging arrays
static int mixed_device(sv_ctx* ctx, const u8* d_kinds, const u8* d_msg, const u8* d_key64, const u8* d_sig, size_t n,
                        u8* d_out, u32* d_scratch, cudaStream_t st) {
    u32* d_count = d_scratch;
    u32* d_idx = d_scratch + 4;
    CK(cudaMemsetAsync(d_count, 0, 16, st));
    CK(cudaMemsetAsync(d_out, 0, n, st));
    k_mixed_index<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_kinds, n, d_count, d_idx);
    ctx->launches += 1;
    u32 count[4];
    CK(cudaMemcpyAsync(count, d_count, 16, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));  // the per-kind launch sizes are needed on the host
    size_t o = 0;
    for (int kind = 0; kind < 3; kind++) {
        size_t c = count[kind];
        if (!c) continue;
        size_t ks = sv_key_size(kind);
        u8 *om = ctx->d_msg + 32 * o, *ok = ctx->d_key + 64 * o, *os = ctx->d_sig + 64 * o, *ov = ctx->d_verdict + o;
        const u32* list = d_idx + (size_t)kind * n;
        k_mixed_gather<<<(unsigned)((c + 255) / 256), 256, 0, st>>>(list, c, (int)ks, d_msg, d_key64, d_sig, om, ok, os);
        int rc = launch_verify(ctx, kind, om, ok, os, c, ov, nullptr, st);
        if (rc) return rc;
        k_mixed_scatter<<<(unsigned)((c + 255) / 256), 256, 0, st>>>(list, c, ov, d_out);
        ctx->launches += 2;
        o += c;
    }
    CK(cudaGetLastError());
    return SV_OK;
}
extern "C" int sv_verify_mixed_device(sv_ctx* ctx, const void* d_kinds, const void* d_msg32, const void* d_key64,
                                      const void* d_sig64, size_t n, void* d_verdicts, void* stream) {
    if (!ctx || (n && (!d_kinds || !d_msg32 || !d_key64 || !d_sig64 || !d_verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    rc = ensure_gbuf(ctx, 16 + 12 * n + 64);
    if (rc) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    return mixed_device(ctx, (const u8*)d_kinds, (const u8*)d_msg32, (const u8*)d_key64, (const u8*)d_sig64, n,
                        (u8*)d_verdicts, ctx->g_buf.at<u32>(0), st);
}
extern "C" int sv_verify_mixed_host(sv_ctx* ctx, const uint8_t* kinds, const uint8_t* msg32, const uint8_t* key64,
                                    const uint8_t* sig64, size_t n, uint8_t* verdicts) {
    if (!ctx || (n && (!kinds || !msg32 || !key64 || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    // aux slab: [count + idx lists][kinds n][msg 32n][key 64n][sig 64n][out n]
    slab_layout L;
    const size_t o_scratch = L.take(16 + 12 * n), o_kinds = L.take(n), o_m = L.take(32 * n), o_k = L.take(64 * n),
                 o_s = L.take(64 * n), o_o = L.take(n);
    int rc = ensure_staging(ctx, n);
    if (!rc) rc = ensure_gbuf(ctx, L.size + 64);
    if (rc) return rc;
    u8 *d_kinds = ctx->g_buf + o_kinds, *d_m = ctx->g_buf + o_m, *d_k = ctx->g_buf + o_k, *d_s = ctx->g_buf + o_s,
       *d_o = ctx->g_buf + o_o;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(d_kinds, kinds, n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_m, msg32, 32 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_k, key64, 64 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_s, sig64, 64 * n, cudaMemcpyHostToDevice, st));
    rc = mixed_device(ctx, d_kinds, d_m, d_k, d_s, n, d_o, ctx->g_buf.at<u32>(o_scratch), st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(verdicts, d_o, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}

// ---- onchaind's HTLC fee grind (onchaind/onchaind.c:389-437) in one call ---------------------------------------------
// The host stages one transaction record, the two script spans, the key and the signature (a few hundred bytes), runs
// k_grind_setup once and then k_grind over ascending chunks of SV_GRIND_CHUNK feerates, reading back the 8-byte best
// feerate after each chunk and stopping at the first chunk with a match.
#define SV_GRIND_CHUNK (1u << 20)
extern "C" int sv_grind_tx_fee_host(sv_ctx* ctx, int kind, const sv_tx* tx, const uint8_t* scripts, size_t scripts_len,
                                    const uint8_t* key, const uint8_t* sig64, uint64_t weight, uint32_t min_feerate,
                                    uint32_t max_feerate, int64_t* feerate_out, uint64_t* fee_out) {
    size_t ks = sv_key_size(kind);
    if (!ctx || ks == 0 || kind == SV_KIND_SCHNORR || !tx || !key || !sig64 || !feerate_out || !fee_out ||
        (scripts_len && !scripts))
        return SV_ERR_ARG;
    if (tx->flags) return fail(ctx, SV_ERR_ARG, "sv_grind_tx_fee_host: tx->flags must be 0 (one input, one output)", cudaSuccess);
    if (weight >> 32) return fail(ctx, SV_ERR_ARG, "sv_grind_tx_fee_host: weight >= 2^32", cudaSuccess);
    if ((size_t)tx->script_off + tx->script_len > scripts_len || (size_t)tx->out_script_off + tx->out_script_len > scripts_len)
        return fail(ctx, SV_ERR_ARG, "script span out of range", cudaSuccess);
    *feerate_out = -1;
    *fee_out = 0;
    if (min_feerate > max_feerate) return SV_OK;
    const u64 last = grind_last_feerate(min_feerate, max_feerate, weight, tx->input_amount);
    if (last < min_feerate) return SV_OK;  // the fee at min_feerate is already above the input: the loop breaks at once
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    // staging: [state | 8 table entries | tx record | best | key 64 | sig 64 | witness script | output script]; everything
    // from the tx record on goes over in one copy
    const size_t blob_len = (size_t)tx->script_len + tx->out_script_len;
    slab_layout L;
    const size_t o_state = L.take(sizeof(sv_grind_state), 256), o_tab = L.take(8 * sizeof(qtab_entry), 256),
                 o_tx = L.take(sizeof(sv_tx_item)), o_best = L.take(16), o_key = L.take(64), o_sig = L.take(64),
                 o_blob = L.take(blob_len);
    int rc = ensure_gbuf(ctx, L.size + 16);
    if (rc) return rc;
    std::vector<u8> h(L.size - o_tx, 0);
    sv_tx_item t;
    memcpy(&t, tx, sizeof t);
    t.script_off = 0;
    t.out_script_off = tx->script_len;
    memcpy(h.data(), &t, sizeof t);
    memset(h.data() + (o_best - o_tx), 0xFF, 8);
    memcpy(h.data() + (o_key - o_tx), key, ks);
    memcpy(h.data() + (o_sig - o_tx), sig64, 64);
    if (tx->script_len) memcpy(h.data() + (o_blob - o_tx), scripts + tx->script_off, tx->script_len);
    if (tx->out_script_len) memcpy(h.data() + (o_blob - o_tx) + tx->script_len, scripts + tx->out_script_off, tx->out_script_len);
    u8* b = ctx->g_buf;
    sv_grind_state* d_state = ctx->g_buf.at<sv_grind_state>(o_state);
    qtab_entry* d_tab = ctx->g_buf.at<qtab_entry>(o_tab);
    const sv_tx_item* d_tx = ctx->g_buf.at<sv_tx_item>(o_tx);
    unsigned long long* d_best = ctx->g_buf.at<unsigned long long>(o_best);
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(b + o_tx, h.data(), h.size(), cudaMemcpyHostToDevice, st));
    k_grind_setup<<<1, 32, 0, st>>>(kind, b + o_key, b + o_sig, d_tx, b + o_blob, d_tab, d_state);
    ctx->launches += 1;
    CK(cudaGetLastError());
    unsigned long long best = ~0ull;
    for (u64 first = min_feerate; first <= last; first += SV_GRIND_CHUNK) {
        u64 count = last - first + 1 < SV_GRIND_CHUNK ? last - first + 1 : SV_GRIND_CHUNK;
        k_grind<<<(unsigned)((count + 127) / 128), 128, 0, st>>>(d_state, d_tx, b + o_blob, b + o_sig, ctx->d_gtab, weight,
                                                                 min_feerate, first, count, d_best);
        ctx->launches += 1;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(&best, d_best, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (best != ~0ull) break;
    }
    if (best != ~0ull) {
        *feerate_out = (int64_t)best;
        *fee_out = best * weight / 1000;
    }
    return SV_OK;
}

// ---- BOLT12: bolt12_check_signature (common/bolt12.c:80-92) for n TLV streams -------------------------------------------
// The host copies bytes only.  The device parses every stream, builds its Merkle root and sighash (k_b12_*), verifies the
// sighashes through the ordinary BIP-340 path (launch_verify) and folds parse status and verdict into one int.  One host
// synchronisation in the middle: the total field count sizes the record / node scratch.
//
// One pass over n streams under ntags sighash tags: tag t is "lightning" || messagenames[t] || fieldnames[t]
// (bip340_sighash_init(sctx, "lightning", messagename, fieldname): the three strings back to back), stream i is hashed
// under tag tag_of[i] (tag_of NULL: every stream under tag 0).  The arguments are checked by the callers.
static int bolt12_pass(sv_ctx* ctx, size_t ntags, const char* const* messagenames, const char* const* fieldnames,
                       const uint32_t* tag_of, const uint8_t* blob, size_t blob_len, const uint64_t* off, const uint32_t* len,
                       const uint8_t* xonly32, const uint8_t* sig64, size_t n, int* status, uint8_t* sighash32_out) {
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    rc = stage_spans(ctx, blob, blob_len, off, len, n);
    if (rc) return rc;
    // the tag table travels in one copy: [tag offsets u64 ntags][tag lengths u32 ntags][tag_of u32 n][tag bytes]
    slab_layout T;
    const size_t t_off = T.take(8 * ntags), t_len = T.take(4 * ntags), t_of = T.take(tag_of ? 4 * n : 0), t_bytes = T.take(0);
    std::vector<u8> tab(t_bytes);
    for (size_t t = 0; t < ntags; t++) {
        const u64 o = tab.size() - t_bytes;
        const size_t a = strlen(messagenames[t]), b = strlen(fieldnames[t]);
        if (9 + a + b > 0xFFFFFFFFu) return fail(ctx, SV_ERR_ARG, "tag too long", cudaSuccess);
        const u32 l = (u32)(9 + a + b);
        memcpy(tab.data() + t_off + 8 * t, &o, 8);
        memcpy(tab.data() + t_len + 4 * t, &l, 4);
        tab.insert(tab.end(), "lightning", "lightning" + 9);
        tab.insert(tab.end(), messagenames[t], messagenames[t] + a);
        tab.insert(tab.end(), fieldnames[t], fieldnames[t] + b);
    }
    if (tag_of) memcpy(tab.data() + t_of, tag_of, 4 * n);
    cudaStream_t st = ctx->stream;
    size_t scan_bytes = 0;
    CK(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, (const u32*)nullptr, (u64*)nullptr, cuda::std::plus<>{}, (u64)0,
                                      n + 1, st));
    // per-call scratch in the auxiliary slab: [cnt u32 n+1][base u64 n+1][status int n][tree tags]
    // [sighash midstates 32 x ntags][tag table][scan scratch].  base: the exclusive prefix sums of the field counts,
    // accumulated in 64 bits (ExclusiveSum would add u32 counts in u32); with cnt[n] = 0, base[n] is the total.
    slab_layout L;
    const size_t o_cnt = L.take(4 * (n + 1)), o_base = L.take(8 * (n + 1)), o_status = L.take(4 * n),
                 o_tags = L.take(sizeof(b12_tags)), o_mid = L.take(32 * ntags), o_tab = L.take(tab.size()),
                 o_scan = L.take(scan_bytes);
    rc = ensure_gbuf(ctx, L.size + 64);
    if (rc) return rc;
    const dev_buf<>& G = ctx->g_buf;
    u32* d_cnt = G.at<u32>(o_cnt);
    u64* d_base = G.at<u64>(o_base);
    int* d_status = G.at<int>(o_status);
    b12_tags* d_tags = G.at<b12_tags>(o_tags);
    u32* d_mid = G.at<u32>(o_mid);
    u8* d_tab = G + o_tab;
    CK(cudaMemcpyAsync(ctx->d_key, xonly32, 32 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_sig, sig64, 64 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_tab, tab.data(), tab.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_cnt + n, 0, 4, st));
    CK(mark(ctx, MK_B12_PARSE, st));
    k_b12_tags<<<(unsigned)((ntags + 1 + 63) / 64), 64, 0, st>>>(d_tab + t_bytes, reinterpret_cast<const u64*>(d_tab + t_off),
                                                              reinterpret_cast<const u32*>(d_tab + t_len), ntags, d_tags, d_mid);
    k_b12_count<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(ctx->d_data, ctx->d_off, ctx->d_len, n, d_cnt);
    ctx->launches += 2;
    CK(cudaGetLastError());
    CK(cub::DeviceScan::ExclusiveScan(G + o_scan, scan_bytes, d_cnt, d_base, cuda::std::plus<>{}, (u64)0, n + 1, st));
    u64 total = 0;
    CK(cudaMemcpyAsync(&total, d_base + n, sizeof total, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const size_t per_field = sizeof(b12_field) + 32;
    if (total > ((size_t)-1) / per_field) return fail(ctx, SV_ERR_NOMEM, "BOLT12 field scratch", cudaSuccess);
    rc = ctx->b12_buf.reserve(ctx, (size_t)total * per_field, SV_SCRATCH_FLOOR);
    if (rc) return rc;
    b12_field* d_recs = ctx->b12_buf.at<b12_field>(0);
    u32* d_nodes = ctx->b12_buf.at<u32>((size_t)total * sizeof(b12_field));
    k_b12_merkle<<<(unsigned)((n + SV_B12_WARPS - 1) / SV_B12_WARPS), 32 * SV_B12_WARPS, 0, st>>>(
        ctx->d_data, ctx->d_off, ctx->d_len, n, d_cnt, d_base, d_tags, d_mid,
        tag_of ? reinterpret_cast<const u32*>(d_tab + t_of) : nullptr, d_recs, d_nodes, ctx->d_msg);
    ctx->launches += 1;
    CK(mark(ctx, MK_B12_SIGHASH, st));
    CK(cudaGetLastError());
    // the sighashes are ordinary BIP-340 messages from here on: small-batch kernel or the throughput kernels
    rc = launch_verify(ctx, SV_KIND_SCHNORR, ctx->d_msg, ctx->d_key, ctx->d_sig, n, ctx->d_verdict, nullptr, st);
    if (rc) return rc;
    k_b12_status<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_cnt, ctx->d_verdict, n, d_status);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(status, d_status, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    if (sighash32_out) CK(cudaMemcpyAsync(sighash32_out, ctx->d_msg, 32 * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ctx->profiling) {
        CK(mark_ms(ctx, MK_B12_PARSE, MK_B12_SIGHASH, &ctx->b12_ms[0]));
        CK(mark_ms(ctx, MK_PREP, MK_END, &ctx->b12_ms[1]));
    }
    return SV_OK;
}
extern "C" int sv_verify_bolt12_host(sv_ctx* ctx, const char* messagename, const char* fieldname, const uint8_t* blob,
                                     size_t blob_len, const uint64_t* off, const uint32_t* len, const uint8_t* xonly32,
                                     const uint8_t* sig64, size_t n, int* status, uint8_t* sighash32_out) {
    if (!ctx || !messagename || !fieldname || (n && (!blob || !off || !len || !xonly32 || !sig64 || !status))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    return bolt12_pass(ctx, 1, &messagename, &fieldname, nullptr, blob, blob_len, off, len, xonly32, sig64, n, status,
                       sighash32_out);
}
// the same with a tag per stream: the whole batch is one pass (one launch sequence) whatever the number of tags
extern "C" int sv_verify_bolt12_tagged_host(sv_ctx* ctx, size_t ntags, const char* const* messagenames,
                                            const char* const* fieldnames, const uint32_t* tag_of, const uint8_t* blob,
                                            size_t blob_len, const uint64_t* off, const uint32_t* len, const uint8_t* xonly32,
                                            const uint8_t* sig64, size_t n, int* status, uint8_t* sighash32_out) {
    if (!ctx || (ntags && (!messagenames || !fieldnames))) return SV_ERR_ARG;
    for (size_t t = 0; t < ntags; t++)
        if (!messagenames[t] || !fieldnames[t]) return SV_ERR_ARG;
    if (n && (!ntags || !tag_of || !blob || !off || !len || !xonly32 || !sig64 || !status)) return SV_ERR_ARG;
    for (size_t i = 0; i < n; i++)
        if (tag_of[i] >= ntags) return fail(ctx, SV_ERR_ARG, "tag_of out of range", cudaSuccess);
    if (n == 0) return SV_OK;
    return bolt12_pass(ctx, ntags, messagenames, fieldnames, tag_of, blob, blob_len, off, len, xonly32, sig64, n, status,
                       sighash32_out);
}

// ---- BOLT11: bolt11_decode's signature step (common/bolt11.c:980-1062) for n invoice strings ---------------------------
// The host copies bytes only.  k_b11_parse gives every invoice its structure, signature and signing hash; two prefix sums
// (cub's device scan) pack the invoices with an `n` key and the ones to recover.  One host synchronisation reads the
// two counts.  `n` invoices then take the ordinary compressed-key ECDSA path (small-batch kernel or throughput kernels,
// launch_verify).  Recovered invoices take k_b11_rec_prep, the plain-flow ladder k_main<SV_KIND_SCHNORR> (which parks the
// Jacobian result) and k_b11_rec_final.  k_b11_status folds both into one int and one key per invoice.
extern "C" int sv_verify_bolt11_host(sv_ctx* ctx, const uint8_t* blob, size_t blob_len, const uint64_t* off,
                                     const uint32_t* len, size_t n, int* status, uint8_t* node_id33_out,
                                     uint8_t* hash32_out) {
    if (!ctx || (n && (!blob || !off || !len || !status || !node_id33_out))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    rc = stage_spans(ctx, blob, blob_len, off, len, n);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    size_t scan_bytes = 0;
    CK(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, (const u32*)nullptr, (u64*)nullptr, cuda::std::plus<>{}, (u64)0,
                                      n + 1, st));
    // per-call scratch in the auxiliary slab.  Per invoice: flags (one more, 0), their exclusive prefix sums in 64 bits
    // (one more, the total), recovery id, `n` key, status and key out.  Packed: the `n` invoices' message / key /
    // signature, the recovered invoices' R.x, status and key.  The scan's scratch.
    slab_layout L;
    const size_t o_isn = L.take(4 * (n + 1)), o_bn = L.take(8 * (n + 1)), o_isr = L.take(4 * (n + 1)),
                 o_br = L.take(8 * (n + 1)), o_recid = L.take(n), o_key = L.take(33 * n), o_status = L.take(4 * n),
                 o_node = L.take(33 * n), o_cmsg = L.take(32 * n), o_ckey = L.take(33 * n), o_csig = L.take(64 * n),
                 o_x = L.take(32 * n), o_rstat = L.take(4 * n), o_rkey = L.take(33 * n), o_scan = L.take(scan_bytes);
    rc = ensure_gbuf(ctx, L.size);
    if (rc) return rc;
    const dev_buf<>& G = ctx->g_buf;
    u32 *is_n = G.at<u32>(o_isn), *is_r = G.at<u32>(o_isr);
    u64 *base_n = G.at<u64>(o_bn), *base_r = G.at<u64>(o_br);
    int *d_status = G.at<int>(o_status), *rstat = G.at<int>(o_rstat);
    u8 *recid = G + o_recid, *key33 = G + o_key, *node = G + o_node, *cmsg = G + o_cmsg, *ckey = G + o_ckey,
       *csig = G + o_csig, *x32 = G + o_x, *rkey = G + o_rkey;
    const unsigned g128 = (unsigned)((n + 127) / 128);
    CK(cudaMemsetAsync(is_n + n, 0, 4, st));
    CK(cudaMemsetAsync(is_r + n, 0, 4, st));
    CK(mark(ctx, MK_B11_PARSE, st));
    k_b11_parse<<<g128, 128, 0, st>>>(ctx->d_data, ctx->d_off, ctx->d_len, n, ctx->d_msg, key33, ctx->d_sig, recid, is_n, is_r);
    CK(cub::DeviceScan::ExclusiveScan(G + o_scan, scan_bytes, is_n, base_n, cuda::std::plus<>{}, (u64)0, n + 1, st));
    CK(cub::DeviceScan::ExclusiveScan(G + o_scan, scan_bytes, is_r, base_r, cuda::std::plus<>{}, (u64)0, n + 1, st));
    k_b11_gather_n<<<g128, 128, 0, st>>>(is_n, base_n, n, ctx->d_msg, key33, ctx->d_sig, cmsg, ckey, csig);
    ctx->launches += 2;
    CK(mark(ctx, MK_B11_PACKED, st));
    CK(cudaGetLastError());
    u64 cnt[2] = {0, 0};
    CK(cudaMemcpyAsync(&cnt[0], base_n + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&cnt[1], base_r + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(mark(ctx, MK_B11_CURVE, st));
    rc = launch_verify(ctx, SV_KIND_ECDSA33, cmsg, ckey, csig, (size_t)cnt[0], ctx->d_verdict, nullptr, st);
    if (rc) return rc;
    const size_t cr = (size_t)cnt[1];
    if (cr) {
        sv_ctx::slot_t* sl = nullptr;
        rc = acquire_slot(ctx, cr, st, &sl);
        if (rc) return rc;
        apply_l2_policy(ctx, st, sl->d_scratch);
        k_b11_rec_prep<<<g128, 128, 0, st>>>(is_r, base_r, n, ctx->d_msg, ctx->d_sig, recid, x32, sl->d_work);
        // the plain BIP-340 curve kernel computes u1 G + u2 E for the x-only key E and parks it; it reads no signature
        // and writes no verdict for this kind
        k_main<SV_KIND_SCHNORR><<<main_grid_for(ctx, cr), SV_MAIN_BLOCK, 0, st>>>(sl->d_work, x32, csig, cr, ctx->d_gtab,
                                                                                   sl->d_scratch, nullptr, nullptr);
        const size_t threads = (cr + SV_FINAL_BATCH - 1) / SV_FINAL_BATCH;
        k_b11_rec_final<<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(sl->d_work, cr, rstat, rkey);
        ctx->launches += 3;
        CK(cudaGetLastError());
        rc = release_slot(ctx, sl, st);
        if (rc) return rc;
    }
    k_b11_status<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(is_n, base_n, is_r, base_r, n, recid, key33, ctx->d_verdict,
                                                             rstat, rkey, d_status, node);
    ctx->launches += 1;
    CK(mark(ctx, MK_B11_DONE, st));
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(status, d_status, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(node_id33_out, node, 33 * n, cudaMemcpyDeviceToHost, st));
    if (hash32_out) CK(cudaMemcpyAsync(hash32_out, ctx->d_msg, 32 * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ctx->profiling) {
        CK(mark_ms(ctx, MK_B11_PARSE, MK_B11_PACKED, &ctx->b11_ms[0]));
        CK(mark_ms(ctx, MK_B11_CURVE, MK_B11_DONE, &ctx->b11_ms[1]));
    }
    return SV_OK;
}

// ---- BIP-340 batch verification, host entry (batch.cuh) --------------------------------------------------------------
#include <sys/random.h>
extern "C" int sv_verify_schnorr_batch_host(sv_ctx* ctx, const uint8_t* msg32, const uint8_t* xonly32, const uint8_t* sig64,
                                            size_t n, const uint8_t* seed32, uint8_t* verdicts, uint32_t* groups_total,
                                            uint32_t* groups_failed) {
    if (!ctx || (n && (!msg32 || !xonly32 || !sig64 || !verdicts))) return SV_ERR_ARG;
    if (groups_total) *groups_total = 0;
    if (groups_failed) *groups_failed = 0;
    if (n == 0) return SV_OK;
    if (n > 0x7FFFFFFFu) return SV_ERR_ARG;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    uint8_t seed[32];
    if (seed32) memcpy(seed, seed32, 32);
    else if (getrandom(seed, 32, 0) != 32) return fail(ctx, SV_ERR_ARG, "getrandom", cudaSuccess);
    int rc = ensure_staging(ctx, n);
    if (rc) return rc;
    const u32 groups = (u32)((n + SV_SB_GROUP - 1) / SV_SB_GROUP);
    // scratch: [seed 32][pts 2n x 96][t n x 32][S groups x W x 128][dig W x 4n][ok n][group_ok groups][out n][idx n x 4]
    slab_layout L;
    const size_t o_seed = L.take(32), o_pts = L.take(2 * n * sizeof(qtab_entry), 64), o_t = L.take(n * sizeof(sc)),
                 o_S = L.take((size_t)groups * SV_SB_WINDOWS * sizeof(sv_jac)), o_dig = L.take((size_t)SV_SB_WINDOWS * 4 * n),
                 o_ok = L.take(n), o_gok = L.take(groups), o_out = L.take(n), o_idx = L.take(4 * n);
    rc = ctx->dd_buf.reserve(ctx, L.size + 64, SV_SCRATCH_FLOOR);
    if (rc) return rc;
    const dev_buf<>& B = ctx->dd_buf;
    u8* d_seed = B + o_seed;
    qtab_entry* d_pts = B.at<qtab_entry>(o_pts);
    sc* d_t = B.at<sc>(o_t);
    sv_jac* d_S = B.at<sv_jac>(o_S);
    signed char* d_dig = B.at<signed char>(o_dig);
    u8 *d_ok = B + o_ok, *d_gok = B + o_gok, *d_out = B + o_out;
    u32* d_idx = B.at<u32>(o_idx);
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(d_seed, seed, 32, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_msg, msg32, 32 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_key, xonly32, 32 * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_sig, sig64, 64 * n, cudaMemcpyHostToDevice, st));
    CK(mark(ctx, MK_PREP, st));
    if (sv_batch_launch(ctx->d_msg, ctx->d_key, ctx->d_sig, n, d_seed, d_pts, d_dig, d_t, d_ok, d_S, d_gok, d_out, ctx->d_gtab, st,
                        ctx->profiling ? ctx->mark_ev[MK_MAIN] : nullptr) != 0)
        return fail(ctx, SV_ERR_CUDA, "batch kernels", cudaGetLastError());
    CK(mark(ctx, MK_END, st));
    ctx->launches += 4;
    std::vector<u8> gok(groups), ok(n);
    CK(cudaMemcpyAsync(gok.data(), d_gok, groups, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ok.data(), d_ok, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // members of failed groups (whose encoding is fine) go through one-by-one verification; their verdicts replace the zeros
    std::vector<u32> idx;
    u32 failed = 0;
    for (u32 g = 0; g < groups; g++) {
        if (gok[g]) continue;
        failed++;
        size_t lo = (size_t)g * SV_SB_GROUP, hi = lo + SV_SB_GROUP < n ? lo + SV_SB_GROUP : n;
        for (size_t i = lo; i < hi; i++)
            if (ok[i]) idx.push_back((u32)i);
    }
    if (groups_total) *groups_total = groups;
    if (groups_failed) *groups_failed = failed;
    if (!idx.empty()) {
        size_t c = idx.size();
        CK(cudaMemcpyAsync(d_idx, idx.data(), 4 * c, cudaMemcpyHostToDevice, st));
        // gathered copies live in the upper halves... of a second staging area: the pts array is dead by now (2n x 96 bytes >= 160 c)
        u8* g_msg = reinterpret_cast<u8*>(d_pts);
        u8* g_key = g_msg + 32 * c;
        u8* g_sig = g_key + 32 * c;
        u8* g_v = g_sig + 64 * c;
        k_sb_gather<<<(unsigned)((c + 255) / 256), 256, 0, st>>>(d_idx, c, ctx->d_msg, ctx->d_key, ctx->d_sig, g_msg, g_key, g_sig);
        ctx->launches += 1;
        rc = launch_verify(ctx, SV_KIND_SCHNORR, g_msg, g_key, g_sig, c, g_v, nullptr, st);
        if (rc) return rc;
        k_mixed_scatter<<<(unsigned)((c + 255) / 256), 256, 0, st>>>(d_idx, c, g_v, d_out);
        ctx->launches += 1;
        CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(verdicts, d_out, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}

// ---- deferral queue -----------------------------------------------------------------------------
extern "C" long sv_enqueue(sv_ctx* ctx, int kind, const uint8_t msg32[32], const uint8_t* key, const uint8_t sig64[64]) {
    size_t ks = sv_key_size(kind);
    if (!ctx || ks == 0 || !msg32 || !key || !sig64) return SV_ERR_ARG;
    sv_queue_item it;
    it.kind = kind;
    memcpy(it.msg, msg32, 32);
    memset(it.key, 0, 64);
    memcpy(it.key, key, ks);
    memcpy(it.sig, sig64, 64);
    ctx->queue.push_back(it);
    return (long)ctx->queue.size() - 1;
}
extern "C" size_t sv_pending(const sv_ctx* ctx) { return ctx ? ctx->queue.size() : 0; }

extern "C" int sv_flush(sv_ctx* ctx, uint8_t* verdicts, size_t capacity) {
    if (!ctx || (!verdicts && !ctx->queue.empty())) return SV_ERR_ARG;
    size_t total = ctx->queue.size();
    if (capacity < total) return SV_ERR_ARG;
    // segregate by kind so that warps stay homogeneous, verify, scatter verdicts back in enqueue order
    for (int kind = 0; kind < 3; kind++) {
        size_t ks = sv_key_size(kind);
        std::vector<size_t> idx;
        for (size_t i = 0; i < total; i++)
            if (ctx->queue[i].kind == kind) idx.push_back(i);
        if (idx.empty()) continue;
        size_t m = idx.size();
        std::vector<u8> msg(32 * m), key(ks * m), sig(64 * m), out(m);
        for (size_t j = 0; j < m; j++) {
            const sv_queue_item& it = ctx->queue[idx[j]];
            memcpy(&msg[32 * j], it.msg, 32);
            memcpy(&key[ks * j], it.key, ks);
            memcpy(&sig[64 * j], it.sig, 64);
        }
        int rc = sv_verify_host(ctx, kind, msg.data(), key.data(), sig.data(), m, out.data());
        if (rc) return rc;
        for (size_t j = 0; j < m; j++) verdicts[idx[j]] = out[j];
    }
    ctx->queue.clear();
    return SV_OK;
}

// ---- self test (test support) ---------------------------------------------------------------------
extern "C" int sv_selftest_host(sv_ctx* ctx, int op, const uint32_t* a, const uint32_t* b, size_t n, uint32_t* out) {
    if (!ctx || op < 0 || op > SV_ST_FE_INV_VAR || (n && (!a || !b || !out))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    dev_buf<u32> ta, tb, to;
    int rc = ta.reserve(ctx, n * 32, n * 32);
    if (!rc) rc = tb.reserve(ctx, n * 32, n * 32);
    if (!rc) rc = to.reserve(ctx, n * 64, n * 64);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ta, a, n * 32, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(tb, b, n * 32, cudaMemcpyHostToDevice, st));
    k_selftest<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(op, ta, tb, n, to, ctx->d_gtab);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, to, n * 64, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}
extern "C" int sv_selftest_group_host(sv_ctx* ctx, int op, const uint32_t* in, size_t n, uint32_t* out) {
    if (!ctx || op < 0 || op > SV_STG_NS_LINEAR_FORM || (n && (!in || !out))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    const size_t ib = n * 4 * SV_STG_IN_WORDS, ob = n * 4 * SV_STG_OUT_WORDS;
    dev_buf<u32> ti, to;
    int rc = ti.reserve(ctx, ib, ib);
    if (!rc) rc = to.reserve(ctx, ob, ob);
    if (rc) return rc;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ti, in, ib, cudaMemcpyHostToDevice, st));
    k_selftest_group<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(op, ti, n, to, ctx->d_gtab);
    ctx->launches += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, to, ob, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SV_OK;
}

// ---- synthetic workload + probes ----------------------------------------------------------------
extern "C" int sv_synth_device(sv_ctx* ctx, int kind, uint64_t seed, size_t n, void* d_msg32, void* d_key,
                               void* d_sig64, void* stream) {
    if (!ctx || sv_key_size(kind) == 0 || (n && (!d_msg32 || !d_key || !d_sig64))) return SV_ERR_ARG;
    if (n == 0) return SV_OK;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    unsigned grid = (unsigned)((n + 127) / 128);
    if (kind == SV_KIND_ECDSA33)
        k_synth<SV_KIND_ECDSA33><<<grid, 128, 0, st>>>(seed, n, ctx->d_gtab, (u8*)d_msg32, (u8*)d_key, (u8*)d_sig64);
    else if (kind == SV_KIND_ECDSA_XY)
        k_synth<SV_KIND_ECDSA_XY><<<grid, 128, 0, st>>>(seed, n, ctx->d_gtab, (u8*)d_msg32, (u8*)d_key, (u8*)d_sig64);
    else
        k_synth<SV_KIND_SCHNORR><<<grid, 128, 0, st>>>(seed, n, ctx->d_gtab, (u8*)d_msg32, (u8*)d_key, (u8*)d_sig64);
    ctx->launches += 1;
    CK(cudaGetLastError());
    return SV_OK;
}

extern "C" int sv_probe(sv_ctx* ctx, int mode, double* ops_per_sec) {
    if (!ctx || !ops_per_sec || mode < 0 || mode > 10) return SV_ERR_ARG;
    dev_guard dg__;
    CK(dg__.enter(ctx->device));
    const int iters = (mode == 2 || mode == 3 || mode >= 9) ? 2000 : 4000;
    // modes 9/10: ONE warp on the whole device — the dependent-chain latency of fe_mul / fe_sqr (small-batch path)
    const int blocks = mode >= 9 ? 1 : ctx->sm_count * 8, threads = mode >= 9 ? 32 : 256;
    // the probe's own events, destroyed on every exit path
    using event_ptr = std::unique_ptr<CUevent_st, cudaError_t (*)(cudaEvent_t)>;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CK(cudaEventCreate(&e0));
    event_ptr own0(e0, cudaEventDestroy);
    CK(cudaEventCreate(&e1));
    event_ptr own1(e1, cudaEventDestroy);
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
        CK(cudaEventRecord(e0, ctx->stream));
        switch (mode) {
            case 0: k_probe_imad_wide<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 1: k_probe_cmad4<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 2: k_probe_fe<0><<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 3: k_probe_fe<1><<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 4: k_probe_chain8<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 5: k_probe_carry_save<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 6: k_probe_imad32<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 8: k_probe_dfma<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 9: k_probe_fe<0><<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            case 10: k_probe_fe<1><<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
            default: k_probe_addc<<<blocks, threads, 0, ctx->stream>>>(iters, ctx->d_sink); break;
        }
        CK(cudaEventRecord(e1, ctx->stream));
        CK(cudaEventSynchronize(e1));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep > 0 && ms < best) best = ms;
        ctx->launches += 1;
    }
    // operations per thread per launch
    static const double per_iter[11] = {32.0, 32.0, 2.0, 2.0, 32.0, 32.0, 32.0, 64.0, 32.0, 2.0, 1.0};  // mode 10: two INDEPENDENT squaring chains -> one chain's rate
    // modes 9/10 report dependent operations per second of ONE thread (the two chains of the probe depend on each other)
    *ops_per_sec = per_iter[mode] * iters * (mode >= 9 ? 1.0 : (double)blocks * threads) / (best * 1e-3);
    return SV_OK;
}
extern "C" int sv_probe_imad_peak(sv_ctx* ctx, double* imad_per_sec) { return sv_probe(ctx, 0, imad_per_sec); }

// pinned host memory for callers that want full-speed H2D/D2H
extern "C" void* sv_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void sv_host_free(void* p) {
    if (p) cudaFreeHost(p);
}
