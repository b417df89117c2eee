// batch.cu — kernels of the BIP-340 batch verification (batch.cuh), a translation unit of their own so that they can be
// compiled with fe_mul / fe_sqr as REAL FUNCTIONS (no -DSV_FE_INLINE): the bucket loop is one mixed addition executed ~100
// times per lane by warps at unrelated program counters; fully inlined it is ~50 KB of straight-line code per iteration
// against a 32 KB instruction cache (the curve kernel shows exactly this effect, see
// engine.cu).  As calls, the two multiplier bodies stay cache resident.
#include <cuda_runtime.h>
#include "batch.cuh"

__global__ void __launch_bounds__(128) k_sb_prep(const u8* __restrict__ msg, const u8* __restrict__ xonly, const u8* __restrict__ sig,
                                                 size_t n, const u8* __restrict__ seed32, qtab_entry* pts, signed char* dig, sc* t,
                                                 u8* ok) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    sc ti;
    bool good = sb_prepare(msg + 32 * i, xonly + 32 * i, sig + 64 * i, seed32, (u64)i, pts + 2 * i, dig + 4 * i, 4 * n, ti);
    t[i] = ti;
    ok[i] = good ? 1 : 0;
}
// one WARP per (group, window): counting sort of the group's digit row into 32 bucket lists (shared memory), lane b sums
// its bucket with mixed additions, then sum_b (b+1) B_b by a suffix scan + tree reduction through shared memory
#define SV_SB_WARPS 2
__global__ void __launch_bounds__(32 * SV_SB_WARPS) k_sb_window(const qtab_entry* __restrict__ pts, const signed char* __restrict__ dig,
                                                              size_t n, u32 groups, sv_jac* S) {
    __shared__ unsigned short list[SV_SB_WARPS][SV_SB_TERMS * SV_SB_GROUP];
    __shared__ u32 cnt[SV_SB_WARPS][32], fill[SV_SB_WARPS][32], offs[SV_SB_WARPS][32];
    __shared__ sv_jac xch[SV_SB_WARPS][32];
    const int wid = threadIdx.x >> 5, b = threadIdx.x & 31;
    const u32 job = blockIdx.x * SV_SB_WARPS + wid;
    if (job >= groups * SV_SB_WINDOWS) return;  // whole warps leave together
    const u32 g = job / SV_SB_WINDOWS, w = job % SV_SB_WINDOWS;
    const size_t first = (size_t)g * SV_SB_GROUP;
    const u32 members = (u32)((n - first < SV_SB_GROUP) ? (n - first) : SV_SB_GROUP);
    const u32 entries = members * SV_SB_TERMS;
    const signed char* row = dig + (size_t)w * 4 * n + 4 * first;
    cnt[wid][b] = 0;
    fill[wid][b] = 0;
    __syncwarp();
    for (u32 e = b; e < entries; e += 32) {
        int d = row[e];
        if (d) atomicAdd(&cnt[wid][(d < 0 ? -d : d) - 1], 1u);
    }
    __syncwarp();
    u32 mine = cnt[wid][b], off = mine;
    for (int k = 1; k < 32; k <<= 1) {  // inclusive prefix sum over the lanes
        u32 v = __shfl_up_sync(0xFFFFFFFFu, off, k);
        if (b >= k) off += v;
    }
    off -= mine;           // first list slot of bucket b
    offs[wid][b] = off;
    __syncwarp();
    for (u32 e = b; e < entries; e += 32) {
        int d = row[e];
        if (d) {
            int bk = (d < 0 ? -d : d) - 1;
            u32 pos = atomicAdd(&fill[wid][bk], 1u);
            list[wid][offs[wid][bk] + pos] = (unsigned short)(e | (d < 0 ? 0x8000u : 0u));
        }
    }
    __syncwarp();
    const qtab_entry* gp = pts + 2 * first;
    gej acc;
    acc.inf = 1;
    fe_set_zero(acc.x); fe_set_zero(acc.y); fe_set_zero(acc.z);
#pragma unroll 1
    for (u32 k = 0; k < mine; k++) {
        unsigned short ent = list[wid][off + k];
        ge p;
        sb_fetch(p, gp, ent & 0x7FFFu, (ent & 0x8000u) != 0);
        gej_add_ge(acc, acc, p);
    }
    // suffix scan: acc_b <- sum_{j >= b} B_j
#pragma unroll 1
    for (int k = 1; k < 32; k <<= 1) {
        small_jac_store(&xch[wid][b], acc);
        __syncwarp();
        if (b + k < 32) {
            gej T;
            small_jac_load(T, &xch[wid][b + k]);
            gej_add_gej(acc, acc, T);
        }
        __syncwarp();
    }
    // tree reduction of the 32 suffix sums: sum_b suffix_b = sum_j (j+1) B_j
#pragma unroll 1
    for (int k = 16; k >= 1; k >>= 1) {
        small_jac_store(&xch[wid][b], acc);
        __syncwarp();
        if (b < k) {
            gej T;
            small_jac_load(T, &xch[wid][b + k]);
            gej_add_gej(acc, acc, T);
        }
        __syncwarp();
    }
    if (b == 0) small_jac_store(&S[(size_t)g * SV_SB_WINDOWS + w], acc);
}
__global__ void __launch_bounds__(64) k_sb_final(const sv_jac* S, const sc* t, size_t n, u32 groups, const ge_mem* gtab, u8* group_ok) {
    u32 g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= groups) return;
    size_t first = (size_t)g * SV_SB_GROUP;
    u32 members = (u32)((n - first < SV_SB_GROUP) ? (n - first) : SV_SB_GROUP);
    group_ok[g] = sb_group_check(S + (size_t)g * SV_SB_WINDOWS, t + first, members, gtab) ? 1 : 0;
}
// verdict = encoding ok AND the group's equation held; members of failed groups are re-verified one by one afterwards
__global__ void k_sb_verdicts(const u8* ok, const u8* group_ok, size_t n, u8* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (ok[i] && group_ok[i / SV_SB_GROUP]) ? 1 : 0;
}

extern "C" int sv_batch_launch(const u8* d_msg, const u8* d_key, const u8* d_sig, size_t n, const u8* d_seed, void* d_pts,
                               signed char* d_dig, void* d_t, u8* d_ok, void* d_S, u8* d_gok, u8* d_out, const void* d_gtab,
                               cudaStream_t st, cudaEvent_t ev_mid) {
    const u32 groups = (u32)((n + SV_SB_GROUP - 1) / SV_SB_GROUP);
    k_sb_prep<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_msg, d_key, d_sig, n, d_seed, (qtab_entry*)d_pts, d_dig, (sc*)d_t, d_ok);
    if (ev_mid && cudaEventRecord(ev_mid, st) != cudaSuccess) return -1;
    u32 jobs = groups * SV_SB_WINDOWS;
    k_sb_window<<<(jobs + SV_SB_WARPS - 1) / SV_SB_WARPS, 32 * SV_SB_WARPS, 0, st>>>((const qtab_entry*)d_pts, d_dig, n, groups, (sv_jac*)d_S);
    k_sb_final<<<(groups + 63) / 64, 64, 0, st>>>((const sv_jac*)d_S, (const sc*)d_t, n, groups, (const ge_mem*)d_gtab, d_gok);
    k_sb_verdicts<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ok, d_gok, n, d_out);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
