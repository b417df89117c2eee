// common.cuh — shared macros for the sm_90a secp256k1 verification engine.
//
// All arithmetic above the 256-bit primitives in u256.cuh is written as portable C++ marked
// SV_HD.  On the device the primitives are inline-PTX carry chains that ptxas fuses into
// IMAD.WIDE.U32(.X); when the same headers are compiled by g++ (tests/host_emul only — a
// developer aid that lets the kernel source be unit-tested without a GPU, never linked into
// the product library) they fall back to uint64_t arithmetic.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
// under nvcc everything is device-only: the product has NO host implementation of the maths
#define SV_HD __device__ __forceinline__
#define SV_D __device__ __forceinline__
#define SV_HD_NOINLINE __device__ __noinline__
#else
#define SV_HD static inline
#define SV_D static inline
#define SV_HD_NOINLINE static
#endif

// all SV_HD functions are __device__-only under nvcc, so the PTX path is selected by the compiler,
// not by the compilation pass (nvcc's host pass merely parses these bodies)
#if defined(__CUDACC__)
#define SV_DEVICE_CODE 1
#define SV_UNROLL _Pragma("unroll")
#else
#define SV_DEVICE_CODE 0
#define SV_UNROLL
#endif

// Constant tables live in __constant__ memory on the device; accesses with compile-time indices
// (the arithmetic is fully unrolled) become immediates / uniform-register loads.
#if defined(__CUDACC__)
#define SV_CDATA __device__ __constant__
#else
#define SV_CDATA
#endif

// CTA-wide re-convergence points of the curve-side kernel (only in the SV_MAIN_SYNC build, where the
// field arithmetic is inlined and the warps of a CTA are kept at the same PC to share instruction fetches)
#if defined(__CUDACC__) && defined(SV_MAIN_SYNC)
// n = number of threads taking part (the whole CTA) or 0: no barrier (callers that run in ONE warp of a larger CTA — the
// small-batch kernel — must not hit CTA-wide barriers)
#define SV_SYNC(n) do { if (n) __syncthreads(); } while (0)
#else
#define SV_SYNC(n) ((void)(n))
#endif

typedef uint32_t u32;
typedef uint64_t u64;
typedef uint8_t u8;
