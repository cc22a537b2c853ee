// common.cuh -- shared helpers for libnats_b200 (sm_90a).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>

#include <utility>

#include "../../include/nats_b200.h"
#include "prof.cuh"

namespace nats {

// ------------------------------------------------------------------ error handling
void set_error(const char* fmt, ...);

#define NATS_CUDA_OK(expr)                                                                   \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            nats::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return 1;                                                                        \
        }                                                                                    \
    } while (0)

#define NATS_LAUNCH_OK()                                                                     \
    do {                                                                                     \
        cudaError_t _e = cudaPeekAtLastError();                                              \
        if (_e != cudaSuccess) {                                                             \
            nats::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
            return 1;                                                                        \
        }                                                                                    \
    } while (0)

#define NATS_TRY(expr)                \
    do {                              \
        int _r = (expr);              \
        if (_r != 0) return _r;       \
    } while (0)

#define NATS_REQUIRE(cond, msg)                                                \
    do {                                                                       \
        if (!(cond)) {                                                         \
            nats::set_error("%s:%d: requirement failed: %s (%s)", __FILE__, __LINE__, #cond, msg); \
            return 2;                                                          \
        }                                                                      \
    } while (0)

}  // namespace nats

struct nats_ctx {
    int device;
    int num_sms;
    int max_smem_optin;
    float* dev_scratch;          // small stream-ordered reduction scratch (kCtxScratchFloats)
};
constexpr int kCtxScratchFloats = 16384;

namespace nats {

int pdl_enabled();
void pdl_set(int on);

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up64(int64_t a, int64_t b) { return cdiv64(a, b) * b; }

// ------------------------------------------------------------------ device math
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide reductions (blockDim.x multiple of 32, <= 1024).  `red` = 32 floats of shared memory.
// All threads receive the result.  Contains __syncthreads(): call from uniform control flow.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : 0.0f;
    return warp_sum(r);
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = (lane < nw) ? red[lane] : -INFINITY;
    return warp_max(r);
}

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// A kernel launched through launch_pdl() may start while its predecessor in the stream is still running: it calls
// pdl_trigger() as early as possible (lets ITS dependents launch) and pdl_wait() before the first access to memory that
// a predecessor may have written or may still read.  Kernels without the attribute keep the ordinary stream order.
// sum_{k<n} p[k*stride] in ascending order, eight loads in flight at a time.  (A runtime-trip-count loop of load+add
// pairs costs one memory round trip per term: the in-order pipeline stalls on every add.)
__device__ __forceinline__ float sum_strided(const float* __restrict__ p, long long stride, int n, float acc = 0.f) {
    for (int k0 = 0; k0 < n; k0 += 8) {
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = (k0 + k < n) ? p[(long long)(k0 + k) * stride] : 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k0 + k < n) acc += v[k];
    }
    return acc;
}
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// streaming (read-once) 128-bit load that does not pollute L1
// L2 eviction policy for the encoder context `cc` (102 MB at config 3, re-streamed by every decoder step): a fraction of
// its lines is marked evict_last so that it survives in the 126 MB L2 from one pass to the next.  mode: 0 none, 1..4 = 25..100 %
__device__ __forceinline__ unsigned long long l2_keep_policy(int mode) {
    unsigned long long pol = 0;
    if (mode == 1) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 0.25;" : "=l"(pol));
    else if (mode == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 0.5;" : "=l"(pol));
    else if (mode == 3) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 0.75;" : "=l"(pol));
    else if (mode == 4) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ float4 ldg_stream4_hint(const float* p, unsigned long long pol) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

}  // namespace nats
