// tma_gemm.cu -- 3xTF32 GEMM on wgmma fed by the Tensor Memory Accelerator, and the host side of TMA (tensor maps).
//
//   Thread 0 keeps a ring of NR raw stages filled with cp.async.bulk.tensor boxes of 32 k x rows of both operands,
//   straight from the caller's layout (K-contiguous or row-contiguous sources: no transposed copies are ever made).
//   The 256 threads (two warpgroups, rows 64w..64w+63 of the 128-row tile) split the next raw stage into tf32 {hi, lo}
//   K-major SWIZZLE_128B tiles (the only layout tf32 wgmma reads) while the tensor cores work on the current one:
//       D += A_hi.B_hi (two alternating accumulators),   D += A_lo.B_hi + A_hi.B_lo (a third).
//   Skinny products (the batch, <= 64, on the N side; NATS_TS=1, the default): the 128-row operand (the weights) is NOT
//   split into shared memory -- each thread reads its wgmma A fragments straight from the raw stage, splits them in
//   registers and issues the register-A form, so only the small B operand goes through the split pass.
//   Wider products (N side > 64) run on tma_gemm_kernel_ws below: warp-specialized, persistent, 128 x 96 / 128 x 112 tiles.
// Requirements: 16-byte aligned base pointers and leading dimensions that are multiples of 4 floats (TMA strides);
// anything else is served by the software-loader kernel in tc_gemm.cu.
#include <cuda.h>

#include <unordered_map>

#include "gemm.cuh"
#include "ops.cuh"
#include "tc_common.cuh"

namespace nats {

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

struct MapKey {
    const void* ptr; long long inner, outer, ld, batch, bstride; int box_outer; int mn;
    bool operator==(const MapKey& o) const {
        return ptr == o.ptr && inner == o.inner && outer == o.outer && ld == o.ld && batch == o.batch &&
               bstride == o.bstride && box_outer == o.box_outer && mn == o.mn;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = std::hash<const void*>()(k.ptr);
        auto mix = [&](long long v) { h ^= std::hash<long long>()(v) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.inner); mix(k.outer); mix(k.ld); mix(k.batch); mix(k.bstride); mix(k.box_outer); mix(k.mn);
        return h;
    }
};
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;


constexpr int kThreads = 256;
constexpr int kBlockK = 32;
constexpr int kNR = 3;                  // raw stages in flight
constexpr int kMaxGroup = 2;

struct TmaProblem {
    float* C;
    const float* bias;
    int Ma, Nb, K;
    long long c_rs, c_cs;
    int batch;
    long long sC;
    int splitk, kchunk;
    long long strideP;
    int accumulate;
    int bias_on_a;
};
struct alignas(64) TmaGroup {
    CUtensorMap mapA[kMaxGroup];
    CUtensorMap mapB[kMaxGroup];
    TmaProblem p[kMaxGroup];
    int zstart[kMaxGroup + 1];
    int istart[kMaxGroup + 1];          // first work item of each problem (tma_gemm_kernel_ws)
    int count;
};

using namespace tc;

// raw stage of an operand: ROWS x 32 fp32 as TMA wrote it: K-major [ROWS][32] or MN-major [32][ROWS] (unswizzled)
template <int ROWS, bool MN>
__device__ __forceinline__ float raw_at(uint32_t raw, int r, int k) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(raw + 4u * (uint32_t)(MN ? k * ROWS + r : r * 32 + k)));
    return v;
}

// raw stage -> {hi, lo} K-major SWIZZLE_128B tiles (16-byte chunk c of row r at chunk c ^ (r & 7)); k >= klim reads as 0
template <int ROWS, bool MN, int NT = kThreads>
__device__ __forceinline__ void split_tile(uint32_t raw, uint32_t hi_base, uint32_t lo_base, int klim, int tid) {
    constexpr int kChunks = ROWS * 8;
#pragma unroll
    for (int i = 0; i < (kChunks + NT - 1) / NT; ++i) {
        const int q = tid + i * NT;
        if (q < kChunks) {
            int r, c;
            float4 v;
            if (!MN) {
                r = q >> 3; c = q & 7;
                asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                             : "r"(raw + 4u * (uint32_t)(r * 32 + 4 * c)));
            } else {                                          // a warp covers 32 consecutive rows: conflict-free reads
                r = q % ROWS; c = q / ROWS;
                v.x = raw_at<ROWS, true>(raw, r, 4 * c); v.y = raw_at<ROWS, true>(raw, r, 4 * c + 1);
                v.z = raw_at<ROWS, true>(raw, r, 4 * c + 2); v.w = raw_at<ROWS, true>(raw, r, 4 * c + 3);
            }
            if (4 * c >= klim) v.x = 0.f;
            if (4 * c + 1 >= klim) v.y = 0.f;
            if (4 * c + 2 >= klim) v.z = 0.f;
            if (4 * c + 3 >= klim) v.w = 0.f;
            float4 hi, lo;
            hi.x = to_tf32(v.x); hi.y = to_tf32(v.y); hi.z = to_tf32(v.z); hi.w = to_tf32(v.w);
            lo.x = to_tf32(v.x - hi.x); lo.y = to_tf32(v.y - hi.y); lo.z = to_tf32(v.z - hi.z); lo.w = to_tf32(v.w - hi.w);
            const uint32_t off = (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
            st_shared_v4(hi_base + off, hi);
            st_shared_v4(lo_base + off, lo);
        }
    }
}

template <int BN>
__device__ __forceinline__ void mma_ss(float (&d)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 32) wgmma_ss_n32(d, da, db);
    else wgmma_ss_n64(d, da, db);
}
template <int BN>
__device__ __forceinline__ void mma_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t db) {
    if constexpr (BN == 32) wgmma_rs_n32(d, a, db);
    else wgmma_rs_n64(d, a, db);
}

template <int BN, bool A_MN, bool B_MN, bool A_REG>
__global__ void __launch_bounds__(kThreads, 1) tma_gemm_kernel(const __grid_constant__ TmaGroup grp) {
    constexpr uint32_t kARaw = 128 * 128, kBRaw = BN * 128;
    constexpr uint32_t kRawStage = kARaw + kBRaw;
    constexpr uint32_t kAHalf = A_REG ? 0 : 128 * 128;              // A hi / lo tiles (none when A goes through registers)
    constexpr uint32_t kSplitStage = 2 * kAHalf + 2 * kBRaw;
    constexpr uint32_t kSplitBase = kNR * kRawStage;
    constexpr int R = BN / 2;
    static_assert(BN == 32 || BN == 64, "BN");

    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ __align__(8) uint64_t full[kNR];

    int z = blockIdx.z, g = 0;
    if (grp.count > 1 && z >= grp.zstart[1]) g = 1;
    const TmaProblem& P = grp.p[g];
    const CUtensorMap* mapA = &grp.mapA[g];
    const CUtensorMap* mapB = &grp.mapB[g];
    z -= grp.zstart[g];
    const int split = z % P.splitk, batch = z / P.splitk;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BN;
    if (m0 >= P.Ma || n0 >= P.Nb) return;

    const int kbeg = split * P.kchunk;
    const int kend = min(P.K, kbeg + P.kchunk);
    const int nkb = (kend > kbeg) ? (kend - kbeg + kBlockK - 1) / kBlockK : 0;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const uint32_t smem_base = (smem_u32(smem) + 1023u) & ~1023u;

    if (tid == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(mapB) : "memory");
        for (int s = 0; s < kNR; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();                          // operands and C may be written by the predecessor

    auto issue = [&](int kb) {           // thread 0: raw boxes of k-block kb into stage kb % kNR
        const int s = kb % kNR;
        const uint32_t raw = smem_base + (uint32_t)s * kRawStage;
        const int k0 = kbeg + kb * kBlockK;
        mbar_expect_tx(&full[s], kRawStage);
        if (A_MN) tma_load_3d(raw, mapA, &full[s], m0, k0, batch);
        else tma_load_3d(raw, mapA, &full[s], k0, m0, batch);
        if (B_MN) tma_load_3d(raw + kARaw, mapB, &full[s], n0, k0, batch);
        else tma_load_3d(raw + kARaw, mapB, &full[s], k0, n0, batch);
    };
    auto split_stage = [&](int kb) {     // raw stage of k-block kb -> split buffer kb & 1
        mbar_wait(&full[kb % kNR], (uint32_t)((kb / kNR) & 1));
        const uint32_t raw = smem_base + (uint32_t)(kb % kNR) * kRawStage;
        const uint32_t sp = smem_base + kSplitBase + (uint32_t)(kb & 1) * kSplitStage;
        const int klim = kend - (kbeg + kb * kBlockK);
        if (!A_REG) split_tile<128, A_MN>(raw, sp, sp + kAHalf, klim, tid);
        split_tile<BN, B_MN>(raw + kARaw, sp + 2 * kAHalf, sp + 2 * kAHalf + kBRaw, klim, tid);
    };

    float acc0[R], acc1[R], accx[R];
#pragma unroll
    for (int i = 0; i < R; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; accx[i] = 0.f; }
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);     // A fragment rows r0, r0 + 8 (register form)
    const int q = lane & 3;

    if (nkb > 0) {
        if (tid == 0)
            for (int kb = 0; kb < min(nkb, kNR); ++kb) issue(kb);
        split_stage(0);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
    __syncthreads();
    for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t sp = smem_base + kSplitBase + (uint32_t)(kb & 1) * kSplitStage;
        const uint64_t b_hi = desc_sw128(sp + 2 * kAHalf), b_lo = desc_sw128(sp + 2 * kAHalf + kBRaw);
        if constexpr (A_REG) {
            // A fragments of the 4 k-steps from the raw stage (full[] of this stage was waited on by split_stage)
            const uint32_t raw = smem_base + (uint32_t)(kb % kNR) * kRawStage;
            const int klim = kend - (kbeg + kb * kBlockK);
            uint32_t ahi[4][4], alo[4][4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                for (int f = 0; f < 4; ++f) {
                    const int r = r0 + 8 * (f & 1), k = 8 * kk + q + 4 * (f >> 1);
                    const float x = k < klim ? raw_at<128, A_MN>(raw, r, k) : 0.f;
                    const float h = to_tf32(x);
                    ahi[kk][f] = __float_as_uint(h);
                    alo[kk][f] = __float_as_uint(to_tf32(x - h));
                }
            }
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                mma_rs<BN>(accx, alo[kk], b_hi + 2 * kk);
                mma_rs<BN>(accx, ahi[kk], b_lo + 2 * kk);
                mma_rs<BN>((kk & 1) ? acc1 : acc0, ahi[kk], b_hi + 2 * kk);
            }
        } else {
            const uint64_t a_hi = desc_sw128(sp + (uint32_t)wg * 8192u), a_lo = desc_sw128(sp + kAHalf + (uint32_t)wg * 8192u);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                mma_ss<BN>(accx, a_lo + 2 * kk, b_hi + 2 * kk);
                mma_ss<BN>(accx, a_hi + 2 * kk, b_lo + 2 * kk);
                mma_ss<BN>((kk & 1) ? acc1 : acc0, a_hi + 2 * kk, b_hi + 2 * kk);
            }
        }
        wgmma_commit();
        if (kb + 1 < nkb) split_stage(kb + 1);    // the other split buffer was drained by the wait of the previous k-block
        wgmma_wait<0>();
        reg_fence(acc0); reg_fence(acc1); reg_fence(accx);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();                          // every thread is done with raw stage kb % kNR
        if (tid == 0 && kb + kNR < nkb) issue(kb + kNR);
    }

    const bool add_bias = (P.bias != nullptr) && (split == 0);
    gemm_epilogue(acc0, acc1, accx, P.C + (long long)batch * P.sC + (long long)split * P.strideP, P.c_rs, P.c_cs, P.Ma, P.Nb,
                  m0 + r0, n0 + 2 * q, (add_bias && P.bias_on_a) ? P.bias : nullptr,
                  (add_bias && !P.bias_on_a) ? P.bias : nullptr, P.accumulate != 0);
}

// ---------------------------------------------------------------------------------------------------------------
// Non-skinny products (N side > 64): warp-specialized, persistent 128 x BN tiles (BN = 112 when the N side fits in one,
// else 96: 1000 x 3000 takes 8 x 32 = 256 tiles, 1.94 waves of 132).
//   warp 0 (one lane)  TMA producer: kWsNR raw stages of 32 k x (128 A rows | BN B rows) in flight, in the caller's layout.
//                      Both boxes are 128-byte swizzled where the source is K-major; the MN-major A box is loaded as four
//                      swizzled 32-row boxes, so the consumers' fragment reads are (nearly) conflict-free.
//   warps 1-3          tf32 split of the B stage into a kWsNS-deep ring of K-major SWIZZLE_128B tiles.  The tensor core
//                      reads the upper 19 bits of an fp32 word, so the raw word is the hi operand and resid() the lo one:
//                      a K-major B box is already the wgmma layout and the raw stage is B_hi, only B_lo is written; an
//                      MN-major B box is transposed into a raw-word hi tile and a lo tile.
//   warpgroups 1, 2    consumers, rows 64 (wg - 1) .. + 63: read their A fragments from the raw stage (hi = the word,
//                      lo = its residual) and issue the register-A wgmma (m64nBNk8); one commit group per k-step, and
//                      ws_in_flight<BN>() of them outstanding while the next k-step's fragments are read.
// Stages are handed over by full / empty mbarrier pairs (no CTA barrier in the loop), so the producer and the split warps
// run ahead into the next tile while the consumers store the current one.  A consumer warpgroup frees a raw stage and its
// split tile once the last MMA that reads them has retired.  The producer warpgroup gives registers to the consumers
// (setmaxnreg 64 / 216), which hold the three accumulators of tma_gemm_kernel (3 x BN/2) beside the fragments of the
// k-steps in flight.  (At BN = 128 the three accumulators do not fit and ptxas serializes the wgmma; one accumulator for
// both A_hi.B_hi halves loses accuracy at deep K.)  Per element the sums are those of tma_gemm_kernel in the same order;
// only the split of each operand differs (truncated hi, exact residual lo instead of rounded hi and lo).
constexpr int kWsThreads = 384;
constexpr int kWsNR = 4, kWsNS = 3;
template <int BN> __host__ __device__ constexpr uint32_t ws_raw() { return 128 * 128 + BN * 128; }    // raw stage: A 16 KB | B
template <int BN, bool B_MN> __host__ __device__ constexpr uint32_t ws_split() { return (B_MN ? 2 : 1) * BN * 128; }
template <int BN, bool B_MN> constexpr size_t ws_smem() {
    return (size_t)kWsNR * ws_raw<BN>() + (size_t)kWsNS * ws_split<BN, B_MN>() + 1024;
}
// MMA k-steps a consumer warpgroup keeps outstanding.  The fragment registers form a ring of four sets indexed by the
// k-step of the k-block (register arrays need compile-time indices); only ws_in_flight + 1 of them are live at a time.
// At BN = 112 the accumulators take 168 registers and ptxas serializes the wgmma with a third live set: one in flight.
template <int BN> __host__ __device__ constexpr int ws_in_flight() { return BN == 96 ? 2 : 1; }

struct WsItem { int g, batch, split, m0, n0, kbeg, kend, nkb; };

template <int BN>
__device__ __forceinline__ WsItem ws_item(const TmaGroup& grp, int it) {
    WsItem w;
    w.g = (grp.count > 1 && it >= grp.istart[1]) ? 1 : 0;
    const TmaProblem& P = grp.p[w.g];
    it -= grp.istart[w.g];
    const int mt = (P.Ma + 127) >> 7, nt = (P.Nb + BN - 1) / BN;
    w.m0 = (it % mt) * 128; it /= mt;                    // m fastest: concurrent tiles share the B panels in L2
    w.n0 = (it % nt) * BN; it /= nt;
    w.split = it % P.splitk; w.batch = it / P.splitk;
    w.kbeg = w.split * P.kchunk;
    w.kend = min(P.K, w.kbeg + P.kchunk);
    w.nkb = (w.kend > w.kbeg) ? (w.kend - w.kbeg + kBlockK - 1) / kBlockK : 0;
    return w;
}

// element (r, k) of the raw A stage: K-major [128 rows][128 B] or MN-major 4 x [32 k][32 rows], 128-byte swizzled
template <bool MN>
__device__ __forceinline__ float raw_a_sw(uint32_t raw, int r, int k) {
    const uint32_t off = MN ? (uint32_t)((r >> 5) * 4096 + k * 128 + ((((r & 31) >> 2) ^ (k & 7)) << 4) + (r & 3) * 4)
                            : (uint32_t)(r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4);
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(raw + off));
    return v;
}
// raw B stage -> tf32 operand tiles, K-major SWIZZLE_128B.  K-major B (!MN) arrives swizzled: chunk q sits where wgmma
// reads it, so only the residual is written, at the same offset.  MN-major B ([32 k][BN rows], unswizzled) is transposed
// into a raw-word hi tile and a residual lo tile.  k past K reads as 0 (TMA fills out-of-bounds elements with zeros;
// chunks of a K split are multiples of 32, so a k-block only ever crosses K itself).
template <int BN, bool MN>
__device__ __forceinline__ void split_b_ws(uint32_t raw, uint32_t hi_base, uint32_t lo_base, int tid) {
    constexpr int kChunks = BN * 8, NT = 96;
#pragma unroll
    for (int i = 0; i < (kChunks + NT - 1) / NT; ++i) {
        const int q = tid + i * NT;
        if (q < kChunks) {
            float4 v;
            uint32_t off;
            if (!MN) {
                off = (uint32_t)q * 16u;
                asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(raw + off));
            } else {                                          // a warp covers 32 consecutive rows: conflict-free reads
                const int r = q % BN, c = q / BN;
                v.x = raw_at<BN, true>(raw, r, 4 * c); v.y = raw_at<BN, true>(raw, r, 4 * c + 1);
                v.z = raw_at<BN, true>(raw, r, 4 * c + 2); v.w = raw_at<BN, true>(raw, r, 4 * c + 3);
                off = (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
                st_shared_v4(hi_base + off, v);
            }
            st_shared_v4(lo_base + off, make_float4(resid(v.x), resid(v.y), resid(v.z), resid(v.w)));
        }
    }
}
template <int N>
__device__ __forceinline__ void reg_fence_u(uint32_t (&a)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// gemm_epilogue, with the two adjacent columns of each fragment pair stored as one float2 where the output rows are
// contiguous and 8-byte aligned: a warp then writes whole 32-byte sectors (same value per element as gemm_epilogue)
template <int R>
__device__ __forceinline__ void ws_epilogue(const float (&acc0)[R], const float (&acc1)[R], const float (&accx)[R], float* C,
                                            long long c_rs, long long c_cs, int Ma, int Nb, int rb, int cb,
                                            const float* bias_a, const float* bias_n, bool accumulate) {
    if (c_cs != 1 || (c_rs & 1) || (cb & 1) || (reinterpret_cast<uintptr_t>(C) & 7)) {
        gemm_epilogue(acc0, acc1, accx, C, c_rs, c_cs, Ma, Nb, rb, cb, bias_a, bias_n, accumulate);
        return;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i_row = rb + 8 * h;
        if (i_row >= Ma) continue;
        const float ba = bias_a ? __ldg(bias_a + i_row) : 0.f;
        float* crow = C + (long long)i_row * c_rs;
#pragma unroll
        for (int j = 0; j < R / 4; ++j) {
            const int idx = 4 * j + 2 * h, col = cb + 8 * j;
            if (col >= Nb) continue;
            float o0 = (acc0[idx] + acc1[idx]) + accx[idx] + ba;
            float o1 = (acc0[idx + 1] + acc1[idx + 1]) + accx[idx + 1] + ba;
            if (col + 1 < Nb) {
                if (bias_n) { o0 += __ldg(bias_n + col); o1 += __ldg(bias_n + col + 1); }
                float2* cp = reinterpret_cast<float2*>(crow + col);
                if (accumulate) { const float2 c = *cp; o0 += c.x; o1 += c.y; }
                *cp = make_float2(o0, o1);
            } else {
                if (bias_n) o0 += __ldg(bias_n + col);
                if (accumulate) o0 += crow[col];
                crow[col] = o0;
            }
        }
    }
}

template <int BN>
__device__ __forceinline__ void mma_rs_ws(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t db) {
    if constexpr (BN == 96) wgmma_rs_n96(d, a, db);
    else wgmma_rs_n112(d, a, db);
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(kWsThreads, 1) tma_gemm_kernel_ws(const __grid_constant__ TmaGroup grp, int items) {
    constexpr uint32_t kRaw = ws_raw<BN>(), kBHalf = BN * 128, kSplit = ws_split<BN, B_MN>();
    constexpr int R = BN / 2, kIF = ws_in_flight<BN>();
    static_assert(BN == 96 || BN == 112, "BN");
    static_assert(kIF >= 1 && kIF <= 3, "the fragment ring holds four k-steps");
    extern __shared__ __align__(1024) unsigned char smem[];
    __shared__ __align__(8) uint64_t full[kWsNR], empty[kWsNR], sfull[kWsNS], sempty[kWsNS];
    // the warp index as a shuffled (provably warp-uniform) value: role branches on it do not serialize the wgmma inside them
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    const uint32_t smem_base = (smem_u32(smem) + 1023u) & ~1023u;
    const uint32_t split_base = smem_base + kWsNR * kRaw;

    if (tid == 0) {
        for (int g = 0; g < grp.count; ++g) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&grp.mapA[g]) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&grp.mapB[g]) : "memory");
        }
        for (int s = 0; s < kWsNR; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 3 + 2); }   // split warps + consumer warpgroups
        for (int s = 0; s < kWsNS; ++s) { mbar_init(&sfull[s], 3); mbar_init(&sempty[s], 2); }    // split warps / consumer warpgroups
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_trigger();
    pdl_wait();                          // operands and C may be written by the predecessor

    if (warp < 4) {
        setmaxnreg_dec<64>();
        if (warp == 0) {
            if (lane != 0) return;
            uint32_t kc = 0;
            for (int it = blockIdx.x; it < items; it += gridDim.x) {
                const WsItem w = ws_item<BN>(grp, it);
                const CUtensorMap* mapA = &grp.mapA[w.g];
                const CUtensorMap* mapB = &grp.mapB[w.g];
                for (int kb = 0; kb < w.nkb; ++kb, ++kc) {
                    const int s = kc % kWsNR;
                    mbar_wait(&empty[s], ((kc / kWsNR) & 1) ^ 1);
                    const uint32_t raw = smem_base + (uint32_t)s * kRaw;
                    const int k0 = w.kbeg + kb * kBlockK;
                    mbar_expect_tx(&full[s], kRaw);
                    if (A_MN) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) tma_load_3d(raw + 4096u * j, mapA, &full[s], w.m0 + 32 * j, k0, w.batch);
                    } else {
                        tma_load_3d(raw, mapA, &full[s], k0, w.m0, w.batch);
                    }
                    if (B_MN) tma_load_3d(raw + 128 * 128, mapB, &full[s], w.n0, k0, w.batch);
                    else tma_load_3d(raw + 128 * 128, mapB, &full[s], k0, w.n0, w.batch);
                }
            }
        } else {
            const int stid = tid - 32;
            uint32_t kc = 0;
            for (int it = blockIdx.x; it < items; it += gridDim.x) {
                const WsItem w = ws_item<BN>(grp, it);
                for (int kb = 0; kb < w.nkb; ++kb, ++kc) {
                    const int s = kc % kWsNR, t = kc % kWsNS;
                    mbar_wait(&full[s], (kc / kWsNR) & 1);
                    mbar_wait(&sempty[t], ((kc / kWsNS) & 1) ^ 1);
                    const uint32_t sp = split_base + (uint32_t)t * kSplit;
                    split_b_ws<BN, B_MN>(smem_base + (uint32_t)s * kRaw + 128 * 128, sp, B_MN ? sp + kBHalf : sp, stid);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma
                    __syncwarp();
                    if (lane == 0) { mbar_arrive(&sfull[t]); mbar_arrive(&empty[s]); }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<216>();
    const int ctid = tid - 128, cw = ctid >> 7;
    const int r0 = 64 * cw + 16 * (warp & 3) + (lane >> 2);     // A fragment rows r0, r0 + 8
    const int q = lane & 3;
    uint32_t kc = 0;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
        const WsItem w = ws_item<BN>(grp, it);
        const TmaProblem& P = grp.p[w.g];
        float acc0[R], acc1[R], accx[R];
#pragma unroll
        for (int i = 0; i < R; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; accx[i] = 0.f; }
        uint32_t fa[4][2][4] = {};       // [k-step][hi, lo][fragment]: the registers of the MMAs in flight
        for (int kb = 0; kb < w.nkb; ++kb, ++kc) {
            const int s = kc % kWsNR, t = kc % kWsNS;
            mbar_wait(&full[s], (kc / kWsNR) & 1);
            mbar_wait(&sfull[t], (kc / kWsNS) & 1);
            const uint32_t raw = smem_base + (uint32_t)s * kRaw;
            const uint32_t sp = split_base + (uint32_t)t * kSplit;
            const uint64_t b_hi = desc_sw128(B_MN ? sp : raw + 128 * 128), b_lo = desc_sw128(B_MN ? sp + kBHalf : sp);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                uint32_t (&ah)[4] = fa[kk][0];
                uint32_t (&al)[4] = fa[kk][1];
                // k beyond the chunk end only occurs at K itself (chunks are multiples of 32), which TMA fills with zeros
#pragma unroll
                for (int f = 0; f < 4; ++f) {
                    const float x = raw_a_sw<A_MN>(raw, r0 + 8 * (f & 1), 8 * kk + q + 4 * (f >> 1));
                    ah[f] = __float_as_uint(x);
                    al[f] = __float_as_uint(resid(x));
                }
                wgmma_fence();
                mma_rs_ws<BN>(accx, al, b_hi + 2 * kk);
                mma_rs_ws<BN>(accx, ah, b_lo + 2 * kk);
                mma_rs_ws<BN>((kk & 1) ? acc1 : acc0, ah, b_hi + 2 * kk);
                wgmma_commit();
                wgmma_wait<kIF>();       // k-step kk - kIF has retired: its fragment registers may be rewritten
                reg_fence_u(fa[(kk + 4 - kIF) & 3][0]); reg_fence_u(fa[(kk + 4 - kIF) & 3][1]);
                // k-step 3 of the previous k-block has retired: its raw stage and split tile are free
                if (kk == kIF - 1 && kb > 0 && (ctid & 127) == 0) {
                    mbar_arrive(&empty[(kc - 1) % kWsNR]);
                    mbar_arrive(&sempty[(kc - 1) % kWsNS]);
                }
            }
        }
        wgmma_wait<0>();
        reg_fence(acc0); reg_fence(acc1); reg_fence(accx);
#pragma unroll
        for (int j = 0; j < 4; ++j) { reg_fence_u(fa[j][0]); reg_fence_u(fa[j][1]); }
        if (w.nkb > 0 && (ctid & 127) == 0) {
            mbar_arrive(&empty[(kc - 1) % kWsNR]);
            mbar_arrive(&sempty[(kc - 1) % kWsNS]);
        }
        const bool add_bias = (P.bias != nullptr) && (w.split == 0);
        ws_epilogue(acc0, acc1, accx, P.C + (long long)w.batch * P.sC + (long long)w.split * P.strideP, P.c_rs, P.c_cs, P.Ma,
                    P.Nb, w.m0 + r0, w.n0 + 2 * q, (add_bias && P.bias_on_a) ? P.bias : nullptr,
                    (add_bias && !P.bias_on_a) ? P.bias : nullptr, P.accumulate != 0);
    }
}

template <int BN, bool A_REG>
constexpr size_t smem_bytes() {
    return (size_t)kNR * (128 * 128 + BN * 128) + 2 * (size_t)(2 * (A_REG ? 0 : 128 * 128) + 2 * BN * 128) + 1024;
}

template <int BN, bool A_REG>
int set_attrs() {
    const int sm = (int)smem_bytes<BN, A_REG>();
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel<BN, false, false, A_REG>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel<BN, false, true, A_REG>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel<BN, true, false, A_REG>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel<BN, true, true, A_REG>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    return 0;
}

template <int BN, bool A_REG>
int launch_bn(cudaStream_t st, const TmaGroup& grp, bool a_mn, bool b_mn, dim3 grid) {
    const size_t sm = smem_bytes<BN, A_REG>();
    cudaError_t e;
    if (!a_mn && !b_mn) e = launch_pdl(tma_gemm_kernel<BN, false, false, A_REG>, grid, dim3(kThreads), sm, st, grp);
    else if (!a_mn && b_mn) e = launch_pdl(tma_gemm_kernel<BN, false, true, A_REG>, grid, dim3(kThreads), sm, st, grp);
    else if (a_mn && !b_mn) e = launch_pdl(tma_gemm_kernel<BN, true, false, A_REG>, grid, dim3(kThreads), sm, st, grp);
    else e = launch_pdl(tma_gemm_kernel<BN, true, true, A_REG>, grid, dim3(kThreads), sm, st, grp);
    NATS_CUDA_OK(e);
    return 0;
}

int g_num_sms = 0;
int g_ts_mode = 1;        // 1: skinny products read the 128-row operand into registers instead of splitting it in shared memory

// operand map: K-major source -> dims (K, rows), box (32, box_rows); MN-major source -> dims (rows, K), box (box_rows, 32)
int operand_map(const float* ptr, bool mn, int rows, int K, int ld, int batch, long long bstride, int box_rows, CUtensorMap* out) {
    const long long d0 = mn ? rows : K, d1 = mn ? K : rows;
    return tma_map_tile3d(ptr, d0, d1, batch, ld, batch > 1 ? bstride : d1 * ld, mn ? box_rows : 32, mn ? 32 : box_rows, 1, out);
}

}  // namespace

bool tma_available() { return g_encode != nullptr; }

namespace {
int encode_tile3d(const float* ptr, long long d0, long long d1, long long d2, long long stride1, long long stride2, int b0, int b1,
                  int b2, bool swizzle128, CUtensorMap* out) {
    NATS_REQUIRE(g_encode != nullptr, "tensor maps not available");
    // cache key reuses MapKey: (inner=d0, outer=d1, ld=stride1, batch=d2, bstride=stride2, box_outer=b0*65536+b1*256+b2,
    // mn=2 plain / 3 swizzled)
    MapKey key{ptr, d0, d1, stride1, d2, stride2, b0 * 65536 + b1 * 256 + b2, swizzle128 ? 3 : 2};
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return 0; }
    if (g_maps.size() > (1u << 16)) g_maps.clear();
    cuuint64_t gdim[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
    cuuint64_t gstr[2] = {(cuuint64_t)stride1 * 4, (cuuint64_t)stride2 * 4};
    cuuint32_t box[3] = {(cuuint32_t)b0, (cuuint32_t)b1, (cuuint32_t)b2};
    cuuint32_t estr[3] = {1, 1, 1};
    CUtensorMap m;
    const CUresult r = g_encode(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), gdim, gstr, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled (tile3d) failed (%d): ptr=%p dims=%lld,%lld,%lld strides=%lld,%lld box=%d,%d,%d", (int)r, ptr, d0,
                  d1, d2, stride1, stride2, b0, b1, b2);
        return 1;
    }
    g_maps.emplace(key, m);
    *out = m;
    return 0;
}

// 128-row side of tma_gemm_kernel_ws, 128-byte swizzled: K-major source -> box (32 k, 128 rows); MN-major source -> box
// (32 rows, 32 k), four boxes per stage
int operand_map_ws_a(const float* ptr, bool mn, int rows, int K, int ld, int batch, long long bstride, CUtensorMap* out) {
    const long long d0 = mn ? rows : K, d1 = mn ? K : rows;
    return encode_tile3d(ptr, d0, d1, batch, ld, batch > 1 ? bstride : d1 * ld, 32, mn ? 32 : 128, 1, true, out);
}
// BN side of tma_gemm_kernel_ws: K-major source -> box (32 k, BN rows) 128-byte swizzled, i.e. the K-major SWIZZLE_128B
// layout wgmma reads; MN-major source -> box (BN rows, 32 k), unswizzled, transposed by the split warps
int operand_map_ws_b(const float* ptr, bool mn, int rows, int K, int ld, int batch, long long bstride, int bn, CUtensorMap* out) {
    if (mn) return operand_map(ptr, true, rows, K, ld, batch, bstride, bn, out);
    return encode_tile3d(ptr, K, rows, batch, ld, batch > 1 ? bstride : rows * (long long)ld, 32, bn, 1, true, out);
}

template <int BN>
int set_attrs_ws() {
    const int sk = (int)ws_smem<BN, false>(), sm = (int)ws_smem<BN, true>();
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel_ws<BN, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sk));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel_ws<BN, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel_ws<BN, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sk));
    NATS_CUDA_OK(cudaFuncSetAttribute(tma_gemm_kernel_ws<BN, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    return 0;
}

template <int BN>
int launch_ws(cudaStream_t st, const TmaGroup& grp, bool a_mn, bool b_mn, int items) {
    const dim3 grid(min(items, g_num_sms)), block(kWsThreads);     // persistent: one CTA per SM at most
    const size_t sm = b_mn ? ws_smem<BN, true>() : ws_smem<BN, false>();
    cudaError_t e;
    if (!a_mn && !b_mn) e = launch_pdl(tma_gemm_kernel_ws<BN, false, false>, grid, block, sm, st, grp, items);
    else if (!a_mn && b_mn) e = launch_pdl(tma_gemm_kernel_ws<BN, false, true>, grid, block, sm, st, grp, items);
    else if (a_mn && !b_mn) e = launch_pdl(tma_gemm_kernel_ws<BN, true, false>, grid, block, sm, st, grp, items);
    else e = launch_pdl(tma_gemm_kernel_ws<BN, true, true>, grid, block, sm, st, grp, items);
    NATS_CUDA_OK(e);
    return 0;
}

}  // namespace

int tma_map_tile3d(const float* ptr, long long d0, long long d1, long long d2, long long stride1, long long stride2, int b0,
                   int b1, int b2, CUtensorMap* out) {
    return encode_tile3d(ptr, d0, d1, d2, stride1, stride2, b0, b1, b2, false, out);
}
void tma_gemm_set_ts(int on) { g_ts_mode = on; }
int tma_gemm_get_ts() { return g_ts_mode; }

int tma_gemm_setup() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    NATS_CUDA_OK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (fn == nullptr || q != cudaDriverEntryPointSuccess) {
        set_error("cuTensorMapEncodeTiled not available from the driver");
        return 1;
    }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    NATS_TRY((set_attrs<32, false>()));
    NATS_TRY((set_attrs<64, false>()));
    NATS_TRY((set_attrs<32, true>()));
    NATS_TRY((set_attrs<64, true>()));
    NATS_TRY(set_attrs_ws<96>());
    NATS_TRY(set_attrs_ws<112>());
    int dev = 0;
    NATS_CUDA_OK(cudaGetDevice(&dev));
    NATS_CUDA_OK(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
    return 0;
}


// can this group be served by TMA?  (16-byte aligned pointers, leading dimensions multiple of 4 floats)
bool tma_gemm_eligible(const GemmProblem* probs, int count) {
    if (g_encode == nullptr || count > kMaxGroup) return false;
    for (int i = 0; i < count; ++i) {
        const GemmProblem& q = probs[i];
        if ((q.lda & 3) || (q.ldb & 3)) return false;
        if ((reinterpret_cast<uintptr_t>(q.A) & 15) || (reinterpret_cast<uintptr_t>(q.B) & 15)) return false;
        if (q.batch > 1 && ((q.strideA & 3) || (q.strideB & 3))) return false;
        if (q.M < 1 || q.N < 1 || q.K < 1) return false;
    }
    return true;
}

int tma_gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB) {
    NATS_REQUIRE(count >= 1 && count <= kMaxGroup, "tma gemm group size");
    TmaGroup grp;
    memset(&grp, 0, sizeof(grp));
    grp.count = count;
    int maxM = 0, maxN = 0;
    for (int i = 0; i < count; ++i) { maxM = max(maxM, probs[i].M); maxN = max(maxN, probs[i].N); }
    const TcTile tile = tc_tile(maxM, maxN);
    const bool swapped = tile.swapped, skinny = tile.nb <= 64;
    const int BN = tile.bn;
    // op(A)(m,k): transA ? m contiguous : k contiguous.  op(B)(k,n): transB ? k contiguous : n contiguous.
    const bool opa_mn = transA, opb_mn = !transB;
    const bool a_mn = swapped ? opb_mn : opa_mn;      // the 128-row side operand
    const bool b_mn = swapped ? opa_mn : opb_mn;
    int z = 0, ga = 0, gb = 0, items = 0;
    double flops = 0.0, bytes = 0.0;
    for (int i = 0; i < count; ++i) {
        const GemmProblem& q = probs[i];
        NATS_REQUIRE(q.splitk >= 1 && q.batch >= 1 && (q.splitk == 1 || !q.accumulate), "tma gemm split/batch");
        TmaProblem& t = grp.p[i];
        // the 128-row side (a) and the BN side (b) of the tile
        const float* pa = swapped ? q.B : q.A;
        const float* pb = swapped ? q.A : q.B;
        const int rows_a = swapped ? q.N : q.M, rows_b = swapped ? q.M : q.N;
        const int ld_a = swapped ? q.ldb : q.lda, ld_b = swapped ? q.lda : q.ldb;
        const long long s_a = swapped ? q.strideB : q.strideA, s_b = swapped ? q.strideA : q.strideB;
        if (skinny) {
            NATS_TRY(operand_map(pa, a_mn, rows_a, q.K, ld_a, q.batch, s_a, 128, &grp.mapA[i]));
            NATS_TRY(operand_map(pb, b_mn, rows_b, q.K, ld_b, q.batch, s_b, BN, &grp.mapB[i]));
        } else {
            NATS_TRY(operand_map_ws_a(pa, a_mn, rows_a, q.K, ld_a, q.batch, s_a, &grp.mapA[i]));
            NATS_TRY(operand_map_ws_b(pb, b_mn, rows_b, q.K, ld_b, q.batch, s_b, BN, &grp.mapB[i]));
        }
        t.Ma = rows_a; t.Nb = rows_b;
        if (!swapped) { t.c_rs = q.ldc; t.c_cs = 1; t.bias_on_a = 0; }
        else { t.c_rs = 1; t.c_cs = q.ldc; t.bias_on_a = 1; }
        t.C = q.C; t.bias = q.bias; t.K = q.K; t.batch = q.batch; t.sC = q.strideC;
        t.splitk = q.splitk;
        t.kchunk = tc_kchunk(q);
        t.strideP = q.strideP; t.accumulate = q.accumulate;
        grp.zstart[i] = z;
        grp.istart[i] = items;
        z += q.batch * q.splitk;
        items += q.batch * q.splitk * cdiv(t.Ma, 128) * cdiv(t.Nb, BN);
        ga = max(ga, cdiv(t.Ma, 128));
        gb = max(gb, cdiv(t.Nb, BN));
        flops += 2.0 * q.M * q.N * q.K * q.batch;
        bytes += 4.0 * q.batch * ((double)q.M * q.K + (double)q.K * q.N + (double)q.M * q.N * q.splitk);
    }
    grp.zstart[count] = z;
    grp.istart[count] = items;
    for (int i = count; i < kMaxGroup; ++i) { grp.zstart[i + 1] = z; grp.istart[i + 1] = items; }
    if (items == 0) return 0;
    ProfScope ps(st, skinny ? K_TC_GEMM_SKINNY : K_TC_GEMM, flops, bytes);
    if (BN == 112) return launch_ws<112>(st, grp, a_mn, b_mn, items);
    if (BN == 96) return launch_ws<96>(st, grp, a_mn, b_mn, items);
    dim3 grid(ga, gb, z);
    const bool areg = g_ts_mode != 0;
    if (BN == 32) return areg ? launch_bn<32, true>(st, grp, a_mn, b_mn, grid) : launch_bn<32, false>(st, grp, a_mn, b_mn, grid);
    return areg ? launch_bn<64, true>(st, grp, a_mn, b_mn, grid) : launch_bn<64, false>(st, grp, a_mn, b_mn, grid);
}

}  // namespace nats
