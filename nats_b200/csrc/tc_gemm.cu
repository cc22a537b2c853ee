// tc_gemm.cu -- fp32-grade GEMM on the Hopper tensor cores: wgmma kind::tf32 with the 3xTF32 split
//   x = hi + lo,  hi = rna_tf32(x),  lo = rna_tf32(x - hi);   a.b ~= a_hi.b_hi + a_hi.b_lo + a_lo.b_hi
// (error ~1e-6 relative per product, i.e. fp32 grade -- the parity tests keep their fp32 tolerances).  The hi.hi products
// alternate between two register accumulators and the two small cross terms go to a third, so that each accumulation
// chain is short; the epilogue adds the three with ordinary round-to-nearest fp32 adds.
//
// One CTA (two warpgroups, 256 threads) computes a [128 x BN] tile, warpgroup w owning rows 64w..64w+63:
//   every thread loads its share of the next 32-deep k-block from global memory into registers while the tensor cores
//   work on the current one, splits it into {hi, lo} and stores both into the other shared-memory stage in the canonical
//   K-major SWIZZLE_128B layout (row = 128 B = 32 tf32, 16-byte chunk c of row r stored at chunk c ^ (r & 7)).  The loader
//   handles K-contiguous AND row-contiguous sources, so every transposition of the caller maps to the same K-major
//   operands (tf32 wgmma reads K-major shared-memory operands only).
//   per k-block and warpgroup: 4 k-steps x 3 wgmma m64 x BN x 8, then a wait before that stage is written again.
// Operand roles are chosen by the host so that the 128-row side is the larger one (skinny recurrent products run
// "swapped": the weight matrix is the 128-row operand, the batch is the N side, the store is transposed).
#include "gemm.cuh"
#include "tc_common.cuh"

namespace nats {

namespace {

constexpr int kTcThreads = 256;
constexpr int kTcBlockK = 32;        // tf32 elements per k-block = one 128-byte swizzle row
constexpr int kTcMaxGroup = 4;

struct TcProblem {
    const float* A;      // 128-row ("M") side operand: element (i,k) at A[i*a_rs + k*a_ks]
    const float* B;      // N side operand:            element (j,k) at B[j*b_rs + k*b_ks]
    float* C;            // output: element (i,j) at C[i*c_rs + j*c_cs]
    const float* bias;   // optional, indexed by i (bias_on_a) or j
    int Ma, Nb, K;
    long long a_rs, a_ks, b_rs, b_ks, c_rs, c_cs;
    int batch;
    long long sA, sB, sC;
    int splitk, kchunk;  // kchunk multiple of 32
    long long strideP;
    int accumulate;
    int bias_on_a;
};
struct TcGroup {
    TcProblem p[kTcMaxGroup];
    int zstart[kTcMaxGroup + 1];
    int count;
};

using namespace tc;

// one operand tile: ROWS x 32 tf32, read from global with arbitrary (row, k) strides, written as hi/lo K-major tiles
template <int ROWS>
struct TileLoader {
    static constexpr int kChunks = ROWS * 8;                                  // 16-byte chunks (4 k each)
    static constexpr int kPer = (kChunks + kTcThreads - 1) / kTcThreads;
    float4 v[kPer];

    __device__ __forceinline__ void load(const float* __restrict__ g, long long rs, long long ks, int row0, int nrows,
                                         int k0, int kend, bool vec_ok, int tid) {
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const int q = tid + i * kTcThreads;
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q < kChunks) {
                int r, c;
                if (ks == 1) { r = q >> 3; c = q & 7; }                      // K contiguous: 8 threads cover a row
                else { r = q % ROWS; c = q / ROWS; }                          // row contiguous: a warp covers 32 rows
                const int gr = row0 + r, gk = k0 + 4 * c;
                if (gr < nrows && gk < kend) {
                    const float* p = g + (long long)gr * rs + (long long)gk * ks;
                    if (ks == 1 && vec_ok && gk + 3 < kend) {
                        val = __ldg(reinterpret_cast<const float4*>(p));
                    } else {
                        val.x = __ldg(p);
                        if (gk + 1 < kend) val.y = __ldg(p + ks);
                        if (gk + 2 < kend) val.z = __ldg(p + 2 * ks);
                        if (gk + 3 < kend) val.w = __ldg(p + 3 * ks);
                    }
                }
            }
            v[i] = val;
        }
    }
    __device__ __forceinline__ void store(uint32_t hi_base, uint32_t lo_base, long long ks, int tid) const {
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const int q = tid + i * kTcThreads;
            if (q < kChunks) {
                int r, c;
                if (ks == 1) { r = q >> 3; c = q & 7; }
                else { r = q % ROWS; c = q / ROWS; }
                const uint32_t off = (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
                float4 hi, lo;
                hi.x = to_tf32(v[i].x); hi.y = to_tf32(v[i].y); hi.z = to_tf32(v[i].z); hi.w = to_tf32(v[i].w);
                lo.x = to_tf32(v[i].x - hi.x); lo.y = to_tf32(v[i].y - hi.y);
                lo.z = to_tf32(v[i].z - hi.z); lo.w = to_tf32(v[i].w - hi.w);
                st_shared_v4(hi_base + off, hi);
                st_shared_v4(lo_base + off, lo);
            }
        }
    }
};

template <int BN>
__device__ __forceinline__ void mma_bn(float (&d)[BN / 2], uint64_t da, uint64_t db) {
    if constexpr (BN == 32) wgmma_ss_n32(d, da, db);
    else wgmma_ss_n64(d, da, db);
}

template <int BN>
__global__ void __launch_bounds__(kTcThreads, 1) tc_gemm_kernel(const __grid_constant__ TcGroup grp) {
    constexpr uint32_t kABytes = 128 * 128;                 // one 128-row operand tile (hi or lo)
    constexpr uint32_t kBBytes = BN * 128;
    constexpr uint32_t kStageBytes = 2 * kABytes + 2 * kBBytes;
    constexpr int R = BN / 2;                               // accumulator registers per thread
    static_assert(BN == 32 || BN == 64, "BN");

    extern __shared__ __align__(1024) unsigned char smem[];

    int z = blockIdx.z, g = 0;
#pragma unroll
    for (int i = 1; i < kTcMaxGroup; ++i)
        if (i < grp.count && z >= grp.zstart[i]) g = i;
    const TcProblem& P = grp.p[g];
    z -= grp.zstart[g];
    const int split = z % P.splitk, batch = z / P.splitk;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BN;
    if (m0 >= P.Ma || n0 >= P.Nb) return;                   // whole CTA leaves together (uniform)

    const int kbeg = split * P.kchunk;
    const int kend = min(P.K, kbeg + P.kchunk);
    const int nkb = (kend > kbeg) ? (kend - kbeg + kTcBlockK - 1) / kTcBlockK : 0;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
    const uint32_t smem_base = (smem_u32(smem) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
    pdl_trigger();
    pdl_wait();

    float acc0[R], acc1[R], accx[R];
#pragma unroll
    for (int i = 0; i < R; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; accx[i] = 0.f; }

    const float* __restrict__ A = P.A + (long long)batch * P.sA;
    const float* __restrict__ B = P.B + (long long)batch * P.sB;
    const bool vecA = (P.a_ks == 1) && ((P.a_rs & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
    const bool vecB = (P.b_ks == 1) && ((P.b_rs & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
    TileLoader<128> la;
    TileLoader<BN> lb;
    if (nkb > 0) {
        la.load(A, P.a_rs, P.a_ks, m0, P.Ma, kbeg, kend, vecA, tid);
        lb.load(B, P.b_rs, P.b_ks, n0, P.Nb, kbeg, kend, vecB, tid);
        la.store(smem_base, smem_base + kABytes, P.a_ks, tid);
        lb.store(smem_base + 2 * kABytes, smem_base + 2 * kABytes + kBBytes, P.b_ks, tid);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
    __syncthreads();
    for (int kb = 0; kb < nkb; ++kb) {
        const uint32_t st = smem_base + (uint32_t)(kb & 1) * kStageBytes;
        const bool next = kb + 1 < nkb;
        if (next) {                                         // next tile's global loads fly while this one is consumed
            const int k0 = kbeg + (kb + 1) * kTcBlockK;
            la.load(A, P.a_rs, P.a_ks, m0, P.Ma, k0, kend, vecA, tid);
            lb.load(B, P.b_rs, P.b_ks, n0, P.Nb, k0, kend, vecB, tid);
        }
        const uint64_t a_hi = desc_sw128(st + (uint32_t)wg * (kABytes / 2)), a_lo = desc_sw128(st + kABytes + (uint32_t)wg * (kABytes / 2));
        const uint64_t b_hi = desc_sw128(st + 2 * kABytes), b_lo = desc_sw128(st + 2 * kABytes + kBBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kTcBlockK / 8; ++kk) {
            const uint64_t adv = (uint64_t)(kk * 2);          // +32 bytes per k-step inside the swizzle row
            mma_bn<BN>(accx, a_lo + adv, b_hi + adv);
            mma_bn<BN>(accx, a_hi + adv, b_lo + adv);
            mma_bn<BN>((kk & 1) ? acc1 : acc0, a_hi + adv, b_hi + adv);
        }
        wgmma_commit();
        if (next) {                                         // the other stage was drained by the wait of the previous k-block
            const uint32_t nx = smem_base + (uint32_t)((kb + 1) & 1) * kStageBytes;
            la.store(nx, nx + kABytes, P.a_ks, tid);
            lb.store(nx + 2 * kABytes, nx + 2 * kABytes + kBBytes, P.b_ks, tid);
        }
        wgmma_wait<0>();
        reg_fence(acc0); reg_fence(acc1); reg_fence(accx);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
    }

    const bool add_bias = (P.bias != nullptr) && (split == 0);
    gemm_epilogue(acc0, acc1, accx, P.C + (long long)batch * P.sC + (long long)split * P.strideP, P.c_rs, P.c_cs, P.Ma, P.Nb,
                  m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2), n0 + 2 * (lane & 3), (add_bias && P.bias_on_a) ? P.bias : nullptr,
                  (add_bias && !P.bias_on_a) ? P.bias : nullptr, P.accumulate != 0);
}

template <int BN>
constexpr size_t tc_smem_bytes() {
    return (size_t)2 * (2 * 128 * 128 + 2 * BN * 128) + 1024;
}

template <int BN>
int tc_launch(cudaStream_t st, const TcGroup& grp, bool skinny) {
    int ga = 0, gb = 0;
    double flops = 0.0, bytes = 0.0;
    for (int i = 0; i < grp.count; ++i) {
        const TcProblem& q = grp.p[i];
        ga = max(ga, cdiv(q.Ma, 128));
        gb = max(gb, cdiv(q.Nb, BN));
        flops += 2.0 * q.Ma * q.Nb * q.K * q.batch;
        bytes += 4.0 * q.batch * ((double)q.Ma * q.K + (double)q.K * q.Nb + (double)q.Ma * q.Nb * q.splitk);
    }
    const int gz = grp.zstart[grp.count];
    if (ga == 0 || gb == 0 || gz == 0) return 0;
    ProfScope ps(st, skinny ? K_TC_GEMM_SKINNY : K_TC_GEMM, flops, bytes);
    dim3 grid(ga, gb, gz);
    NATS_CUDA_OK(launch_pdl(tc_gemm_kernel<BN>, grid, dim3(kTcThreads), tc_smem_bytes<BN>(), st, grp));
    return 0;
}

}  // namespace

// One-time kernel attribute setup (must not happen lazily inside a stream capture).
int tc_gemm_setup() {
    NATS_CUDA_OK(cudaFuncSetAttribute(tc_gemm_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes<32>()));
    NATS_CUDA_OK(cudaFuncSetAttribute(tc_gemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes<64>()));
    return 0;
}

// Same contract as gemm_launch (gemm.cuh) -- C = op(A).op(B) row-major, grouped / batched / split-K slabs -- on the
// tensor cores.  All problems of a group must agree on the operand roles picked here (they do: same shapes class).
int tc_gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB) {
    NATS_REQUIRE(count >= 1 && count <= kTcMaxGroup, "tc gemm group size");
    TcGroup grp;
    memset(&grp, 0, sizeof(grp));
    grp.count = count;
    int z = 0, maxM = 0, maxN = 0;
    for (int i = 0; i < count; ++i) { maxM = max(maxM, probs[i].M); maxN = max(maxN, probs[i].N); }
    if (maxM == 0 || maxN == 0) return 0;
    const TcTile tile = tc_tile(maxM, maxN);
    const bool swapped = tile.swapped;
    for (int i = 0; i < count; ++i) {
        const GemmProblem& q = probs[i];
        NATS_REQUIRE(q.splitk >= 1 && q.batch >= 1 && (q.splitk == 1 || !q.accumulate), "tc gemm split/batch");
        TcProblem& t = grp.p[i];
        // op(A)(m,k) and op(B)(k,n) as (row stride, k stride)
        const long long am_rs = transA ? 1 : q.lda, am_ks = transA ? q.lda : 1;
        const long long bn_rs = transB ? q.ldb : 1, bn_ks = transB ? 1 : q.ldb;
        if (!swapped) {
            t.A = q.A; t.a_rs = am_rs; t.a_ks = am_ks; t.Ma = q.M; t.sA = q.strideA;
            t.B = q.B; t.b_rs = bn_rs; t.b_ks = bn_ks; t.Nb = q.N; t.sB = q.strideB;
            t.c_rs = q.ldc; t.c_cs = 1; t.bias_on_a = 0;
        } else {
            t.A = q.B; t.a_rs = bn_rs; t.a_ks = bn_ks; t.Ma = q.N; t.sA = q.strideB;
            t.B = q.A; t.b_rs = am_rs; t.b_ks = am_ks; t.Nb = q.M; t.sB = q.strideA;
            t.c_rs = 1; t.c_cs = q.ldc; t.bias_on_a = 1;
        }
        t.C = q.C; t.bias = q.bias; t.K = q.K; t.batch = q.batch; t.sC = q.strideC;
        t.splitk = q.splitk;
        t.kchunk = tc_kchunk(q);
        t.strideP = q.strideP; t.accumulate = q.accumulate;
        grp.zstart[i] = z;
        z += q.batch * q.splitk;
    }
    grp.zstart[count] = z;
    for (int i = count; i < kTcMaxGroup; ++i) grp.zstart[i + 1] = z;
    return tile.bn == 32 ? tc_launch<32>(st, grp, true) : tc_launch<64>(st, grp, tile.nb <= 64);
}

}  // namespace nats
