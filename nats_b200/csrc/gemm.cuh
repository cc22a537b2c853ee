// gemm.cuh -- fp32 GEMM engine used by every dense product of the hot path.
//
// C[M,N] (+)= op(A)[M,K] * op(B)[K,N] (+ bias[N]),   row-major with leading dimensions,
//   transA: A is stored [K,M] (M contiguous)      transB: B is stored [N,K] (K contiguous)
// grouped (up to 4 problems per launch: e.g. both encoder directions), batched (strided), split-K
// (each split writes its own partial slab, summed by the consumer kernel => deterministic, no atomics).
//
// Three engines, chosen by gemm_launch from the problems alone: exact-fp32 FFMA tiles (gemm.cu) for products below 64
// rows or 32 deep, and fp32-grade 3xTF32 products on the tensor cores (wgmma): fed by TMA where the operands allow it
// (tma_gemm.cu), else by software loaders (tc_gemm.cu).
#pragma once
#include "common.cuh"

namespace nats {


struct GemmProblem {
    const float* A;
    const float* B;
    float* C;
    const float* bias;  // optional [N]; added by split 0 only
    int M, N, K;
    int lda, ldb, ldc;
    int batch;             // >= 1
    long long strideA, strideB, strideC;
    int splitk;            // >= 1
    int kchunk;            // K range per split (multiple of 16)
    long long strideP;     // distance between split slabs of C
    int accumulate;        // C += result (only with splitk == 1)
};

constexpr int kGemmMaxGroup = 4;
constexpr int kGemmMaxSplit = 32;

struct GemmGroup {
    GemmProblem p[kGemmMaxGroup];
    int zstart[kGemmMaxGroup + 1];
    int count;
};

// Tile of the FFMA engine for a group whose largest M is maxM and smallest N is minN.
struct SgemmTile { int bm, bn; };
inline SgemmTile sgemm_tile(int maxM, int minN) {
    if (maxM <= 32) return {32, 128};
    if (maxM >= 512 && minN >= 512) return {128, 128};
    return {64, 64};
}

// Operand roles and N tile of the tensor-core engines for a group whose largest problem is maxM x maxN.  The larger
// dimension goes on the 128-row side unless M already fills it ("swapped": skinny products put the weights on the
// 128-row side, the batch on the N side, and store transposed).  ma / nb: the 128-row / N extents; bn: the TMA
// engine's tile width (the software-loader engine caps it at 64).
struct TcTile { bool swapped; int ma, nb, bn; };
inline TcTile tc_tile(int maxM, int maxN) {
    TcTile t;
    t.swapped = maxM < 128 && maxN > maxM;
    t.ma = t.swapped ? maxN : maxM;
    t.nb = t.swapped ? maxM : maxN;
    t.bn = t.nb <= 32 ? 32 : t.nb <= 64 ? 64 : t.nb <= 112 ? 112 : 96;
    return t;
}

inline GemmProblem gemm_problem(const float* A, int lda, const float* B, int ldb, float* C, int ldc,
                                int M, int N, int K) {
    GemmProblem p;
    memset(&p, 0, sizeof(p));
    p.A = A; p.B = B; p.C = C; p.bias = nullptr;
    p.M = M; p.N = N; p.K = K; p.lda = lda; p.ldb = ldb; p.ldc = ldc;
    p.batch = 1; p.splitk = 1; p.kchunk = ((K + 15) / 16) * 16; if (p.kchunk == 0) p.kchunk = 16;
    p.accumulate = 0;
    return p;
}
inline void gemm_set_split(GemmProblem& p, int splits, long long strideP) {
    if (splits < 1) splits = 1;
    int chunk = (p.K + splits - 1) / splits;
    chunk = ((chunk + 15) / 16) * 16;
    if (chunk == 0) chunk = 16;
    p.kchunk = chunk;
    p.splitk = splits;
    p.strideP = strideP;
}
// K range per split of the tensor-core engines: the split's chunk rounded up to whole 32-deep k-blocks
inline int tc_kchunk(const GemmProblem& q) {
    const int chunk = q.splitk > 1 ? cdiv(q.K, q.splitk) : q.kchunk;
    return chunk > 0 ? ((chunk + 31) / 32) * 32 : 32;
}

// The engines gemm_launch picks from, also called directly by nats_debug_gemm.  FFMA (gemm.cu): any shape.
int sgemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB);
// tensor-core path (tc_gemm.cu): 3xTF32 on wgmma
int tc_gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB);
int tc_gemm_setup();
// TMA-fed variant (tma_gemm.cu): needs 16-byte aligned operands with leading dimensions multiple of 4
int tma_gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB);
bool tma_gemm_eligible(const GemmProblem* probs, int count);
int tma_gemm_setup();

// Low-level launch: all problems share transposition flags; the engine and its tile are chosen from the problems.
int gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB);

// Number of K-splits that fill the machine for a skinny (M = batch) weight-streaming product.
int gemm_pick_split(const nats_ctx* ctx, int M, int N, int K, int groups = 1);

// Convenience: single problem, picks the tile configuration; if the problem would launch too few CTAs and K
// is deep, runs split-K into `scratch` (scratch_floats available) and reduces (+bias, +accumulate).
int gemm_auto(const nats_ctx* ctx, cudaStream_t st, GemmProblem p, bool transA, bool transB,
              float* scratch, long long scratch_floats);

// out[m,n] (+)= sum_s part[s][m][n] (+ bias[n])
int reduce_splits(cudaStream_t st, const float* part, int nsplit, long long strideP, int M, int N, int ldp,
                  float* out, int ldo, const float* bias, int accumulate);

}  // namespace nats
