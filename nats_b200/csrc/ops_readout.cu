// ops_readout.cu -- softmax / cross-entropy rows of the readout (nats.py:763-770, 861-864).
#include "ops.cuh"

#include <cooperative_groups.h>

namespace nats {

namespace {

constexpr int kRowThreads = 512;

__global__ void __launch_bounds__(kRowThreads) nll_rows_kernel(const float* __restrict__ logits, int V,
                                                               const int64_t* __restrict__ y,
                                                               const float* __restrict__ ymask,
                                                               float* __restrict__ lse, float* __restrict__ rowcost) {
    __shared__ float red[32];
    const int r = blockIdx.x;
    const float* row = logits + (long long)r * V;
    float mx = -INFINITY;
    for (int v = threadIdx.x; v < V; v += kRowThreads) mx = fmaxf(mx, row[v]);
    mx = block_max(mx, red);
    float s = 0.f;
    for (int v = threadIdx.x; v < V; v += kRowThreads) s += expf(row[v] - mx);
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        const float l = mx + logf(s);
        lse[r] = l;
        const long long id = y[r];
        const float tgt = (id >= 0 && id < V) ? row[id] : 0.f;
        rowcost[r] = (l - tgt) * (ymask ? ymask[r] : 1.f);      // nats.py:768-770
    }
}

__global__ void dlogits_kernel(float* __restrict__ logits, int rows, int V, const int64_t* __restrict__ y,
                               const float* __restrict__ ymask, const float* __restrict__ lse, float scale) {
    // rows on grid.x (2^31 - 1 blocks), vocabulary chunks on grid.y: rows = Ty*B exceeds the 65535 limit of grid.y for
    // large batches (e.g. batch 160 at maxlen 500)
    const int r = blockIdx.x;
    const float w = (ymask ? ymask[r] : 1.f) * scale;
    const float l = lse[r];
    const long long id = y[r];
    float* row = logits + (long long)r * V;
    for (int v = blockIdx.y * blockDim.x + threadIdx.x; v < V; v += gridDim.y * blockDim.x) {
        float p = expf(row[v] - l);
        if (v == id) p -= 1.f;
        row[v] = p * w;
    }
}

// counter-based uniform in [0,1): splitmix64 of (seed, step, row)
__device__ __forceinline__ float uniform01(uint64_t seed, uint64_t step, uint64_t row) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (step * 0x100000001B3ull + row + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (float)(z >> 40) * (1.0f / 16777216.0f);
}

__global__ void __launch_bounds__(kRowThreads) softmax_sample_kernel(const float* __restrict__ logits, int V,
                                                                     float* __restrict__ probs,
                                                                     int64_t* __restrict__ sample, uint64_t seed,
                                                                     uint64_t step) {
    __shared__ float red[32];
    __shared__ float chunk_sum[kRowThreads];
    __shared__ int s_pick;
    const int r = blockIdx.x, tid = threadIdx.x;
    const float* row = logits + (long long)r * V;
    float* prow = probs + (long long)r * V;
    float mx = -INFINITY;
    for (int v = tid; v < V; v += kRowThreads) mx = fmaxf(mx, row[v]);
    mx = block_max(mx, red);
    float s = 0.f;
    for (int v = tid; v < V; v += kRowThreads) s += expf(row[v] - mx);
    s = block_sum(s, red);
    const float inv = 1.f / s;
    // contiguous chunk per thread so that the inverse-CDF walk is in vocabulary order
    const int per = (V + kRowThreads - 1) / kRowThreads;
    const int v0 = tid * per, v1 = min(V, v0 + per);
    float cs = 0.f;
    for (int v = v0; v < v1; ++v) {
        const float p = expf(row[v] - mx) * inv;                 // nats.py:861
        prow[v] = p;
        cs += p;
    }
    chunk_sum[tid] = cs;
    if (tid == 0) s_pick = -1;
    __syncthreads();
    if (sample) {
        const float u = uniform01(seed, step, (uint64_t)r);
        if (tid == 0) {
            float c = 0.f;
            int pick = kRowThreads - 1;
            for (int i = 0; i < kRowThreads; ++i) {
                if (u < c + chunk_sum[i]) { pick = i; break; }
                c += chunk_sum[i];
            }
            s_pick = pick;
            red[0] = c;
        }
        __syncthreads();
        if (tid == s_pick) {                                      // nats.py:864 (multinomial -> argmax)
            float c = red[0];
            int choice = (v1 > v0) ? (v1 - 1) : (V - 1);
            for (int v = v0; v < v1; ++v) {
                c += prow[v];
                if (u < c) { choice = v; break; }
            }
            sample[r] = choice;
        }
    }
}

// Beam-search shapes (a handful of rows, no sampling, |V| <= 32768): one CTA per row leaves 138 SMs idle and walks the
// row three times.  A cluster of 8 CTAs per row keeps its eighth of the row in registers (one read), and the row maximum
// and the normaliser are combined through distributed shared memory in a fixed order (same value in every CTA).
constexpr int kSmCluster = 8, kSmThreads = 512, kSmPer = 8;

__global__ void __cluster_dims__(kSmCluster, 1, 1) __launch_bounds__(kSmThreads)
    softmax_cluster_kernel(const float* __restrict__ logits, int V, float* __restrict__ probs) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ float red[32];
    __shared__ float s_part[2];
    const int seg = blockIdx.x, tid = threadIdx.x;
    const float* row = logits + (long long)blockIdx.y * V;
    float* prow = probs + (long long)blockIdx.y * V;
    const int seglen = (V + kSmCluster - 1) / kSmCluster;
    const int base = seg * seglen, end = min(V, base + seglen);
    float x[kSmPer];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < kSmPer; ++k) {
        const int i = base + k * kSmThreads + tid;
        x[k] = (i < end) ? row[i] : -INFINITY;
        mx = fmaxf(mx, x[k]);
    }
    mx = block_max(mx, red);
    if (tid == 0) s_part[0] = mx;
    cluster.sync();
    float gmx = -INFINITY;
#pragma unroll
    for (int q = 0; q < kSmCluster; ++q) gmx = fmaxf(gmx, *cluster.map_shared_rank(&s_part[0], q));
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kSmPer; ++k) {
        const int i = base + k * kSmThreads + tid;
        x[k] = (i < end) ? expf(x[k] - gmx) : 0.f;
        s += x[k];
    }
    s = block_sum(s, red);
    if (tid == 0) s_part[1] = s;
    cluster.sync();
    float gs = 0.f;
#pragma unroll
    for (int q = 0; q < kSmCluster; ++q) gs += *cluster.map_shared_rank(&s_part[1], q);
    const float inv = 1.f / gs;
#pragma unroll
    for (int k = 0; k < kSmPer; ++k) {
        const int i = base + k * kSmThreads + tid;
        if (i < end) prow[i] = x[k] * inv;                               // nats.py:861
    }
    cluster.sync();                                                      // remote reads done before any CTA exits
}


// ------------------------------------------------------------------------------------------------
// Few rows x narrow output (f_next's readout hidden layer, nats.py:850-857):
//     out[n, N] = act( sum_p x_p[n, K_p] . W_p[K_p, N] + sum_p bias_p ),   n <= 16, N <= 128, up to 3 parts.
// Three library GEMMs + two slab reductions + a tanh are pure launch latency at this size (~30 us per beam step); here a
// cluster of 8 CTAs splits the concatenated K, 16 warps x (4 columns per lane) per CTA accumulate in exact fp32 FFMA, the
// partial sums meet in distributed shared memory in a fixed order and rank r finishes 16 columns.
// ------------------------------------------------------------------------------------------------
constexpr int kNpCluster = 8, kNpThreads = 512, kNpWarps = kNpThreads / 32, kNpCols = 128, kNpMaxRows = 16;

// Code size matters here: the kernel runs for a few microseconds on 8 SMs and every instruction is fetched cold.  A first
// version with the weight loads unrolled 6-12 deep in registers and the parts selected per row was 58 KB of straight-line
// SASS and ran 25 us, bound by instruction fetch (time fell with the number of rows n because whole blocks were skipped).
// Now the CTA's slice of [W_0; W_1; W_2] is staged in shared memory by a small copy loop (all loads in flight), and the
// product is a rolled loop over weight rows: per row and warp one 16-byte read per lane (4 columns), <= 4 broadcast reads
// of the 16 x values of that k, 64 FFMA.
__global__ void __cluster_dims__(kNpCluster, 1, 1) __launch_bounds__(kNpThreads)
    narrow_proj_kernel(const __grid_constant__ NarrowProj a, int rows_per_cta) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float np_sm[];
    float* ws = np_sm;                                            // [rows_per_cta][N] this CTA's rows of [W_0; W_1; W_2]
    const size_t ws_floats = max((size_t)rows_per_cta * a.N, (size_t)kNpWarps * a.n * kNpCols);
    float* xs = ws + ws_floats;                                   // [rows_per_cta][16] the same rows of [x_0 | x_1 | x_2]
    float* red = xs + (size_t)rows_per_cta * kNpMaxRows;          // [n][128] partial sums of this CTA
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = blockIdx.x;
    const int Kt = a.K[0] + a.K[1] + a.K[2];
    const int j0 = rank * rows_per_cta, j1 = min(Kt, j0 + rows_per_cta);
    const int n4 = a.N >> 2;
#ifdef NARROW_TRACE
    unsigned long long ts[10]; int nts = 0;
#define NP_STAMP() do { if (tid == 0 && rank == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); ts[nts++] = t_; } } while (0)
#else
#define NP_STAMP() do { } while (0)
#endif
    NP_STAMP();
    pdl_trigger();
    // weights do not depend on the predecessor: staged before the dependency wait
    int base = 0;
#pragma unroll 1
    for (int p = 0; p < 3; ++p) {
        const int lo = max(j0, base), hi = min(j1, base + a.K[p]);        // rows of part p in this CTA's slice
        const float* W = a.W[p];
        const long long ldw = a.ldw[p];
#pragma unroll 4
        for (int i = tid; i < (hi - lo) * n4; i += kNpThreads) {
            const int r = i / n4, c4 = i - r * n4;
            const float4 v = __ldg(reinterpret_cast<const float4*>(W + (long long)(lo + r - base) * ldw) + c4);
            reinterpret_cast<float4*>(ws + (size_t)(lo + r - j0) * a.N)[c4] = v;
        }
        base += a.K[p];
    }
    NP_STAMP();
    pdl_wait();
    base = 0;
#pragma unroll 1
    for (int p = 0; p < 3; ++p) {
        const int lo = max(j0, base), hi = min(j1, base + a.K[p]);
        const float* x = a.x[p];
        const long long ldx = a.ldx[p];
#pragma unroll 4
        for (int i = tid; i < (hi - lo) * kNpMaxRows; i += kNpThreads) {
            const int r = i >> 4, b = i & (kNpMaxRows - 1);
            xs[(size_t)(lo + r - j0) * kNpMaxRows + b] = (b < a.n) ? x[(long long)b * ldx + (lo + r - base)] : 0.f;
        }
        base += a.K[p];
    }
    __syncthreads();
    NP_STAMP();
    float4 acc[kNpMaxRows];
#pragma unroll
    for (int b = 0; b < kNpMaxRows; ++b) acc[b] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int nq = (a.n + 3) >> 2;
    if (lane < n4) {
#pragma unroll 2
        for (int jl = warp; jl < j1 - j0; jl += kNpWarps) {
            const float4 w = reinterpret_cast<const float4*>(ws + (size_t)jl * a.N)[lane];
            const float4* xr = reinterpret_cast<const float4*>(xs + (size_t)jl * kNpMaxRows);
#pragma unroll
            for (int q = 0; q < kNpMaxRows / 4; ++q)
                if (q < nq) {
                    const float4 x4 = xr[q];
                    const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float4& c = acc[4 * q + e];
                        c.x = fmaf(xv[e], w.x, c.x); c.y = fmaf(xv[e], w.y, c.y); c.z = fmaf(xv[e], w.z, c.z); c.w = fmaf(xv[e], w.w, c.w);
                    }
                }
        }
    }
    NP_STAMP();
    // the 16 warps' partial sums: each warp parks its own in the (now free) weight stage, then every (row, column) adds
    // the 16 values in warp order -- deterministic, one barrier instead of 16 serial rounds
    __syncthreads();                                              // all warps are done reading ws
    float* part = ws;                                             // [16 warps][n][128]
    if (lane < n4) {
#pragma unroll
        for (int b = 0; b < kNpMaxRows; ++b)
            if (b < a.n) reinterpret_cast<float4*>(part + ((size_t)warp * a.n + b) * kNpCols)[lane] = acc[b];
    }
    __syncthreads();
    for (int i = tid; i < a.n * a.N; i += kNpThreads) {
        const int b = i / a.N, c = i - b * a.N;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < kNpWarps; ++w) v += part[((size_t)w * a.n + b) * kNpCols + c];
        red[b * kNpCols + c] = v;
    }
    NP_STAMP();
    cluster.sync();
    NP_STAMP();
    constexpr int kPer = kNpCols / kNpCluster;
    if (tid < a.n * kPer) {
        const int b = tid / kPer, c = rank * kPer + (tid - b * kPer);
        if (c < a.N) {
            float v = 0.f;
#pragma unroll
            for (int q = 0; q < kNpCluster; ++q) v += cluster.map_shared_rank(red, q)[b * kNpCols + c];
            for (int p = 0; p < 3; ++p)
                if (a.bias[p] != nullptr) v += __ldg(a.bias[p] + c);
            if (a.act_tanh) v = tanhf(v);
            a.out[(long long)b * a.ldo + c] = v;
        }
    }
    NP_STAMP();
    cluster.sync();                                               // remote reads done before any CTA exits
    NP_STAMP();
#ifdef NARROW_TRACE
    if (tid == 0 && rank == 0) printf("[narrow] stage_w +%llu | xs +%llu | main +%llu | reduce +%llu | csync +%llu | tail +%llu | csync +%llu ns\n", ts[1]-ts[0], ts[2]-ts[1], ts[3]-ts[2], ts[4]-ts[3], ts[5]-ts[4], ts[6]-ts[5], ts[7]-ts[6]);
#endif
#undef NP_STAMP
}

size_t narrow_proj_smem(const NarrowProj& a) {
    const int rows = cdiv(a.K[0] + a.K[1] + a.K[2], kNpCluster);
    size_t wsf = (size_t)rows * a.N;                              // the weight stage doubles as the per-warp partial sums
    if (wsf < (size_t)kNpWarps * a.n * kNpCols) wsf = (size_t)kNpWarps * a.n * kNpCols;
    return (wsf + (size_t)rows * kNpMaxRows + (size_t)a.n * kNpCols) * sizeof(float);
}
int g_np_dyn_limit = 48 * 1024;

}  // namespace

int narrow_proj_setup(const nats_ctx* ctx) {
    cudaFuncAttributes fa;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, narrow_proj_kernel));
    const int lim = ctx->max_smem_optin - (int)fa.sharedSizeBytes;
    NATS_CUDA_OK(cudaFuncSetAttribute(narrow_proj_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    g_np_dyn_limit = lim;
    return 0;
}

bool narrow_proj_eligible(const NarrowProj& a) {
    static const int off = [] { const char* e = getenv("NATS_NARROW_PROJ"); return e && atoi(e) == 0; }();
    if (off || a.n < 1 || a.n > kNpMaxRows || a.N < 4 || a.N > kNpCols || (a.N & 3)) return false;
    for (int p = 0; p < 3; ++p)                                    // 16-byte weight rows
        if (a.K[p] > 0 && ((a.ldw[p] & 3) || (reinterpret_cast<uintptr_t>(a.W[p]) & 15))) return false;
    return a.K[0] + a.K[1] + a.K[2] >= 1 && narrow_proj_smem(a) <= (size_t)g_np_dyn_limit;
}

int narrow_proj(cudaStream_t st, const NarrowProj& a) {
    NATS_REQUIRE(narrow_proj_eligible(a), "narrow_proj shape");
    const int Kt = a.K[0] + a.K[1] + a.K[2];
    const int rows = cdiv(Kt, kNpCluster);
    ProfScope ps(st, K_ELEMWISE, 2.0 * a.n * Kt * a.N, 4.0 * ((double)Kt * a.N + (double)a.n * Kt + (double)a.n * a.N));
    NATS_CUDA_OK(launch_pdl(narrow_proj_kernel, dim3(kNpCluster), dim3(kNpThreads), narrow_proj_smem(a), st, a, rows));
    return 0;
}

int nll_rows(cudaStream_t st, const float* logits, int rows, int V, const int64_t* y, const float* ymask, float* lse,
             float* rowcost) {
    if (rows == 0) return 0;
    ProfScope ps(st, K_NLL, 0.0, 8.0 * rows * V);
    nll_rows_kernel<<<rows, kRowThreads, 0, st>>>(logits, V, y, ymask, lse, rowcost);
    NATS_LAUNCH_OK();
    return 0;
}
int dlogits_inplace(cudaStream_t st, float* logits, int rows, int V, const int64_t* y, const float* ymask,
                    const float* lse, float scale) {
    if (rows == 0) return 0;
    int gy = cdiv(V, 256 * 4);
    if (gy < 1) gy = 1;
    if (gy > 65535) gy = 65535;
    dim3 grid(rows, gy);
    ProfScope ps(st, K_DLOGITS, 0.0, 8.0 * rows * V);
    dlogits_kernel<<<grid, 256, 0, st>>>(logits, rows, V, y, ymask, lse, scale);
    NATS_LAUNCH_OK();
    return 0;
}
int softmax_sample_rows(cudaStream_t st, const float* logits, int rows, int V, float* probs, int64_t* sample,
                        uint64_t seed, uint64_t step) {
    if (rows == 0) return 0;
    ProfScope ps(st, K_SOFTMAX_SAMPLE, 0.0, 16.0 * rows * V);
    static const int force_simple = [] { const char* e = getenv("NATS_SOFTMAX_SIMPLE"); return e && atoi(e) != 0; }();
    if (!force_simple && sample == nullptr && rows <= 132 && V <= kSmCluster * kSmThreads * kSmPer) {
        softmax_cluster_kernel<<<dim3(kSmCluster, rows), kSmThreads, 0, st>>>(logits, V, probs);
        NATS_LAUNCH_OK();
        return 0;
    }
    softmax_sample_kernel<<<rows, kRowThreads, 0, st>>>(logits, V, probs, sample, seed, step);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace nats
