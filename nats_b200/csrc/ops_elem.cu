// ops_elem.cu -- embedding gather/scatter, GRU gate epilogues (forward + backward), small reductions.
#include "ops.cuh"
#include "gates.cuh"

namespace nats {

namespace {

// ------------------------------------------------------------------ embedding
__global__ void gather_rows_kernel(const float* __restrict__ Wemb, const int64_t* __restrict__ ids, int n_rows, int W,
                                   int V, int shift, float* __restrict__ out) {
    const long long total = (long long)n_rows * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(i / W), w = (int)(i % W);
        float v = 0.f;
        if (row >= shift) {
            const long long id = ids[row - shift];
            if (id >= 0 && id < V) v = __ldg(Wemb + id * W + w);
        }
        out[i] = v;
    }
}

__global__ void scatter_add_rows_kernel(float* __restrict__ dWemb, const int64_t* __restrict__ ids, int n_rows, int W,
                                        int V, int shift, const float* __restrict__ src) {
    const long long total = (long long)n_rows * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(i / W), w = (int)(i % W);
        if (row < shift) continue;
        const long long id = ids[row - shift];
        if (id >= 0 && id < V) atomicAdd(dWemb + id * W + w, src[i]);
    }
}

// ------------------------------------------------------------------ GRU gates
struct GateFwdPack { GateFwd g[2]; int trace; };
struct GateBwdPack { GateBwd g[2]; int trace; };

constexpr int kGateThreads = 512;       // 125 CTAs per direction at D = 1000: measured 0.3 ms / step faster than 256-thread CTAs (grid completion)
static int g_gate_trace = 0;
static long long g_gate_no = 0;

template <int MODE>
__global__ void gru_gates_fwd_kernel(const __grid_constant__ GateFwdPack pack, int B, int D) {
#ifdef NATS_TRACE_BUILD
    const bool tr = pack.trace && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
#else
    constexpr bool tr = false;
#endif
    const unsigned long long t0 = tr ? gtimer() : 0ull;
    pdl_trigger();
    // the kernel parameters (cold constant cache on every launch) and the index arithmetic do not depend on the
    // predecessor: fetch them while it is still running
    const GateFwd a = pack.g[blockIdx.y];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = idx / D, j = idx - b * D;
    asm volatile("" ::"l"(a.part), "l"(a.xproj), "l"(a.part2), "l"(a.bias), "l"(a.h_prev), "l"(a.mask), "l"(a.h_out), "l"(a.r),
                 "l"(a.ctxsum), "l"(a.part_stride), "r"(a.nsplit), "r"(a.nsplit2), "r"(j));
    pdl_wait();
    const unsigned long long t1 = tr ? gtimer() : 0ull;
    if (idx >= B * D) return;
    gru_gate_fwd_elem<MODE>(a, b, j, D, idx);
#ifdef NATS_TRACE_BUILD
    if (tr) printf("[trace gates_fwd] start %llu | wait_done +%llu | end +%llu ns\n", t0 % 100000000ull, t1 - t0, gtimer() - t0);
#endif
}

__global__ void gru_gates_bwd_kernel(const __grid_constant__ GateBwdPack pack, int B, int D) {
    pdl_trigger();
    const GateBwd a = pack.g[blockIdx.y];             // parameters + indices before the dependency wait (see forward)
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = idx / D, j = idx - b * D;
    asm volatile("" ::"l"(a.part), "l"(a.part2), "l"(a.dh_a), "l"(a.dh_b), "l"(a.h_prev), "l"(a.mask), "l"(a.mean_grad), "l"(a.r),
                 "l"(a.dG), "l"(a.dGx), "l"(a.dh_elem), "l"(a.part_stride), "r"(a.nsplit), "r"(a.nsplit2), "r"(j));
    pdl_wait();
    if (idx >= B * D) return;
    const float m = a.mask ? a.mask[b] : 1.f;
    // all loads first (one L2 round trip), then the sums in the fixed order
    const float r = a.r[idx], u = a.u[idx], c = a.c[idx], p = a.p[idx];
    const float hp = a.h_prev ? a.h_prev[(long long)b * a.ld_hprev + j] : 0.f;
    const float va = a.dh_a ? a.dh_a[(long long)b * a.ld_a + j] : 0.f;
    const float vb = a.dh_b ? a.dh_b[(long long)b * a.ld_b + j] : 0.f;
    const float vm = a.mean_grad ? a.coef[b] * a.mean_grad[(long long)b * a.ld_mean + j] : 0.f;
    float dh = 0.f;
    if (a.dh_a) dh += va;
    if (a.dh_b) dh += vb;
    {
        const int n1 = a.nsplit, n2 = a.nsplit2;
        const float* p1 = a.part + (long long)b * a.part_ld + j;
        const float* p2 = a.part2 + (long long)b * a.part2_ld + j;
        for (int s0 = 0; s0 < n1; s0 += 4) {
            float v[4];
            load4(p1, a.part_stride, s0, n1, v);
            dh = add4(dh, v, s0, n1);
        }
        for (int s0 = 0; s0 < n2; s0 += 4) {
            float v[4];
            load4(p2, a.part2_stride, s0, n2, v);
            dh = add4(dh, v, s0, n2);
        }
    }
    if (a.mean_grad) dh += m * vm;
    const float dhn = m * dh;
    const float du = dhn * (hp - c);
    const float dc = dhn * (1.f - u);
    const float dpc = dc * (1.f - c * c);
    const float dp = dpc * r;
    const float dr = dpc * p;
    const float dgr = dr * r * (1.f - r);
    const float dgu = du * u * (1.f - u);
    const long long row3 = (long long)b * 3 * D;
    a.dG[row3 + j] = dgr; a.dG[row3 + D + j] = dgu; a.dG[row3 + 2 * D + j] = dp;
    a.dGx[row3 + j] = dgr; a.dGx[row3 + D + j] = dgu; a.dGx[row3 + 2 * D + j] = dpc;
    a.dh_elem[idx] = (1.f - m) * dh + dhn * u;
}

// ------------------------------------------------------------------ small elementwise
__global__ void tanh_inplace_kernel(float* x, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        x[i] = tanhf(x[i]);
}
__global__ void dtanh_kernel(const float* __restrict__ g, const float* __restrict__ y, float* __restrict__ dst,
                             long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float t = y[i];
        dst[i] = g[i] * (1.f - t * t);
    }
}
__global__ void sum_parts_dtanh_kernel(const float* __restrict__ a, const float* __restrict__ part, int nsplit,
                                       long long part_stride, const float* __restrict__ y, float* __restrict__ dst,
                                       int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float s = a ? a[i] : 0.f;
    s = sum_strided(part + i, part_stride, nsplit, s);
    const float t = y[i];
    dst[i] = s * (1.f - t * t);
}
__global__ void mask_lengths_kernel(const float* __restrict__ mask, int Tx, int B, float* __restrict__ xlen,
                                    float* __restrict__ inv) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float s = 0.f;
    if (mask) { for (int t = 0; t < Tx; ++t) s += mask[(long long)t * B + b]; }
    else s = (float)Tx;
    xlen[b] = s;
    inv[b] = 1.f / s;
}
__global__ void scale_rows_kernel(const float* __restrict__ src, const float* __restrict__ inv, int B, int C,
                                  float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * C) return;
    out[i] = src[i] * inv[i / C];
}

// column sums: stage 1 -> part[ks][N], stage 2 -> out
template <bool PROD>
__global__ void colsum_stage1(const float* __restrict__ X, const float* __restrict__ Y, long long K, int N, int ld,
                              long long rows_per, float* __restrict__ part) {
    __shared__ float red[8][33];
    const int n = blockIdx.x * 32 + threadIdx.x;
    const long long k0 = blockIdx.y * rows_per;
    const long long k1 = (k0 + rows_per < K) ? (k0 + rows_per) : K;
    float s = 0.f;
    if (n < N) {
        for (long long k = k0 + threadIdx.y; k < k1; k += 8) {
            const float x = X[k * ld + n];
            s += PROD ? x * Y[k * ld + n] : x;
        }
    }
    red[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
        part[(long long)blockIdx.y * N + n] = t;
    }
}
__global__ void colsum_stage2(const float* __restrict__ part, int ks, int N, float* __restrict__ out, int accumulate,
                              float* __restrict__ out2, float* __restrict__ out3) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float s = 0.f;
    for (int i = 0; i < ks; ++i) s += part[(long long)i * N + n];
    out[n] = accumulate ? out[n] + s : s;
    if (out2) out2[n] = accumulate ? out2[n] + s : s;       // the same sums feed several gradients (three readout biases)
    if (out3) out3[n] = accumulate ? out3[n] + s : s;
}

__global__ void cost_reduce_kernel(const float* __restrict__ rowcost, int Ty, int B, float* __restrict__ cost,
                                   float scale, const float* __restrict__ weight, float* __restrict__ total) {
    __shared__ float red[32];
    float acc = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        float s = 0.f;
        for (int t = 0; t < Ty; ++t) s += rowcost[(long long)t * B + b];
        if (cost) cost[b] = s;
        acc += weight ? weight[b] * s : s;
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0 && total) *total = acc * scale;
}

inline int grid_for(long long n, int block) {
    long long g = (n + block - 1) / block;
    if (g > 148LL * 32) g = 148LL * 32;
    if (g < 1) g = 1;
    return (int)g;
}

}  // namespace

int gather_rows(cudaStream_t st, const float* Wemb, const int64_t* ids, int n_rows, int W, int V, int shift,
                float* out) {
    const long long total = (long long)n_rows * W;
    if (total == 0) return 0;
    ProfScope ps(st, K_EMBED, 0.0, 8.0 * total);
    gather_rows_kernel<<<grid_for(total, 256), 256, 0, st>>>(Wemb, ids, n_rows, W, V, shift, out);
    NATS_LAUNCH_OK();
    return 0;
}
int scatter_add_rows(cudaStream_t st, float* dWemb, const int64_t* ids, int n_rows, int W, int V, int shift,
                     const float* src) {
    const long long total = (long long)n_rows * W;
    if (total == 0) return 0;
    ProfScope ps(st, K_EMBED, 0.0, 12.0 * total);
    scatter_add_rows_kernel<<<grid_for(total, 256), 256, 0, st>>>(dWemb, ids, n_rows, W, V, shift, src);
    NATS_LAUNCH_OK();
    return 0;
}

int gru_gates_fwd(cudaStream_t st, const GateFwd* groups, int ngroups, int B, int D, int mode) {
    NATS_REQUIRE(ngroups >= 1 && ngroups <= 2, "gate groups");
    GateFwdPack pack;
    memset(&pack, 0, sizeof(pack));
    for (int i = 0; i < ngroups; ++i) pack.g[i] = groups[i];
    if (g_gate_trace) { ++g_gate_no; pack.trace = (g_gate_no >= g_gate_trace - 1 && g_gate_no < g_gate_trace + 4) ? 1 : 0; }
    dim3 grid(cdiv(B * D, kGateThreads), ngroups);
    ProfScope ps(st, K_GATES_FWD);
    if (mode == 0) NATS_CUDA_OK(launch_pdl(gru_gates_fwd_kernel<0>, grid, dim3(kGateThreads), 0, st, pack, B, D));
    else NATS_CUDA_OK(launch_pdl(gru_gates_fwd_kernel<1>, grid, dim3(kGateThreads), 0, st, pack, B, D));
    return 0;
}
int gru_gates_bwd(cudaStream_t st, const GateBwd* groups, int ngroups, int B, int D) {
    NATS_REQUIRE(ngroups >= 1 && ngroups <= 2, "gate groups");
    GateBwdPack pack;
    memset(&pack, 0, sizeof(pack));
    for (int i = 0; i < ngroups; ++i) pack.g[i] = groups[i];
    dim3 grid(cdiv(B * D, kGateThreads), ngroups);
    ProfScope ps(st, K_GATES_BWD);
    NATS_CUDA_OK(launch_pdl(gru_gates_bwd_kernel, grid, dim3(kGateThreads), 0, st, pack, B, D));
    return 0;
}

int tanh_inplace(cudaStream_t st, float* x, long long n) {
    if (n == 0) return 0;
    ProfScope ps(st, K_ELEMWISE);
    tanh_inplace_kernel<<<grid_for(n, 256), 256, 0, st>>>(x, n);
    NATS_LAUNCH_OK();
    return 0;
}
int dtanh(cudaStream_t st, const float* g, const float* y, float* dst, long long n) {
    if (n == 0) return 0;
    ProfScope ps(st, K_ELEMWISE);
    dtanh_kernel<<<grid_for(n, 256), 256, 0, st>>>(g, y, dst, n);
    NATS_LAUNCH_OK();
    return 0;
}
int sum_parts_dtanh(cudaStream_t st, const float* a, const float* part, int nsplit, long long part_stride,
                    const float* y, float* dst, int B, int D) {
    const int n = B * D;
    ProfScope ps(st, K_ELEMWISE);
    sum_parts_dtanh_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, part, nsplit, part_stride, y, dst, n);
    NATS_LAUNCH_OK();
    return 0;
}
int mask_lengths(cudaStream_t st, const float* mask, int Tx, int B, float* xlen, float* inv) {
    ProfScope ps(st, K_ELEMWISE);
    mask_lengths_kernel<<<cdiv(B, 128), 128, 0, st>>>(mask, Tx, B, xlen, inv);
    NATS_LAUNCH_OK();
    return 0;
}
int scale_rows(cudaStream_t st, const float* src, const float* inv, int B, int C, float* out) {
    ProfScope ps(st, K_ELEMWISE);
    scale_rows_kernel<<<cdiv(B * C, 256), 256, 0, st>>>(src, inv, B, C, out);
    NATS_LAUNCH_OK();
    return 0;
}

static int colsum_impl(cudaStream_t st, const float* X, const float* Y, long long K, int N, int ld, float* out,
                       int accumulate, float* scratch, float* out2 = nullptr, float* out3 = nullptr) {
    if (N == 0) return 0;
    int ks = (int)((K + 255) / 256);
    if (ks > 64) ks = 64;
    if (ks < 1) ks = 1;
    const long long rows_per = (K + ks - 1) / ks;
    dim3 grid(cdiv(N, 32), ks), block(32, 8);
    ProfScope ps(st, K_COLSUM, 0.0, 4.0 * (double)K * N * (Y ? 2 : 1));
    if (Y) colsum_stage1<true><<<grid, block, 0, st>>>(X, Y, K, N, ld, rows_per, scratch);
    else colsum_stage1<false><<<grid, block, 0, st>>>(X, nullptr, K, N, ld, rows_per, scratch);
    NATS_LAUNCH_OK();
    colsum_stage2<<<cdiv(N, 256), 256, 0, st>>>(scratch, ks, N, out, accumulate, out2, out3);
    NATS_LAUNCH_OK();
    return 0;
}
int colsum(cudaStream_t st, const float* X, long long K, int N, int ld, float* out, int accumulate, float* scratch) {
    return colsum_impl(st, X, nullptr, K, N, ld, out, accumulate, scratch);
}
int colsum3(cudaStream_t st, const float* X, long long K, int N, int ld, float* out, float* out2, float* out3, int accumulate,
            float* scratch) {
    return colsum_impl(st, X, nullptr, K, N, ld, out, accumulate, scratch, out2, out3);
}
int colsum_prod(cudaStream_t st, const float* X, const float* Y, long long K, int N, int ld, float* out,
                int accumulate, float* scratch) {
    return colsum_impl(st, X, Y, K, N, ld, out, accumulate, scratch);
}
int cost_reduce(cudaStream_t st, const float* rowcost, int Ty, int B, float* cost, float scale, const float* weight,
                float* total) {
    ProfScope ps(st, K_ELEMWISE);
    cost_reduce_kernel<<<1, 256, 0, st>>>(rowcost, Ty, B, cost, scale, weight, total);
    NATS_LAUNCH_OK();
    return 0;
}

void gates_trace(int on) { g_gate_trace = on; g_gate_no = 0; }

}  // namespace nats
