// gemm.cu -- fp32 tiled SGEMM (grouped / batched / split-K).  See gemm.cuh.
#include "gemm.cuh"

namespace nats {

namespace {

constexpr int kPad = 4;

// tile element (x, k) = src[x*ld + k]  (k contiguous in memory); staged in registers as float4 along k
template <int BX, int BK, int NT, int PT>
__device__ __forceinline__ void load_kcontig(const float* __restrict__ src, int ld, int x0, int X, int k0,
                                             int kend, bool vec, int tid, float4 (&r)[PT]) {
#pragma unroll
    for (int i = 0; i < PT; ++i) {
        const int v = tid + i * NT;
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (v < BX * BK / 4) {
            const int x = v / (BK / 4), kq = (v % (BK / 4)) * 4;
            const int gx = x0 + x, gk = k0 + kq;
            if (gx < X && gk < kend) {
                const float* p = src + (long long)gx * ld + gk;
                if (vec && gk + 3 < kend) {
                    val = __ldg(reinterpret_cast<const float4*>(p));
                } else {
                    val.x = __ldg(p);
                    if (gk + 1 < kend) val.y = __ldg(p + 1);
                    if (gk + 2 < kend) val.z = __ldg(p + 2);
                    if (gk + 3 < kend) val.w = __ldg(p + 3);
                }
            }
        }
        r[i] = val;
    }
}
template <int BX, int BK, int NT, int PT>
__device__ __forceinline__ void store_kcontig(float (*S)[BX + kPad], int tid, const float4 (&r)[PT]) {
#pragma unroll
    for (int i = 0; i < PT; ++i) {
        const int v = tid + i * NT;
        if (v < BX * BK / 4) {
            const int x = v / (BK / 4), kq = (v % (BK / 4)) * 4;
            S[kq + 0][x] = r[i].x;
            S[kq + 1][x] = r[i].y;
            S[kq + 2][x] = r[i].z;
            S[kq + 3][x] = r[i].w;
        }
    }
}
// tile element (x, k) = src[k*ld + x]  (x contiguous in memory); float4 along x
template <int BX, int BK, int NT, int PT>
__device__ __forceinline__ void load_xcontig(const float* __restrict__ src, int ld, int x0, int X, int k0,
                                             int kend, bool vec, int tid, float4 (&r)[PT]) {
#pragma unroll
    for (int i = 0; i < PT; ++i) {
        const int v = tid + i * NT;
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (v < BX * BK / 4) {
            const int k = v / (BX / 4), xq = (v % (BX / 4)) * 4;
            const int gk = k0 + k, gx = x0 + xq;
            if (gk < kend && gx < X) {
                const float* p = src + (long long)gk * ld + gx;
                if (vec && gx + 3 < X) {
                    val = __ldg(reinterpret_cast<const float4*>(p));
                } else {
                    val.x = __ldg(p);
                    if (gx + 1 < X) val.y = __ldg(p + 1);
                    if (gx + 2 < X) val.z = __ldg(p + 2);
                    if (gx + 3 < X) val.w = __ldg(p + 3);
                }
            }
        }
        r[i] = val;
    }
}
template <int BX, int BK, int NT, int PT>
__device__ __forceinline__ void store_xcontig(float (*S)[BX + kPad], int tid, const float4 (&r)[PT]) {
#pragma unroll
    for (int i = 0; i < PT; ++i) {
        const int v = tid + i * NT;
        if (v < BX * BK / 4) {
            const int k = v / (BX / 4), xq = (v % (BX / 4)) * 4;
            *reinterpret_cast<float4*>(&S[k][xq]) = r[i];
        }
    }
}

template <int BM, int BN, int BK, int TM, int TN, bool TA, bool TB>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
sgemm_kernel(const __grid_constant__ GemmGroup grp) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int RM = TM / 4, RN = TN / 4;
    constexpr int APT = (BM * BK / 4 + NT - 1) / NT, BPT = (BN * BK / 4 + NT - 1) / NT;
    static_assert(TM % 4 == 0 && TN % 4 == 0 && BK % 4 == 0, "tile shape");

    __shared__ __align__(16) float As[2][BK][BM + kPad];
    __shared__ __align__(16) float Bs[2][BK][BN + kPad];

    int z = blockIdx.z, g = 0;
#pragma unroll
    for (int i = 1; i < kGemmMaxGroup; ++i)
        if (i < grp.count && z >= grp.zstart[i]) g = i;
    const GemmProblem& P = grp.p[g];
    z -= grp.zstart[g];
    const int split = z % P.splitk, batch = z / P.splitk;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    if (m0 >= P.M || n0 >= P.N) return;
    pdl_trigger();
    pdl_wait();

    const int kbeg = split * P.kchunk;
    const int kend = min(P.K, kbeg + P.kchunk);
    const float* __restrict__ A = P.A + (long long)batch * P.strideA;
    const float* __restrict__ B = P.B + (long long)batch * P.strideB;
    float* __restrict__ C = P.C + (long long)batch * P.strideC + (long long)split * P.strideP;
    const bool vecA = ((P.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
    const bool vecB = ((P.ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
    const bool vecC = ((P.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);

    const int tid = threadIdx.x;
    const int tx = tid % (BN / TN), ty = tid / (BN / TN);

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float4 ra[APT], rb[BPT];
    auto load_tiles = [&](int k0) {
        if (TA) load_xcontig<BM, BK, NT, APT>(A, P.lda, m0, P.M, k0, kend, vecA, tid, ra);
        else    load_kcontig<BM, BK, NT, APT>(A, P.lda, m0, P.M, k0, kend, vecA, tid, ra);
        if (TB) load_kcontig<BN, BK, NT, BPT>(B, P.ldb, n0, P.N, k0, kend, vecB, tid, rb);
        else    load_xcontig<BN, BK, NT, BPT>(B, P.ldb, n0, P.N, k0, kend, vecB, tid, rb);
    };
    auto store_tiles = [&](int buf) {
        if (TA) store_xcontig<BM, BK, NT, APT>(As[buf], tid, ra);
        else    store_kcontig<BM, BK, NT, APT>(As[buf], tid, ra);
        if (TB) store_kcontig<BN, BK, NT, BPT>(Bs[buf], tid, rb);
        else    store_xcontig<BN, BK, NT, BPT>(Bs[buf], tid, rb);
    };

    int cur = 0;
    if (kbeg < kend) {
        load_tiles(kbeg);
        store_tiles(0);
    }
    __syncthreads();
    for (int kt = kbeg; kt < kend; kt += BK) {
        const bool has_next = (kt + BK) < kend;
        if (has_next) load_tiles(kt + BK);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[TM], b[TN];
#pragma unroll
            for (int r = 0; r < RM; ++r) {
                const float4 t = *reinterpret_cast<const float4*>(&As[cur][kk][r * (BM / RM) + ty * 4]);
                a[r * 4 + 0] = t.x; a[r * 4 + 1] = t.y; a[r * 4 + 2] = t.z; a[r * 4 + 3] = t.w;
            }
#pragma unroll
            for (int c = 0; c < RN; ++c) {
                const float4 t = *reinterpret_cast<const float4*>(&Bs[cur][kk][c * (BN / RN) + tx * 4]);
                b[c * 4 + 0] = t.x; b[c * 4 + 1] = t.y; b[c * 4 + 2] = t.z; b[c * 4 + 3] = t.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (has_next) store_tiles(cur ^ 1);
        __syncthreads();
        cur ^= 1;
    }

    const bool add_bias = (P.bias != nullptr) && (split == 0);
#pragma unroll
    for (int r = 0; r < RM; ++r) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int gm = m0 + r * (BM / RM) + ty * 4 + i;
            if (gm >= P.M) continue;
#pragma unroll
            for (int c = 0; c < RN; ++c) {
                const int gn = n0 + c * (BN / RN) + tx * 4;
                if (gn >= P.N) continue;
                float v[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) v[j] = acc[r * 4 + i][c * 4 + j];
                float* cp = C + (long long)gm * P.ldc + gn;
                if (vecC && gn + 3 < P.N) {
                    if (add_bias) {
                        v[0] += __ldg(P.bias + gn); v[1] += __ldg(P.bias + gn + 1);
                        v[2] += __ldg(P.bias + gn + 2); v[3] += __ldg(P.bias + gn + 3);
                    }
                    float4 o = make_float4(v[0], v[1], v[2], v[3]);
                    if (P.accumulate) {
                        const float4 old = *reinterpret_cast<const float4*>(cp);
                        o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
                    }
                    *reinterpret_cast<float4*>(cp) = o;
                } else {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if (gn + j < P.N) {
                            float o = v[j];
                            if (add_bias) o += __ldg(P.bias + gn + j);
                            if (P.accumulate) o += cp[j];
                            cp[j] = o;
                        }
                    }
                }
            }
        }
    }
}

template <int BM, int BN, int BK, int TM, int TN>
int launch_cfg(cudaStream_t st, const GemmGroup& grp, bool ta, bool tb) {
    int gx = 0, gy = 0;
    for (int i = 0; i < grp.count; ++i) {
        gx = max(gx, cdiv(grp.p[i].N, BN));
        gy = max(gy, cdiv(grp.p[i].M, BM));
    }
    const int gz = grp.zstart[grp.count];
    if (gx == 0 || gy == 0 || gz == 0) return 0;
    dim3 grid(gx, gy, gz), block((BM / TM) * (BN / TN));
    double flops = 0.0, bytes = 0.0;
    if (prof_enabled())
        for (int i = 0; i < grp.count; ++i) {
            const GemmProblem& q = grp.p[i];
            flops += 2.0 * q.M * q.N * q.K * q.batch;
            bytes += 4.0 * q.batch * ((double)q.M * q.K + (double)q.K * q.N + (double)q.M * q.N * q.splitk);
        }
    const int cfg_id = (BM == 128) ? 0 : (BM == 64 ? 1 : 2);
    ProfScope ps(st, K_GEMM_BASE + cfg_id * 4 + (ta ? 2 : 0) + (tb ? 1 : 0), flops, bytes);
    cudaError_t le;
    if (!ta && !tb) le = launch_pdl(sgemm_kernel<BM, BN, BK, TM, TN, false, false>, grid, block, 0, st, grp);
    else if (!ta && tb) le = launch_pdl(sgemm_kernel<BM, BN, BK, TM, TN, false, true>, grid, block, 0, st, grp);
    else if (ta && !tb) le = launch_pdl(sgemm_kernel<BM, BN, BK, TM, TN, true, false>, grid, block, 0, st, grp);
    else le = launch_pdl(sgemm_kernel<BM, BN, BK, TM, TN, true, true>, grid, block, 0, st, grp);
    NATS_CUDA_OK(le);
    return 0;
}

__global__ void reduce_splits_kernel(const float* __restrict__ part, int nsplit, long long strideP, int M, int N,
                                     int ldp, float* __restrict__ out, int ldo, const float* __restrict__ bias,
                                     int accumulate) {
    pdl_trigger();
    pdl_wait();
    const long long total = (long long)M * N;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / N), n = (int)(i % N);
        float s = sum_strided(part + (long long)m * ldp + n, strideP, nsplit);
        if (bias) s += __ldg(bias + n);
        float* o = out + (long long)m * ldo + n;
        if (accumulate) s += *o;
        *o = s;
    }
}

}  // namespace

static int g_use_tc = 2;      // 0: FFMA, 1: wgmma with software loaders, 2: wgmma fed by TMA where possible
void gemm_set_tensor_cores(int on) { g_use_tc = on; }
int gemm_get_tensor_cores() { return g_use_tc; }

// is this group worth a 128-row tensor-core tile?  (tiny problems stay on the FFMA kernels)
static bool tc_eligible(const GemmProblem* probs, int count) {
    if (!g_use_tc) return false;
    for (int i = 0; i < count; ++i) {
        const int big = probs[i].M > probs[i].N ? probs[i].M : probs[i].N;
        if (big < 64 || probs[i].K < 32) return false;
    }
    return true;
}


int gemm_launch(cudaStream_t st, const GemmProblem* probs, int count, bool transA, bool transB, int cfg) {
    NATS_REQUIRE(count >= 1 && count <= kGemmMaxGroup, "gemm group size");
    if (tc_eligible(probs, count)) {
        if (g_use_tc >= 2 && tma_gemm_eligible(probs, count)) return tma_gemm_launch(st, probs, count, transA, transB);
        return tc_gemm_launch(st, probs, count, transA, transB);
    }
    GemmGroup grp;
    memset(&grp, 0, sizeof(grp));
    grp.count = count;
    int z = 0, maxM = 0, minN = 1 << 30;
    for (int i = 0; i < count; ++i) {
        grp.p[i] = probs[i];
        NATS_REQUIRE(probs[i].splitk >= 1 && probs[i].splitk <= kGemmMaxSplit && probs[i].batch >= 1, "gemm split/batch");
        NATS_REQUIRE(probs[i].splitk == 1 || !probs[i].accumulate, "split-K cannot accumulate in place");
        NATS_REQUIRE(probs[i].kchunk % 16 == 0 && probs[i].kchunk > 0, "kchunk");
        grp.zstart[i] = z;
        z += probs[i].batch * probs[i].splitk;
        maxM = max(maxM, probs[i].M);
        minN = min(minN, probs[i].N);
    }
    grp.zstart[count] = z;
    for (int i = count; i < kGemmMaxGroup; ++i) grp.zstart[i + 1] = z;
    if (maxM == 0) return 0;
    if (cfg == GEMM_CFG_AUTO) {
        if (maxM <= 32) cfg = GEMM_CFG_SMALLM;
        else if (maxM >= 512 && minN >= 512) cfg = GEMM_CFG_BIG;
        else cfg = GEMM_CFG_MID;
    }
    switch (cfg) {
        case GEMM_CFG_BIG: return launch_cfg<128, 128, 8, 8, 8>(st, grp, transA, transB);
        case GEMM_CFG_MID: return launch_cfg<64, 64, 16, 4, 4>(st, grp, transA, transB);
        case GEMM_CFG_SMALLM: return launch_cfg<32, 128, 16, 4, 4>(st, grp, transA, transB);
        default: break;
    }
    set_error("gemm_launch: bad cfg %d", cfg);
    return 2;
}

int gemm_step_cfg(int M) { return M <= 32 ? GEMM_CFG_SMALLM : GEMM_CFG_MID; }

int gemm_pick_split(const nats_ctx* ctx, int M, int N, int K, int groups) {
    int tiles;
    if (g_use_tc && (M >= 128 || N >= 128) && K >= 32) {
        const int a = M > N ? M : N, b = M > N ? N : M;      // 128-row side / N side of the tensor-core tile
        const int bn = b <= 32 ? 32 : b <= 64 ? 64 : b <= 112 ? 112 : 96;     // tile widths of tma_gemm_launch
        tiles = cdiv(a, 128) * cdiv(b, bn);
    } else {
        const int bm = (M <= 32) ? 32 : 64, bn = (M <= 32) ? 128 : 64;
        tiles = cdiv(N, bn) * cdiv(M, bm);
    }
    tiles *= (groups > 0 ? groups : 1);          // grouped launches (both encoder directions) share the machine
    int s = ctx->num_sms / (tiles > 0 ? tiles : 1);
    s = min(s, K / 64);
    s = min(s, kGemmMaxSplit);
    s = max(s, 1);
    // chunks are multiples of 32: drop splits that would be empty
    const int chunk = ((cdiv(K, s) + 31) / 32) * 32;
    return max(cdiv(K, chunk), 1);
}

int reduce_splits(cudaStream_t st, const float* part, int nsplit, long long strideP, int M, int N, int ldp,
                  float* out, int ldo, const float* bias, int accumulate) {
    const long long total = (long long)M * N;
    if (total == 0) return 0;
    const int block = 256;
    long long gl = (total + block - 1) / block;
    if (gl > 132LL * 16) gl = 132LL * 16;
    const int grid = (int)gl;
    ProfScope ps(st, K_REDUCE_SPLITS, 0.0, 4.0 * total * (nsplit + 1));
    NATS_CUDA_OK(launch_pdl(reduce_splits_kernel, dim3(grid), dim3(block), 0, st, part, nsplit, strideP, M, N, ldp, out, ldo, bias,
                            accumulate));
    return 0;
}

int gemm_auto(const nats_ctx* ctx, cudaStream_t st, GemmProblem p, bool transA, bool transB, float* scratch,
              long long scratch_floats) {
    if (p.M == 0 || p.N == 0) return 0;
    const bool tc = tc_eligible(&p, 1);
    int cfg = GEMM_CFG_AUTO;
    long long tiles;
    if (tc) {
        const int a = p.M > p.N ? p.M : p.N, b = p.M > p.N ? p.N : p.M;
        const bool swapped = p.M < 128 && p.N > p.M;
        const int nb = swapped ? p.M : p.N, ma = swapped ? p.N : p.M;
        (void)a; (void)b;
        const int bn = nb <= 32 ? 32 : nb <= 64 ? 64 : nb <= 112 ? 112 : 96;
        tiles = (long long)cdiv(ma, 128) * cdiv(nb, bn) * p.batch;
    } else {
        int bm, bn;
        if (p.M <= 32) { cfg = GEMM_CFG_SMALLM; bm = 32; bn = 128; }
        else if (p.M >= 512 && p.N >= 512) { cfg = GEMM_CFG_BIG; bm = 128; bn = 128; }
        else { cfg = GEMM_CFG_MID; bm = 64; bn = 64; }
        tiles = (long long)cdiv(p.M, bm) * cdiv(p.N, bn) * p.batch;
    }
    int splits = 1;
    if (tc && p.batch == 1 && tiles >= ctx->num_sms && p.K >= 4096 && scratch != nullptr) {
        // deep products whose tile count is not a multiple of the SM count (d[U|Ux] of the encoder at dim 1000: 8 x 32 tiles
        // of 128 x 96, K = 12768, on 132 SMs): pick the split-K factor that minimises waves x (k-blocks per CTA + fixed cost)
        // + the slab reduction.  The k-block cost is measured: that product unsplit took 692-726 us for 2 waves of 399
        // k-blocks on an H100 80GB HBM3 at a 700 W power limit, i.e. 0.9 us per 128 x 96 x 32 k-block of 3xTF32.  The fixed
        // cost per tile and the slab bandwidth (5 TB/s, L2-resident slabs) are estimates.
        double best = 1e30;
        for (int s2 = 1; s2 <= 4; ++s2) {
            if ((long long)s2 * p.M * p.N > scratch_floats) break;
            const long long waves = (tiles * s2 + ctx->num_sms - 1) / ctx->num_sms;
            double t = (double)waves * ((double)p.K / s2 / 32.0 * 0.9 + 3.0);
            if (s2 > 1) t += (double)(s2 + 1) * p.M * p.N * 4.0 / 5.0e6;
            if (t < best) { best = t; splits = s2; }
        }
    } else if (p.batch == 1 && tiles < ctx->num_sms && p.K >= 256 && scratch != nullptr) {
        long long want = ((tc ? 1LL : 2LL) * ctx->num_sms + tiles - 1) / tiles;
        if (want > p.K / 128) want = p.K / 128;
        splits = (int)want;
        splits = min(splits, kGemmMaxSplit);
        while (splits > 1 && (long long)splits * p.M * p.N > scratch_floats) --splits;
        if (splits < 1) splits = 1;
    }
    if (splits == 1) return gemm_launch(st, &p, 1, transA, transB, cfg);
    GemmProblem q = p;
    q.C = scratch; q.ldc = p.N; q.bias = nullptr; q.accumulate = 0;
    gemm_set_split(q, splits, (long long)p.M * p.N);
    NATS_TRY(gemm_launch(st, &q, 1, transA, transB, cfg));
    return reduce_splits(st, scratch, splits, (long long)p.M * p.N, p.M, p.N, p.N, p.C, p.ldc, p.bias, p.accumulate);
}

}  // namespace nats
