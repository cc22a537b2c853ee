// ops_att.cu -- Bahdanau attention with distraction (nats.py:527-546, 569-570): forward and backward.
//
// Forward, per decoder step:
//   att_scores_kernel   e[b,t]  = U_att . tanh(pctx[t,b,:] + ps[b,:] + acc_alpha[b,t]*D_wei) + c_att
//   att_context_kernel  alpha   = masked softmax_t(e);  c_raw = sum_t alpha[t] cc[t,b,:]   <-- the HBM-bound stream
//                       ctx     = tanh(U_con*c_raw + W_con*acc_ctx);  acc_ctx += m*ctx;  acc_alpha += m*alpha
//   The [Tx, C] slab of encoder states of one sample is streamed through shared memory by the TMA engine
//   (cp.async.bulk + mbarrier ring, one elected warp issues, all warps consume); the grid is
//   (column slices) x (samples) so that >= 2 CTAs per SM keep ~50 KB of bulk copies in flight each.
// Backward, per decoder step: att_bwd_ctx_kernel, att_bwd_dalpha_kernel (re-streams cc), att_bwd_softmax_kernel.
#include "ops.cuh"
#include "tc_common.cuh"

#include <cooperative_groups.h>
#include <cstdlib>

namespace nats {

namespace {

constexpr int kAttThreads = 256;
constexpr int kRowsPerCta = 32;   // scores kernel: rows of Tx per CTA
constexpr int kBwdRows = 16;      // backward kernels: rows of Tx per CTA (more CTAs in flight for the cc re-stream)
constexpr int kStages = 4;        // context kernel: tile ring depth (7 stages measured no faster)
constexpr int kStageRows = 16;    // rows of cc per stage
constexpr int kMaxSlice = 256;    // columns per CTA (one per thread)
constexpr int kScoreAk = 8;       // scores kernel: register path for dim_att <= 256

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    const uint32_t addr = smem_u32(bar);
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!ok);
}

// ------------------------------------------------------------------ forward: energies
__global__ void __launch_bounds__(kAttThreads) att_scores_kernel(const __grid_constant__ AttFwd a) {
    extern __shared__ float sm[];
    pdl_trigger();
    pdl_wait();
    float* s_ps = sm;
    float* s_dw = sm + a.A;
    float* s_ua = sm + 2 * a.A;
    const int b = blockIdx.y;
    const int src = b / a.rows_per_src;
    const int len = a.src_len ? min(a.Tx, (int)a.src_len[src]) : a.Tx;      // energies past the source are never read
    const float* pctx_s = a.pctx + (long long)src * a.pctx_bstride;
    for (int i = threadIdx.x; i < a.A; i += blockDim.x) {
        const float s = sum_strided(a.ps_part + (long long)b * a.A + i, a.ps_stride, a.ps_nsplit);
        s_ps[i] = s;
        if (blockIdx.x == 0 && a.ps_save) a.ps_save[(long long)b * a.A + i] = s;
        s_dw[i] = __ldg(a.D_wei + i);
        s_ua[i] = __ldg(a.U_att + i);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float catt = __ldg(a.c_att);
    const int t_end = min(len, (int)(blockIdx.x + 1) * kRowsPerCta);
    if (a.A <= 32 * kScoreAk) {
        // all loads of a row are issued before the first tanh (a runtime-length load/tanh/add loop serialises one
        // memory round trip per 32 columns), and the next row's loads are in flight during this row's arithmetic
        float v[kScoreAk], vn[kScoreAk];
        float accv = 0.f, accn = 0.f;
        int t = blockIdx.x * kRowsPerCta + warp;
        auto fetch = [&](int tt, float (&dst)[kScoreAk], float& av) {
            if (tt < t_end) {
                const float* pr = pctx_s + (long long)tt * a.pctx_tstride;
                av = a.acc_alpha_in[(long long)b * a.Tx + tt];
#pragma unroll
                for (int k = 0; k < kScoreAk; ++k) dst[k] = (lane + 32 * k < a.A) ? __ldg(pr + lane + 32 * k) : 0.f;
            }
        };
        fetch(t, v, accv);
        for (; t < t_end; t += kAttThreads / 32) {
            fetch(t + kAttThreads / 32, vn, accn);
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < kScoreAk; ++k) {
                const int i = lane + 32 * k;
                if (i < a.A) s += s_ua[i] * tanhf(v[k] + s_ps[i] + accv * s_dw[i]);
            }
            s = warp_sum(s);
            if (lane == 0) a.escore[(long long)b * a.Tx + t] = s + catt;
#pragma unroll
            for (int k = 0; k < kScoreAk; ++k) v[k] = vn[k];
            accv = accn;
        }
        return;
    }
    for (int t = blockIdx.x * kRowsPerCta + warp; t < t_end; t += kAttThreads / 32) {
        const float accv = a.acc_alpha_in[(long long)b * a.Tx + t];
        const float* pr = pctx_s + (long long)t * a.pctx_tstride;
        float s = 0.f;
        for (int i = lane; i < a.A; i += 32) s += s_ua[i] * tanhf(__ldg(pr + i) + s_ps[i] + accv * s_dw[i]);
        s = warp_sum(s);
        if (lane == 0) a.escore[(long long)b * a.Tx + t] = s + catt;
    }
}

// ------------------------------------------------------------------ forward: softmax + context + distraction
// BULK: 0 = plain loads, 1 = one bulk copy per row, 2 = one tensor-map tile (16 rows x slice) per stage
template <int BULK>
__global__ void __launch_bounds__(kAttThreads) att_context_kernel(const __grid_constant__ AttFwd a, int slice_len,
                                                                 int slice_pad, const __grid_constant__ CUtensorMap cmap) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ float red[32];
    const int Txp = (a.Tx + 31) & ~31;
    float* s_alpha = reinterpret_cast<float*>(smem_raw);
    float* s_tile = s_alpha + Txp;
    uint64_t* bars = reinterpret_cast<uint64_t*>(s_tile + (BULK ? kStages * kStageRows * slice_pad : 0));

    const int b = blockIdx.y, tid = threadIdx.x;
    const int src = b / a.rows_per_src;
    const int Ts = a.src_len ? min(a.Tx, (int)a.src_len[src]) : a.Tx;     // positions of this row's source
    const int c0 = blockIdx.x * slice_len;
    const int len = min(slice_len, a.C - c0);
    const float* ccb = a.cc + (long long)src * a.cc_bstride + c0;
    const int nblk = (Ts + kStageRows - 1) / kStageRows;
    const unsigned long long keep_pol = l2_keep_policy(a.cc_keep);

    auto issue = [&](int blk) {   // executed by warp 0
        const int stage = blk % kStages;
        const int t0 = blk * kStageRows;
        const int rows = min(kStageRows, Ts - t0);
        const int lane = tid & 31;
        if (BULK == 2) {
            // the whole stage is ONE TMA instruction: box (slice_pad columns, 1 sample, 16 positions); out-of-range
            // columns / positions are zero-filled and count towards the transaction bytes
            if (lane == 0) {
                mbar_arrive_expect_tx(&bars[stage], (uint32_t)(kStageRows * slice_pad * 4));
                if (a.cc_keep > 0) {
                    asm volatile(
                        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
                        ::"r"(smem_u32(s_tile + (long long)stage * kStageRows * slice_pad)), "l"(reinterpret_cast<uint64_t>(&cmap)),
                        "r"(smem_u32(&bars[stage])), "r"(c0), "r"(src), "r"(t0), "l"(keep_pol)
                        : "memory");
                } else {
                    asm volatile(
                        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                        ::"r"(smem_u32(s_tile + (long long)stage * kStageRows * slice_pad)), "l"(reinterpret_cast<uint64_t>(&cmap)),
                        "r"(smem_u32(&bars[stage])), "r"(c0), "r"(src), "r"(t0)
                        : "memory");
                }
            }
            return;
        }
        if (lane == 0) mbar_arrive_expect_tx(&bars[stage], (uint32_t)(rows * len * 4));
        __syncwarp();
        if (lane < rows)
            bulk_g2s(s_tile + ((long long)stage * kStageRows + lane) * slice_pad,
                     ccb + (long long)(t0 + lane) * a.cc_tstride, (uint32_t)(len * 4), &bars[stage]);
    };

    pdl_trigger();
    if (BULK) {
        if (tid == 0) {
            if (BULK == 2) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&cmap)) : "memory");
            for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
            fence_barrier_init();
        }
        __syncthreads();
        // the encoder context cc is not written by any kernel of the decoder scan: its first tiles are requested
        // before the predecessor (the energies kernel) has finished
        if (tid < 32)
            for (int blk = 0; blk < kStages && blk < nblk; ++blk) issue(blk);
    }
    pdl_wait();

    // masked softmax over the source positions (nats.py:537-540); max taken over valid positions only; positions past
    // the row's source get weight 0 exactly
    float lmax = -INFINITY;
    for (int t = tid; t < Ts; t += kAttThreads) {
        const float e = a.escore[(long long)b * a.Tx + t];
        s_alpha[t] = e;
        const float mk = a.xmask ? a.xmask[(long long)t * a.n + b] : 1.f;
        if (mk > 0.f) lmax = fmaxf(lmax, e);
    }
    float mx = block_max(lmax, red);
    if (mx == -INFINITY) mx = 0.f;
    float lsum = 0.f;
    for (int t = tid; t < a.Tx; t += kAttThreads) {
        if (t >= Ts) { s_alpha[t] = 0.f; continue; }
        const float mk = a.xmask ? a.xmask[(long long)t * a.n + b] : 1.f;
        const float w = expf(s_alpha[t] - mx) * mk;
        s_alpha[t] = w;
        lsum += w;
    }
    const float S = block_sum(lsum, red);
    const float inv = 1.f / S;
    __syncthreads();

    // c_raw[c] = sum_t alpha[t] * cc[t, b, c]   (nats.py:541)
    float acc = 0.f;
    if (BULK) {
        for (int blk = 0; blk < nblk; ++blk) {
            const int stage = blk % kStages;
            mbar_wait(&bars[stage], (uint32_t)((blk / kStages) & 1));
            const int t0 = blk * kStageRows;
            const int rows = min(kStageRows, Ts - t0);
            if (tid < len) {
                const float* tp = s_tile + (long long)stage * kStageRows * slice_pad + tid;
#pragma unroll 4
                for (int r = 0; r < rows; ++r) acc = fmaf(s_alpha[t0 + r], tp[r * slice_pad], acc);
            }
            __syncthreads();   // every thread is done with this stage before it is refilled
            if (tid < 32 && blk + kStages < nblk) issue(blk + kStages);
        }
    } else {
        if (tid < len) {
            const float* p = ccb + tid;
            int t = 0;
            for (const int t8 = Ts & ~7; t < t8; t += 8) {
                float v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) v[k] = __ldg(p + (long long)(t + k) * a.cc_tstride);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc = fmaf(s_alpha[t + k], v[k], acc);
            }
            for (; t < Ts; ++t) acc = fmaf(s_alpha[t], __ldg(p + (long long)t * a.cc_tstride), acc);
        }
    }

    const float m = a.ymask ? a.ymask[b] : 1.f;
    if (tid < len) {
        const int gc = c0 + tid;
        const long long o = (long long)b * a.C + gc;
        const float craw = acc * inv;
        const float accc = a.acc_ctx_in[o];
        const float cv = tanhf(__ldg(a.U_con + gc) * craw + __ldg(a.W_con + gc) * accc);   // nats.py:545-546
        if (a.craw_out) a.craw_out[o] = craw;
        a.ctx_out[o] = cv;
        a.acc_ctx_out[o] = accc + m * cv;                                                   // nats.py:569
    }
    if (blockIdx.x == 0) {
        for (int t = tid; t < a.Tx; t += kAttThreads) {
            const long long o = (long long)b * a.Tx + t;
            const float al = s_alpha[t] * inv;
            a.alpha_out[o] = al;
            a.acc_alpha_out[o] = a.acc_alpha_in[o] + m * al;                                // nats.py:570
        }
    }
}


// ------------------------------------------------------------------ forward, beam search: ONE source for all rows
// f_next of beam search runs k hypotheses against the encoder states of a single sentence (zero batch stride): the
// [Tx, C] slab is the same for every row.  The per-(row, column slice) grid above re-streams it k times with a handful of
// active lanes; here a cluster of 8 CTAs splits the source positions, every CTA walks its positions once for a 128-column
// group and ALL rows (n <= 16 accumulator sets in registers), the 8 partial sums meet in distributed shared memory in a
// fixed order, and rank r finishes 16 of the 128 columns (nats.py:541-546, 569-570).
// Beam search over a group of sentences (rows_per_src = k, src_len set): blockIdx.z = source; its cluster takes the k rows
// of that source, walks only the source's own positions, and writes alpha = 0 past them.
constexpr int kBcCluster = 8, kBcCols = 128, kBcMaxN = 16, kBcWarps = kAttThreads / 32;

__global__ void __cluster_dims__(kBcCluster, 1, 1) __launch_bounds__(kAttThreads)
    att_context_bcast_kernel(const __grid_constant__ AttFwd a, int chunk) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float bc_sm[];
    const int src = blockIdx.z, r0 = src * a.rows_per_src;       // rows [r0, r0 + nr) read this source
    const int nr = min(a.rows_per_src, a.n - r0);
    const int Ts = a.src_len ? min(a.Tx, (int)a.src_len[src]) : a.Tx;
    float* s_alpha = bc_sm;                                   // [nr][chunk] normalised weights of this CTA's positions
    float* s_part = bc_sm + (((size_t)a.rows_per_src * chunk + 3) & ~(size_t)3);   // [nr][128] partial context (16-byte aligned)
    __shared__ float s_mx[kBcMaxN], s_inv[kBcMaxN];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = blockIdx.x, c0 = blockIdx.y * kBcCols;
    const int my_chunk = (Ts + kBcCluster - 1) / kBcCluster;   // <= chunk (the shared-memory stride)
    const int t0 = rank * my_chunk, t1 = min(Ts, t0 + my_chunk);
    const float* ccs = a.cc + (long long)src * a.cc_bstride;
    pdl_trigger();
    pdl_wait();
    // masked softmax statistics of every row over ALL positions (nats.py:537-540); max over valid positions only
    for (int b = warp; b < nr; b += kBcWarps) {
        const int row = r0 + b;
        float mx = -INFINITY;
        for (int t = lane; t < Ts; t += 32) {
            const float mk = a.xmask ? a.xmask[(long long)t * a.n + row] : 1.f;
            if (mk > 0.f) mx = fmaxf(mx, a.escore[(long long)row * a.Tx + t]);
        }
        mx = warp_max(mx);
        if (mx == -INFINITY) mx = 0.f;
        float sum = 0.f;
        for (int t = lane; t < Ts; t += 32) {
            const float mk = a.xmask ? a.xmask[(long long)t * a.n + row] : 1.f;
            sum += expf(a.escore[(long long)row * a.Tx + t] - mx) * mk;
        }
        sum = warp_sum(sum);
        if (lane == 0) { s_mx[b] = mx; s_inv[b] = 1.f / sum; }
    }
    for (int i = tid; i < nr * kBcCols; i += kAttThreads) s_part[i] = 0.f;
    __syncthreads();
    for (int i = tid; i < nr * (t1 - t0); i += kAttThreads) {
        const int b = i / (t1 - t0), tl = i - b * (t1 - t0), t = t0 + tl, row = r0 + b;
        const float mk = a.xmask ? a.xmask[(long long)t * a.n + row] : 1.f;
        const float al = expf(a.escore[(long long)row * a.Tx + t] - s_mx[b]) * mk * s_inv[b];
        s_alpha[b * chunk + tl] = al;
        if (blockIdx.y == 0) {
            const float m = a.ymask ? a.ymask[row] : 1.f;
            const long long o = (long long)row * a.Tx + t;
            a.alpha_out[o] = al;
            a.acc_alpha_out[o] = a.acc_alpha_in[o] + m * al;                               // nats.py:570
        }
    }
    if (blockIdx.y == 0 && Ts < a.Tx) {                       // positions past the source: alpha = 0
        const int pad = a.Tx - Ts;
        for (int i = rank * kAttThreads + tid; i < nr * pad; i += kBcCluster * kAttThreads) {
            const int b = i / pad;
            const long long o = (long long)(r0 + b) * a.Tx + Ts + (i - b * pad);
            a.alpha_out[o] = 0.f;
            a.acc_alpha_out[o] = a.acc_alpha_in[o];
        }
    }
    __syncthreads();

    // c_raw[b, c] = sum_t alpha[b, t] * cc[t, c]: lane = 4 columns, warp = every 8th position of the chunk
    float4 acc[kBcMaxN];
#pragma unroll
    for (int b = 0; b < kBcMaxN; ++b) acc[b] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int col = c0 + lane * 4;
    if (col < a.C) {
        const float* base = ccs + col;
        int t = t0 + warp;
        for (; t + 3 * kBcWarps < t1; t += 4 * kBcWarps) {
            float4 v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                v[j] = __ldg(reinterpret_cast<const float4*>(base + (long long)(t + j * kBcWarps) * a.cc_tstride));
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int tl = t + j * kBcWarps - t0;
#pragma unroll
                for (int b = 0; b < kBcMaxN; ++b)
                    if (b < nr) {
                        const float al = s_alpha[b * chunk + tl];
                        acc[b].x = fmaf(al, v[j].x, acc[b].x); acc[b].y = fmaf(al, v[j].y, acc[b].y);
                        acc[b].z = fmaf(al, v[j].z, acc[b].z); acc[b].w = fmaf(al, v[j].w, acc[b].w);
                    }
            }
        }
        for (; t < t1; t += kBcWarps) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(base + (long long)t * a.cc_tstride));
            const int tl = t - t0;
#pragma unroll
            for (int b = 0; b < kBcMaxN; ++b)
                if (b < nr) {
                    const float al = s_alpha[b * chunk + tl];
                    acc[b].x = fmaf(al, v.x, acc[b].x); acc[b].y = fmaf(al, v.y, acc[b].y);
                    acc[b].z = fmaf(al, v.z, acc[b].z); acc[b].w = fmaf(al, v.w, acc[b].w);
                }
        }
    }
    for (int w = 0; w < kBcWarps; ++w) {                      // warps add in order: deterministic
        if (warp == w) {
#pragma unroll
            for (int b = 0; b < kBcMaxN; ++b)
                if (b < nr) {
                    float4* p = reinterpret_cast<float4*>(s_part + b * kBcCols + lane * 4);
                    float4 q = *p;
                    q.x += acc[b].x; q.y += acc[b].y; q.z += acc[b].z; q.w += acc[b].w;
                    *p = q;
                }
        }
        __syncthreads();
    }
    cluster.sync();
    // rank r finishes columns [16 r, 16 r + 16) of the group for every row
    constexpr int kPer = kBcCols / kBcCluster;
    if (tid < nr * kPer) {
        const int b = tid / kPer, cl = rank * kPer + (tid - b * kPer), gc = c0 + cl, row = r0 + b;
        if (gc < a.C) {
            float craw = 0.f;
#pragma unroll
            for (int q = 0; q < kBcCluster; ++q) craw += cluster.map_shared_rank(s_part, q)[b * kBcCols + cl];
            const float m = a.ymask ? a.ymask[row] : 1.f;
            const long long o = (long long)row * a.C + gc;
            const float accc = a.acc_ctx_in[o];
            const float cv = tanhf(__ldg(a.U_con + gc) * craw + __ldg(a.W_con + gc) * accc);   // nats.py:545-546
            if (a.craw_out) a.craw_out[o] = craw;
            a.ctx_out[o] = cv;
            a.acc_ctx_out[o] = accc + m * cv;                                                   // nats.py:569
        }
    }
    cluster.sync();                                           // remote reads done before any CTA exits
}

// ------------------------------------------------------------------ backward kernels
__global__ void att_bwd_ctx_kernel(const __grid_constant__ AttBwd a) {
    pdl_trigger();
    pdl_wait();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.B * a.C) return;
    const int b = idx / a.C, c = idx - b * a.C;
    const float m = a.ymask ? a.ymask[b] : 1.f;
    float d = a.dctx_a ? a.dctx_a[idx] : 0.f;
    d = sum_strided(a.dctx_part + idx, a.dctx_stride, a.dctx_nsplit, d);
    const float dacc = a.dacc_ctx_in[idx];
    d += m * dacc;
    const float cv = a.ctx[idx];
    const float dq = d * (1.f - cv * cv);
    a.dq[idx] = dq;
    a.dcraw[idx] = dq * __ldg(a.U_con + c);
    a.dacc_ctx_out[idx] = dacc + dq * __ldg(a.W_con + c);
}

__global__ void __launch_bounds__(kAttThreads) att_bwd_dalpha_kernel(const __grid_constant__ AttBwd a) {
    extern __shared__ __align__(16) float s_dcraw[];
    __shared__ float s_dot[kAttThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < a.C; i += blockDim.x) s_dcraw[i] = a.dcraw[(long long)b * a.C + i];
    __syncthreads();
    const float m = a.ymask ? a.ymask[b] : 1.f;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool vec = ((a.C & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.cc) & 15) == 0);
    const bool keep = a.cc_keep > 0;
    const unsigned long long keep_pol = l2_keep_policy(a.cc_keep);
    const int t_end = min(a.Tx, (int)(blockIdx.x + 1) * kBwdRows);
    float dot = 0.f;                                   // this warp's share of sum_t alpha[t] * dalpha[t]
    for (int t = blockIdx.x * kBwdRows + warp; t < t_end; t += kAttThreads / 32) {
        const float* row = a.cc + ((long long)t * a.B + b) * a.C;
        float s = 0.f;
        if (vec) {
            const int n4 = a.C >> 2;
            const float4* d4 = reinterpret_cast<const float4*>(s_dcraw);
            // eight 16-byte loads per lane in flight before the first dependent FMA (the accumulation order is unchanged)
            for (int i0 = lane; i0 < n4; i0 += 32 * 8) {
                float4 v[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int i = i0 + 32 * k;
                    if (i < n4) v[k] = keep ? ldg_stream4_hint(row + 4 * i, keep_pol) : ldg_stream4(row + 4 * i);
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const int i = i0 + 32 * k;
                    if (i < n4) {
                        const float4 d = d4[i];
                        s = fmaf(v[k].x, d.x, s); s = fmaf(v[k].y, d.y, s); s = fmaf(v[k].z, d.z, s); s = fmaf(v[k].w, d.w, s);
                    }
                }
            }
        } else {
            for (int i = lane; i < a.C; i += 32) s = fmaf(__ldg(row + i), s_dcraw[i], s);
        }
        s = warp_sum(s);
        if (lane == 0) {
            const long long o = (long long)b * a.Tx + t;
            const float da = s + m * a.dacc_alpha[o];
            a.dalpha[o] = da;
            dot = fmaf(a.alpha[o], da, dot);
        }
    }
    if (lane == 0) s_dot[warp] = dot;
    __syncthreads();
    if (threadIdx.x == 0) {
        float d = 0.f;
#pragma unroll
        for (int w = 0; w < kAttThreads / 32; ++w) d += s_dot[w];
        a.dot_part[(long long)b * gridDim.x + blockIdx.x] = d;       // fixed-order partial of the softmax-backward dot
    }
}

constexpr int kSoftThreads = 256;
constexpr int kSoftWarps = kSoftThreads / 32;
constexpr int kMaxAk = 8;   // A <= 256

// grid (chunks of kBwdRows source positions, B).  Output partials part[b][chunk][3A+1] = {d ps, d U_att, d D_wei, d c_att}
__global__ void __launch_bounds__(kSoftThreads) att_bwd_softmax_kernel(const __grid_constant__ AttBwd a) {
    extern __shared__ float sm[];
    __shared__ float s_dot;
    pdl_trigger();
    pdl_wait();
    const int A = a.A, Tx = a.Tx, b = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x, tid = threadIdx.x;
    float* s_ps = sm;                 // [A]
    float* s_dw = s_ps + A;           // [A]
    float* s_ua = s_dw + A;           // [A]
    float* s_part = s_ua + A;         // [warps][3][A]
    float* s_gc = s_part + kSoftWarps * 3 * A;   // [warps]
    if (tid < 32) {                   // dot = sum_t alpha dalpha, from the fixed-order partials of the dalpha kernel
        float d = 0.f;
        for (int i = tid; i < nchunks; i += 32) d += a.dot_part[(long long)b * nchunks + i];
        d = warp_sum(d);
        if (tid == 0) s_dot = d;
    }
    for (int i = tid; i < A; i += kSoftThreads) {
        s_ps[i] = a.ps[(long long)b * A + i];
        s_dw[i] = __ldg(a.D_wei + i);
        s_ua[i] = __ldg(a.U_att + i);
    }
    __syncthreads();
    const float dot = s_dot;
    const int warp = tid >> 5, lane = tid & 31;
    float r_dps[kMaxAk], r_gu[kMaxAk], r_gd[kMaxAk];
#pragma unroll
    for (int k = 0; k < kMaxAk; ++k) { r_dps[k] = 0.f; r_gu[k] = 0.f; r_gd[k] = 0.f; }
    float gc = 0.f;
    const int t_end = min(Tx, (chunk + 1) * kBwdRows);
    for (int t = chunk * kBwdRows + warp; t < t_end; t += kSoftWarps) {
        const long long o = (long long)b * Tx + t;
        const long long base = ((long long)t * a.B + b) * A;
        // every load of the row first (pctx and dpctx may alias as far as the compiler knows: interleaving the
        // read-modify-write with the loads serialises one memory round trip per 32 columns)
        float pv[kMaxAk], dv[kMaxAk];
#pragma unroll
        for (int k = 0; k < kMaxAk; ++k) {
            const int i = lane + 32 * k;
            pv[k] = (i < A) ? __ldg(a.pctx + base + i) : 0.f;
            dv[k] = (i < A) ? a.dpctx[base + i] : 0.f;
        }
        const float al = a.alpha[o], dal = a.dalpha[o];
        const float accv = a.acc_alpha[o];
        const float de = al * (dal - dot);                           // masked-softmax backward (nats.py:537-540)
        gc += de;
        float rowsum = 0.f;
#pragma unroll
        for (int k = 0; k < kMaxAk; ++k) {
            const int i = lane + 32 * k;
            if (i < A) {
                const float z = tanhf(pv[k] + s_ps[i] + accv * s_dw[i]);
                const float dzp = de * s_ua[i] * (1.f - z * z);
                a.dpctx[base + i] = dv[k] + dzp;
                r_dps[k] += dzp;
                r_gu[k] += de * z;
                r_gd[k] += accv * dzp;
                rowsum += dzp * s_dw[i];
            }
        }
        rowsum = warp_sum(rowsum);
        if (lane == 0) a.dacc_alpha[o] += rowsum;                    // through nats.py:532
    }
#pragma unroll
    for (int k = 0; k < kMaxAk; ++k) {
        const int i = lane + 32 * k;
        if (i < A) {
            s_part[(warp * 3 + 0) * A + i] = r_dps[k];
            s_part[(warp * 3 + 1) * A + i] = r_gu[k];
            s_part[(warp * 3 + 2) * A + i] = r_gd[k];
        }
    }
    if (lane == 0) s_gc[warp] = gc;       // every lane of the warp holds the same gc (de is warp-uniform per row)
    __syncthreads();
    float* out = a.soft_part + ((long long)b * nchunks + chunk) * (3 * A + 1);
    for (int i = tid; i < 3 * A; i += kSoftThreads) {
        const int q = i / A, ia = i - q * A;
        float d = 0.f;
        for (int w = 0; w < kSoftWarps; ++w) d += s_part[(w * 3 + q) * A + ia];
        out[i] = d;
    }
    if (tid == 0) {
        float d = 0.f;
        for (int w = 0; w < kSoftWarps; ++w) d += s_gc[w];
        out[3 * A] = d;
    }
}

// dps[b,:] = sum_chunks part ; gatt_part[b,:] += sum_chunks part   (fixed order)
__global__ void att_bwd_reduce_kernel(const __grid_constant__ AttBwd a, int nchunks) {
    pdl_trigger();
    const int A = a.A, b = blockIdx.x, W = 3 * A + 1;
    const int i = blockIdx.y * blockDim.x + threadIdx.x;      // one element per thread
    const float* src = a.soft_part + (long long)b * nchunks * W + i;
    pdl_wait();
    if (i >= W) return;
    const float d = sum_strided(src, W, nchunks);
    if (i < A) a.dps[(long long)b * A + i] = d;
    else a.gatt_part[(long long)b * (2 * A + 1) + (i - A)] += d;     // [dU_att | dD_wei | dc_att]
}

inline size_t context_smem(int Tx, bool bulk, int slice_pad) {
    size_t s = (size_t)((Tx + 31) & ~31) * 4;
    if (bulk) s += (size_t)kStages * kStageRows * slice_pad * 4 + kStages * 8;
    return s + 16;
}

}  // namespace

template <class K>
static int set_max_dyn_smem(K kernel, int optin, int* out_limit) {
    cudaFuncAttributes fa;
    NATS_CUDA_OK(cudaFuncGetAttributes(&fa, kernel));
    const int lim = optin - (int)fa.sharedSizeBytes;      // dynamic + static must fit the opt-in limit
    NATS_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    if (out_limit && lim < *out_limit) *out_limit = lim;
    return 0;
}

static int g_att_dyn_limit = 0;
static int g_cc_keep = 0;
void attention_set_cc_keep(int mode) { g_cc_keep = mode < 0 ? 0 : (mode > 4 ? 4 : mode); }

int attention_setup(const nats_ctx* ctx) {
    int lim = ctx->max_smem_optin;
    NATS_TRY(set_max_dyn_smem(att_context_kernel<2>, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_context_kernel<1>, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_context_kernel<0>, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_context_bcast_kernel, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_bwd_softmax_kernel, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_bwd_dalpha_kernel, ctx->max_smem_optin, &lim));
    NATS_TRY(set_max_dyn_smem(att_scores_kernel, ctx->max_smem_optin, &lim));
    g_att_dyn_limit = lim;
    return 0;
}

int attention_fwd(const nats_ctx* ctx, cudaStream_t st, const AttFwd& a_in) {
    AttFwd a = a_in;
    a.cc_keep = g_cc_keep;
    NATS_REQUIRE(a.Tx >= 1 && a.n >= 1, "attention shape");
    if (a.cc_bstride == 0) a.rows_per_src = a.n;           // every row reads the one source
    if (a.rows_per_src < 1) a.rows_per_src = 1;
    const int nsrc = cdiv(a.n, a.rows_per_src);
    {
        dim3 grid(cdiv(a.Tx, kRowsPerCta), a.n);
        ProfScope ps(st, K_ATT_SCORES, 0.0, 4.0 * a.Tx * (a.pctx_bstride == 0 ? 1 : nsrc) * a.A);
        NATS_CUDA_OK(launch_pdl(att_scores_kernel, grid, dim3(kAttThreads), 3 * a.A * sizeof(float), st, a));
    }
    // the cluster kernel serves rows grouped by source: one shared source, or the k rows of each sentence of a beam group
    static const int no_bcast = [] { const char* e = getenv("NATS_ATT_BCAST"); return e && atoi(e) == 0; }();
    if (!no_bcast && (a.cc_bstride == 0 || a.src_len != nullptr) && a.rows_per_src <= kBcMaxN && (a.C & 3) == 0 &&
        (a.cc_tstride & 3) == 0 && (a.cc_bstride & 3) == 0 && (reinterpret_cast<uintptr_t>(a.cc) & 15) == 0) {
        const int chunk = cdiv(a.Tx, kBcCluster);
        const size_t rows = (size_t)a.rows_per_src;
        const size_t smem = (((rows * chunk + 3) & ~(size_t)3) + rows * kBcCols) * sizeof(float);
        if (smem <= (size_t)g_att_dyn_limit && nsrc <= 65535) {
            ProfScope ps(st, K_ATT_CONTEXT, 2.0 * a.Tx * a.n * a.C, 4.0 * ((double)a.Tx * nsrc * a.C + 3.0 * a.n * a.Tx + 4.0 * a.n * a.C));
            NATS_CUDA_OK(launch_pdl(att_context_bcast_kernel, dim3(kBcCluster, cdiv(a.C, kBcCols), nsrc), dim3(kAttThreads), smem, st,
                                    a, chunk));
            return 0;
        }
    }
    // column slices: as many CTAs as fit in ONE co-resident wave of 2 CTAs per SM (a partial second wave would run at
    // the per-CTA latency-bound rate and cost as much as the first)
    int target = (2 * ctx->num_sms) / a.n;
    if (target < 1) target = 1;
    int slice = cdiv(a.C, target);
    slice = ((slice + 3) / 4) * 4;
    if (slice < 32) slice = 32;
    if (slice > kMaxSlice) slice = kMaxSlice;
    const int nslices = cdiv(a.C, slice);
    const int slice_pad = slice;   // multiple of 4 floats -> 16-byte aligned rows in shared memory
    const bool aligned = ((a.C & 3) == 0) && ((a.cc_tstride & 3) == 0) && ((a.cc_bstride & 3) == 0) &&
                         ((reinterpret_cast<uintptr_t>(a.cc) & 15) == 0);
    bool bulk = aligned;
    size_t smem = context_smem(a.Tx, bulk, slice_pad);
    if (bulk && smem > (size_t)g_att_dyn_limit) { bulk = false; smem = context_smem(a.Tx, false, slice_pad); }
    NATS_REQUIRE(smem <= (size_t)g_att_dyn_limit, "source too long for the attention kernel's shared memory");
    dim3 grid(nslices, a.n);
    ProfScope ps(st, K_ATT_CONTEXT, 2.0 * a.Tx * a.n * a.C,
                 4.0 * ((double)a.Tx * (a.cc_bstride == 0 ? 1 : nsrc) * a.C + 3.0 * a.n * a.Tx + 4.0 * a.n * a.C));
    CUtensorMap cmap;
    memset(&cmap, 0, sizeof(cmap));
    const bool tiled = bulk && tma_available() && a.cc_bstride >= a.C && a.cc_tstride >= (long long)nsrc * a.cc_bstride && slice_pad <= 256;
    if (tiled) NATS_TRY(tma_map_tile3d(a.cc, a.C, nsrc, a.Tx, a.cc_bstride, a.cc_tstride, slice_pad, 1, kStageRows, &cmap));
    if (tiled) NATS_CUDA_OK(launch_pdl(att_context_kernel<2>, grid, dim3(kAttThreads), smem, st, a, slice, slice_pad, cmap));
    else if (bulk) NATS_CUDA_OK(launch_pdl(att_context_kernel<1>, grid, dim3(kAttThreads), smem, st, a, slice, slice_pad, cmap));
    else NATS_CUDA_OK(launch_pdl(att_context_kernel<0>, grid, dim3(kAttThreads), smem, st, a, slice, slice_pad, cmap));
    return 0;
}

int attention_bwd(const nats_ctx* ctx, cudaStream_t st, const AttBwd& a_in) {
    AttBwd a = a_in;
    a.cc_keep = g_cc_keep;
    NATS_REQUIRE(a.A <= 32 * kMaxAk, "dim_att > 256 not supported by the attention backward kernel");
    {
        ProfScope ps(st, K_ATT_BWD_CTX);
        NATS_CUDA_OK(launch_pdl(att_bwd_ctx_kernel, dim3(cdiv(a.B * a.C, 512)), dim3(512), 0, st, a));
    }
    const int nchunks = cdiv(a.Tx, kBwdRows);
    NATS_REQUIRE(a.dot_part != nullptr && a.soft_part != nullptr, "attention backward scratch");
    {
        dim3 grid(nchunks, a.B);
        ProfScope ps(st, K_ATT_BWD_DALPHA, 2.0 * a.Tx * a.B * a.C, 4.0 * ((double)a.Tx * a.B * a.C + 2.0 * a.B * a.Tx));
        NATS_CUDA_OK(launch_pdl(att_bwd_dalpha_kernel, grid, dim3(kAttThreads), (size_t)a.C * sizeof(float), st, a));
    }
    {
        const size_t smem = ((size_t)3 * a.A + (size_t)kSoftWarps * 3 * a.A + kSoftWarps) * sizeof(float);
        dim3 grid(nchunks, a.B);
        ProfScope ps(st, K_ATT_BWD_SOFTMAX, 0.0, 12.0 * a.Tx * a.B * a.A);
        NATS_CUDA_OK(launch_pdl(att_bwd_softmax_kernel, grid, dim3(kSoftThreads), smem, st, a));
        NATS_CUDA_OK(launch_pdl(att_bwd_reduce_kernel, dim3(a.B, cdiv(3 * a.A + 1, 128)), dim3(128), 0, st, a, nchunks));
    }
    return 0;
}

}  // namespace nats
