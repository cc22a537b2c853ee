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
                               const float* __restrict__ ymask, const float* __restrict__ lse, float scale,
                               const float* __restrict__ weight, int B) {
    // rows on grid.x (2^31 - 1 blocks), vocabulary chunks on grid.y: rows = Ty*B exceeds the 65535 limit of grid.y for
    // large batches (e.g. batch 160 at maxlen 500)
    const int r = blockIdx.x;
    float w = (ymask ? ymask[r] : 1.f) * scale;
    if (weight) w *= weight[r % B];                              // row r = t*B + b carries sample b's weight
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
// Filtered sampling (an addition beyond the reference; the rule is nats_sample_step_many's in include/nats_b200.h).
// A cluster of 8 CTAs per row, 512 threads each; CTA r owns the contiguous slice [r*ceil(V/8), ...) of the row, which it
// reads once from global memory into shared memory (15 KB at |V| = 30000; any |V| up to ~430000) and keeps there through
// every pass: the weights w, then the top-k / top-p cut by radix select on the bit pattern of w (non-negative floats
// order as unsigned integers), then the inverse CDF in vocabulary order.
//   - Radix select: up to four 8-bit passes for top-k (bin counts) and four for top-p (bin mass).  Each CTA bins its
//     slice in shared memory with INTEGER atomics (counts, and masses in 2^-40 fixed point of the largest weight), so the
//     bins do not depend on the order of the adds; the 8 CTAs' bins are summed through distributed shared memory in rank
//     order, and every CTA picks the same bin with one warp scan.  Ties at the cut value are kept in index order.
//   - Draw: thread t owns a contiguous run of its CTA's slice; per-thread sums -> block prefix (fixed tree) -> CTA prefix
//     (rank order) give every word a cumulative sum; the smallest kept index whose cumulative sum exceeds u*Z wins.
// Every reduction has a fixed order, so a repeated run gives the same bits.
// ------------------------------------------------------------------------------------------------
constexpr int kSfCluster = 8, kSfThreads = 512, kSfWarps = kSfThreads / 32, kSfBins = 256;
constexpr float kSfFixed = 1099511627776.f;                             // 2^40: top-p masses in fixed point

// exclusive prefix of v over the block in thread order (a fixed tree: the same bits on every run); *total = block sum.
// Contains __syncthreads(): call from uniform control flow.  s_part: kSfWarps entries of shared memory.
template <class T>
__device__ __forceinline__ T sf_block_prefix(T v, T* s_part, T* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    T exc = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) exc = T(0);
    __syncthreads();                                                    // s_part may still be read by a previous call
    if (lane == 31) s_part[warp] = inc;
    __syncthreads();
    T before = T(0), all = T(0);
#pragma unroll
    for (int w = 0; w < kSfWarps; ++w) {
        const T t = s_part[w];
        if (w < warp) before += t;
        all += t;
    }
    *total = all;
    return before + exc;
}

__global__ void __cluster_dims__(kSfCluster, 1, 1) __launch_bounds__(kSfThreads)
    sample_filter_kernel(const float* __restrict__ probs, int V, const int32_t* __restrict__ row_done, int mask_unk,
                         int ban_eos, float inv_t, int unit_t, int top_k, float top_p, uint64_t seed, int step, uint64_t row_base,
                         int32_t* __restrict__ pick) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ uint32_t s_w[];                                   // this CTA's slice: p, then the bits of w
    __shared__ uint32_t s_cnt[2][kSfBins];                              // per-pass bins (ping-pong: one cluster barrier
    __shared__ unsigned long long s_mass[2][kSfBins];                   // per pass suffices)
    __shared__ unsigned long long s_tot[kSfBins];                       // the cluster's bins of the current pass
    __shared__ uint32_t s_totc[kSfBins];
    __shared__ float s_pf[kSfWarps];
    __shared__ int s_pi[kSfWarps];
    __shared__ int s_bf[kSfWarps], s_bl[kSfWarps];
    __shared__ unsigned long long s_sel[3];                             // chosen bin, quantity above it, top-p target
    __shared__ float s_xf[2];                                           // cluster exchange slots, each written once
    __shared__ int s_xi[5];
    const int row = blockIdx.y;
    if (row_done != nullptr && row_done[row] != 0) return;              // the same for all 8 CTAs of the row
    const int rank = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int seglen = (V + kSfCluster - 1) / kSfCluster;
    const int base = rank * seglen;
    const int len = max(0, min(V, base + seglen) - base);
    const float* prow = probs + (long long)row * V + base;

    // 1. admissible probabilities (n-gram bans are already 0 in probs; UNK when mask_unk, EOS when ban_eos -- probs keeps
    // their f_next values, which the bookkeeping reads), their maximum and count
    float mx = 0.f;
    int npos = 0;
    for (int i = tid; i < len; i += kSfThreads) {
        float x = __ldg(prow + i);
        if (!(x > 0.f) || (mask_unk && base + i == 1) || (ban_eos && base + i == 0)) x = 0.f;
        s_w[i] = __float_as_uint(x);
        mx = fmaxf(mx, x);
        npos += x > 0.f ? 1 : 0;
    }
    mx = block_max(mx, s_pf);
    {
        int ntot;
        sf_block_prefix<int>(npos, s_pi, &ntot);                        // the block count (the prefix is not needed)
        npos = ntot;
    }
    if (tid == 0) { s_xf[0] = mx; s_xi[0] = npos; }
    cluster.sync();
    float pmax = 0.f;
    npos = 0;
#pragma unroll
    for (int q = 0; q < kSfCluster; ++q) {
        pmax = fmaxf(pmax, *cluster.map_shared_rank(&s_xf[0], q));
        npos += *cluster.map_shared_rank(&s_xi[0], q);
    }

    int result = 0;                                                     // no admissible word: the row ends with word 0
    if (npos > 0) {
        // 2. weights w = (p / p_max)^(1/T) (T = 1: w = p), and how many are > 0: for T < 1 the power underflows to 0 for
        // small p (T = 0.1: p / p_max below ~3e-5), so fewer words may carry weight than are admissible
        int nw = 0;
        for (int i = tid; i < len; i += kSfThreads) {
            const float x = __uint_as_float(s_w[i]);
            const float w = unit_t ? x : (x > 0.f ? powf(x / pmax, inv_t) : 0.f);
            s_w[i] = __float_as_uint(w);
            nw += w > 0.f ? 1 : 0;
        }
        const float qs = kSfFixed / (unit_t ? pmax : 1.f);              // the largest weight -> 2^40
        {
            int ntot;
            sf_block_prefix<int>(nw, s_pi, &ntot);                      // (its barriers also order the s_w stores)
            if (tid == 0) s_xi[4] = ntot;
        }
        cluster.sync();
        nw = 0;
#pragma unroll
        for (int q = 0; q < kSfCluster; ++q) nw += *cluster.map_shared_rank(&s_xi[4], q);   // >= 1: p_max itself has w = 1

        // 3. the cut: keep every word whose key (bits of w) is > cut, and the first `ties` words (index order) with key == cut
        uint32_t cut = 0u;
        unsigned long long ties = 0ull;
        int pass = 0;
        // one radix pass over the keys below `prefix` (the top 8*d bits of the cut found so far); members: key > 0 and,
        // when the top-k cut is on, key > kcut plus `kties` copies of kcut.  mode 0 selects by count, mode 1 by mass.
        auto radix = [&](int mode, int d, uint32_t prefix, unsigned long long& rem, uint32_t kcut, unsigned long long kties,
                         int total_target, float frac) -> uint32_t {
            const int shift = 24 - 8 * d, buf = pass & 1;
            ++pass;
            for (int b = tid; b < kSfBins; b += kSfThreads) { s_cnt[buf][b] = 0u; s_mass[buf][b] = 0ull; }
            __syncthreads();
            for (int i = tid; i < len; i += kSfThreads) {
                const uint32_t key = s_w[i];
                if (key == 0u || key <= kcut) continue;
                if (d > 0 && (key >> (shift + 8)) != prefix) continue;
                const int bin = (key >> shift) & (kSfBins - 1);
                atomicAdd(&s_cnt[buf][bin], 1u);
                if (mode == 1) atomicAdd(&s_mass[buf][bin], (unsigned long long)__float2ull_rz(__uint_as_float(key) * qs));
            }
            if (tid == 0 && kties > 0ull && rank == 0 && (d == 0 || (kcut >> (shift + 8)) == prefix)) {   // the top-k ties
                const int bin = (kcut >> shift) & (kSfBins - 1);
                atomicAdd(&s_cnt[buf][bin], (uint32_t)kties);
                if (mode == 1) atomicAdd(&s_mass[buf][bin], kties * (unsigned long long)__float2ull_rz(__uint_as_float(kcut) * qs));
            }
            cluster.sync();
            for (int b = tid; b < kSfBins; b += kSfThreads) {
                unsigned long long m = 0ull;
                uint32_t c = 0u;
#pragma unroll
                for (int q = 0; q < kSfCluster; ++q) {
                    c += cluster.map_shared_rank(&s_cnt[buf][0], q)[b];
                    if (mode == 1) m += cluster.map_shared_rank(&s_mass[buf][0], q)[b];
                }
                s_totc[b] = c;
                s_tot[b] = mode == 1 ? m : (unsigned long long)c;
            }
            __syncthreads();
            if (warp == 0) {                                            // lane l: bins 255 - 8l .. 248 - 8l, descending
                if (lane == 0) { s_sel[0] = 0ull; s_sel[1] = 0ull; }    // never read stale: a crossing always exists
                __syncwarp();                                           // (want <= the members), this is only a guard
                unsigned long long own = 0ull;
#pragma unroll
                for (int e = 0; e < 8; ++e) own += s_tot[kSfBins - 1 - 8 * lane - e];
                unsigned long long inc = own;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += y;
                }
                unsigned long long want = rem;
                if (total_target) {                                     // first top-p pass: ceil(P * total mass)
                    const unsigned long long all = __shfl_sync(0xffffffffu, inc, 31);
                    const unsigned long long t = (unsigned long long)ceil((double)frac * (double)all);
                    want = t < 1ull ? 1ull : (t > all ? all : t);
                    if (lane == 0) s_sel[2] = want;
                }
                const unsigned long long exc = inc - own;
                if (exc < want && want <= inc) {                        // exactly one lane
                    unsigned long long acc = exc;
                    int b = kSfBins - 1 - 8 * lane;
                    for (int e = 0; e < 7; ++e, --b) {
                        if (acc + s_tot[b] >= want) break;
                        acc += s_tot[b];
                    }
                    s_sel[0] = (unsigned long long)b;
                    s_sel[1] = acc;
                }
            }
            __syncthreads();
            const uint32_t b = (uint32_t)s_sel[0] & (kSfBins - 1);
            if (total_target) rem = s_sel[2];
            rem -= s_sel[1];
            if (d == 3) {                                               // the cut key: how many of its copies to keep
                const unsigned long long avail = s_totc[b];
                if (mode == 1) {
                    const unsigned long long wq = __float2ull_rz(__uint_as_float((prefix << 8) | b) * qs);
                    unsigned long long m = wq > 0ull ? (rem + wq - 1ull) / wq : avail;
                    rem = m < 1ull ? 1ull : (m > avail ? avail : m);
                } else {
                    rem = rem > avail ? avail : rem;
                }
            }
            __syncthreads();                                            // s_sel / s_tot are rewritten by the next pass
            return (prefix << 8) | b;
        };
        if (top_k >= 1 && top_k < nw) {                                 // else every word of positive weight is kept
            unsigned long long rem = (unsigned long long)top_k;
            uint32_t prefix = 0u;
            for (int d = 0; d < 4; ++d) prefix = radix(0, d, prefix, rem, 0u, 0ull, 0, 0.f);
            cut = prefix; ties = rem;
        }
        if (top_p < 1.f) {
            const uint32_t kcut = ties > 0ull ? cut : 0u;
            const unsigned long long kties = ties;
            unsigned long long rem = 0ull;
            uint32_t prefix = 0u;
            for (int d = 0; d < 4; ++d) prefix = radix(1, d, prefix, rem, kcut, kties, d == 0, top_p);
            cut = prefix; ties = rem;
        }

        // 4. tie ranks at the cut key, in vocabulary order (only when a cut is on)
        const int per = (len + kSfThreads - 1) / kSfThreads;
        const int r0 = min(len, tid * per), r1 = min(len, r0 + per);
        long long trank = 0;
        if (ties > 0ull) {
            int c = 0;
            for (int i = r0; i < r1; ++i) c += s_w[i] == cut ? 1 : 0;
            int ctot;
            const int cex = sf_block_prefix<int>(c, s_pi, &ctot);
            if (tid == 0) s_xi[1] = ctot;
            cluster.sync();
            long long off = 0;
            for (int q = 0; q < rank; ++q) off += *cluster.map_shared_rank(&s_xi[1], q);
            trank = off + cex;
        }
        auto kept = [&](uint32_t key, long long& tr) -> bool {
            if (key == cut && key != 0u) return (unsigned long long)(tr++) < ties;
            return key > cut;
        };

        // 5. kept sums in vocabulary order: thread run -> block prefix -> CTA prefix in rank order
        float s = 0.f;
        int last = -1;
        {
            long long tr = trank;
            for (int i = r0; i < r1; ++i) {
                const uint32_t key = s_w[i];
                if (kept(key, tr)) { s += __uint_as_float(key); last = base + i; }
            }
        }
        float ctot;
        const float sex = sf_block_prefix<float>(s, s_pf, &ctot);
        if (tid == 0) s_xf[1] = ctot;
        cluster.sync();
        float off = 0.f, Z = 0.f;
#pragma unroll
        for (int q = 0; q < kSfCluster; ++q) {
            const float t = *cluster.map_shared_rank(&s_xf[1], q);
            if (q < rank) off += t;
            Z += t;
        }

        // 6. the draw: the smallest kept index v with u*Z < (cumulative kept weight through v); rounding: the last kept word
        const float uz = uniform01(seed, (uint64_t)step, row_base + (uint64_t)row) * Z;
        int found = 0x7fffffff;
        if (Z > 0.f) {
            float c = off + sex;
            long long tr = trank;
            for (int i = r0; i < r1; ++i) {
                const uint32_t key = s_w[i];
                if (kept(key, tr)) {
                    c += __uint_as_float(key);
                    if (uz < c) { found = base + i; break; }
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {                              // block min of `found`, max of `last`
            found = min(found, __shfl_xor_sync(0xffffffffu, found, o));
            last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
        }
        if (lane == 0) { s_bf[warp] = found; s_bl[warp] = last; }
        __syncthreads();
        int bf = 0x7fffffff, bl = -1;
#pragma unroll
        for (int w = 0; w < kSfWarps; ++w) { bf = min(bf, s_bf[w]); bl = max(bl, s_bl[w]); }
        if (tid == 0) { s_xi[2] = bf; s_xi[3] = bl; }
        cluster.sync();
        int gf = 0x7fffffff, gl = -1;
#pragma unroll
        for (int q = 0; q < kSfCluster; ++q) {
            gf = min(gf, *cluster.map_shared_rank(&s_xi[2], q));
            gl = max(gl, *cluster.map_shared_rank(&s_xi[3], q));
        }
        if (Z > 0.f && gl >= 0) result = gf != 0x7fffffff ? gf : gl;
    }
    if (rank == 0 && tid == 0) pick[row] = result;
    cluster.sync();                                                     // remote reads done before any CTA exits
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
                    const float* lse, float scale, const float* weight, int B) {
    if (rows == 0) return 0;
    int gy = cdiv(V, 256 * 4);
    if (gy < 1) gy = 1;
    if (gy > 65535) gy = 65535;
    dim3 grid(rows, gy);
    ProfScope ps(st, K_DLOGITS, 0.0, 8.0 * rows * V);
    dlogits_kernel<<<grid, 256, 0, st>>>(logits, rows, V, y, ymask, lse, scale, weight, B);
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

int sample_filter(cudaStream_t st, const float* probs, int rows, int V, const int32_t* row_done, int mask_unk, int ban_eos,
                  float temperature, int top_k, float top_p, uint64_t seed, int step, uint64_t row_base, int32_t* pick) {
    NATS_REQUIRE(rows >= 1 && rows <= 65535 && V >= 2, "sample_filter shape");
    NATS_REQUIRE(temperature > 0.f && top_k >= 0 && top_p > 0.f && top_p <= 1.f, "sample_filter arguments");
    const size_t smem = (size_t)((V + kSfCluster - 1) / kSfCluster) * sizeof(uint32_t);
    if (smem > 48 * 1024) {                                                // beyond the default: opt in (up to the SM's limit)
        NATS_CUDA_OK(cudaFuncSetAttribute(sample_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    ProfScope ps(st, K_SAMPLE, 0.0, 4.0 * rows * V);
    sample_filter_kernel<<<dim3(kSfCluster, rows), kSfThreads, smem, st>>>(probs, V, row_done, mask_unk, ban_eos,
                                                                          1.f / temperature, temperature == 1.f ? 1 : 0, top_k,
                                                                          top_p, seed, step, row_base, pick);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace nats
