// ops_beam.cu -- the distraction re-ranking terms of beam search (nats.py:982-995) and the history
// bookkeeping copies (nats.py:1015-1023) on device.
#include "ops.cuh"

#include <cooperative_groups.h>

namespace nats {

namespace {

// rows of a beam group that are not live in their sentence (counters [S][8] of beam_select; NULL = every row is live)
__device__ __forceinline__ bool beam_row_idle(const int32_t* counters, int k, int i) {
    if (counters == nullptr) return false;
    const int32_t* c = counters + (i / k) * 8;
    return c[2] != 0 || i - (i / k) * k >= c[0];
}

// one CTA per (history step s, hypothesis i): KL(alpha_s || alpha_now), cos-dist(ctx_s, ctx_now), cos-dist(h_s, h_now)
__global__ void __launch_bounds__(256) beam_pair_kernel(const float* __restrict__ hist_alpha,
                                                        const float* __restrict__ hist_ctx,
                                                        const float* __restrict__ hist_state, int len_cap, int hist_len,
                                                        int Tx, int C, int D, const float* __restrict__ cur_alpha,
                                                        const float* __restrict__ cur_ctx,
                                                        const float* __restrict__ cur_state, const int32_t* __restrict__ counters,
                                                        int k, float* __restrict__ scratch) {
    __shared__ float red[32];
    const int s = blockIdx.x, i = blockIdx.y, tid = threadIdx.x;
    if (beam_row_idle(counters, k, i)) return;
    const long long h = (long long)i * len_cap + s;
    float* out = scratch + ((long long)i * hist_len + s) * 3;
    {   // scipy.stats.entropy(pk, qk): both normalised to sum 1, sum pk*log(pk/qk) with 0*log(0) = 0  (nats.py:990)
        const float* p = hist_alpha + h * Tx;
        const float* q = cur_alpha + (long long)i * Tx;
        float sp = 0.f, sq = 0.f;
        for (int t = tid; t < Tx; t += 256) { sp += p[t]; sq += q[t]; }
        sp = block_sum(sp, red);
        sq = block_sum(sq, red);
        float kl = 0.f;
        for (int t = tid; t < Tx; t += 256) {
            const float pn = p[t] / sp, qn = q[t] / sq;
            if (pn > 0.f) kl += pn * logf(pn / qn);
        }
        kl = block_sum(kl, red);
        if (tid == 0) out[0] = kl;
    }
    {   // scipy.spatial.distance.cosine (nats.py:991)
        const float* u = hist_ctx + h * C;
        const float* v = cur_ctx + (long long)i * C;
        float uv = 0.f, uu = 0.f, vv = 0.f;
        for (int t = tid; t < C; t += 256) { const float a = u[t], b = v[t]; uv = fmaf(a, b, uv); uu = fmaf(a, a, uu); vv = fmaf(b, b, vv); }
        uv = block_sum(uv, red); uu = block_sum(uu, red); vv = block_sum(vv, red);
        if (tid == 0) out[1] = 1.f - uv / (sqrtf(uu) * sqrtf(vv));
    }
    {   // nats.py:992
        const float* u = hist_state + h * D;
        const float* v = cur_state + (long long)i * D;
        float uv = 0.f, uu = 0.f, vv = 0.f;
        for (int t = tid; t < D; t += 256) { const float a = u[t], b = v[t]; uv = fmaf(a, b, uv); uu = fmaf(a, a, uu); vv = fmaf(b, b, vv); }
        uv = block_sum(uv, red); uu = block_sum(uu, red); vv = block_sum(vv, red);
        if (tid == 0) out[2] = 1.f - uv / (sqrtf(uu) * sqrtf(vv));
    }
}

__global__ void beam_minmax_kernel(const float* __restrict__ scratch, int hist_len, int live_k, float kl, float cf,
                                   float sf, const int32_t* __restrict__ counters, int k, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= live_k || beam_row_idle(counters, k, i)) return;
    float mn = INFINITY, mc = -INFINITY, ms = -INFINITY;
    for (int s = 0; s < hist_len; ++s) {
        const float* v = scratch + ((long long)i * hist_len + s) * 3;
        mn = fminf(mn, v[0]); mc = fmaxf(mc, v[1]); ms = fmaxf(ms, v[2]);
    }
    out[i] = -kl * mn;                 // nats.py:993
    out[live_k + i] = cf * mc;         // nats.py:994
    out[2 * live_k + i] = sf * ms;     // nats.py:995
}

__global__ void beam_reorder_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                    const float* __restrict__ cur, const int32_t* __restrict__ parent, int len_cap,
                                    int hist_len, int dim) {
    const int j = blockIdx.x, s = blockIdx.y;
    const int par = parent[j];
    if (par < 0) return;                                              // row not alive after this step
    const float* from = (s < hist_len) ? src + ((long long)par * len_cap + s) * dim : cur + (long long)par * dim;
    float* to = dst + ((long long)j * len_cap + s) * dim;
    for (int t = threadIdx.x; t < dim; t += blockDim.x) to[t] = from[t];
}

}  // namespace

int beam_distraction_scores(cudaStream_t st, const float* hist_alpha, const float* hist_ctx, const float* hist_state,
                            int len_cap, int hist_len, int live_k, int Tx, int C, int D, const float* cur_alpha,
                            const float* cur_ctx, const float* cur_state, float kl, float cf, float sf, const int32_t* counters,
                            int k, float* scratch, float* out) {
    NATS_REQUIRE(hist_len >= 1 && live_k >= 1 && hist_len <= len_cap, "beam history shape");
    NATS_REQUIRE(counters == nullptr || k >= 1, "beam group shape");
    dim3 grid(hist_len, live_k);
    ProfScope ps(st, K_BEAM);
    beam_pair_kernel<<<grid, 256, 0, st>>>(hist_alpha, hist_ctx, hist_state, len_cap, hist_len, Tx, C, D, cur_alpha,
                                           cur_ctx, cur_state, counters, k, scratch);
    NATS_LAUNCH_OK();
    beam_minmax_kernel<<<cdiv(live_k, 64), 64, 0, st>>>(scratch, hist_len, live_k, kl, cf, sf, counters, k, out);
    NATS_LAUNCH_OK();
    return 0;
}

int beam_reorder_append(cudaStream_t st, const float* src, float* dst, const float* cur, const int32_t* parent,
                        int n_new, int len_cap, int hist_len, int dim) {
    NATS_REQUIRE(n_new >= 1 && hist_len < len_cap, "beam reorder shape");
    dim3 grid(n_new, hist_len + 1);
    ProfScope ps(st, K_BEAM);
    beam_reorder_kernel<<<grid, 256, 0, st>>>(src, dst, cur, parent, len_cap, hist_len, dim);
    NATS_LAUNCH_OK();
    return 0;
}


namespace {

constexpr int kMaxBeam = 32;

// ---------------------------------------------------------------------------------------------------------------
// Device-resident beam bookkeeping (nats.py:976-1066), ONE warp per sentence of a group of S (grid S; S = 1 is the
// single-sentence search): candidate costs from the per-row top-k, distraction re-ranking (nats.py:997-999; the stored cost
// stays un-penalised, :1004), selection of the k - dead_k best in the stable order of a flattened argsort, then the
// reference's loop over the selected candidates in rank order: a candidate ending in word 0 retires into the result slots
// (:1037-1041), the others become the live rows of the next step.  Sentence s owns rows [s k, s k + k) of every per-row
// buffer, counters[8 s .. 8 s + 8) and its result slots; parents / fin_parent hold row indices local to the sentence.
//   counters[8 s + 0] live_k, [1] dead_k, [2] done flag (set when live_k < 1 or dead_k >= k, :1057), [3] finished so far,
//   [4] index of the last step that was carried out (steps issued after `done` change nothing)
//   counters[5] (sentence 0 only): number of sentences of the group that are done; counters[6]: arrival ticket (kept 0)
//   scores / tokens are ping-pong buffers selected by the step parity; tokens rows hold `step` words on entry
//   host_counters (optional): device-visible pinned host memory that receives counters[5] (S = 1: also words 0..4)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void beam_group_count(int32_t* counters, int32_t* host_counters) {
    // the last sentence warp to arrive counts the sentences that are done (the others' flags are visible after the fence)
    const int S = gridDim.x;
    int nd = -1;
    if (S == 1) {
        nd = counters[2] != 0 ? 1 : 0;
    } else {
        __threadfence();
        if (atomicAdd(&counters[6], 1) == S - 1) {
            nd = 0;
            for (int s = 0; s < S; ++s) nd += (*(volatile int32_t*)&counters[8 * s + 2] != 0) ? 1 : 0;
            counters[6] = 0;
        }
    }
    if (nd < 0) return;
    counters[5] = nd;
    if (host_counters != nullptr) {
        *(volatile int32_t*)&host_counters[5] = nd;
        __threadfence_system();
    }
}

__global__ void __launch_bounds__(32) beam_select_kernel(const float* __restrict__ top_p, const int32_t* __restrict__ top_i,
                                                         const float* __restrict__ pen, int k, int maxlen, int step,
                                                         int32_t* __restrict__ counters, float* __restrict__ scores,
                                                         int32_t* __restrict__ tokens, int32_t* __restrict__ parents,
                                                         long long* __restrict__ next_w, int32_t* __restrict__ out_tokens,
                                                         int32_t* __restrict__ out_len, float* __restrict__ out_score,
                                                         int32_t* __restrict__ fin_parent, int32_t* host_counters) {
    __shared__ float s_rank[kMaxBeam * kMaxBeam];
    __shared__ float s_cost[kMaxBeam * kMaxBeam];
    __shared__ int s_word[kMaxBeam * kMaxBeam];                       // top_i, read once (every later use is on the serial path)
    __shared__ int s_sel[kMaxBeam];
    __shared__ int s_slot[kMaxBeam];                                  // destination row of selected candidate r; bit 30: retired
    const int lane = threadIdx.x;
    const int sent = blockIdx.x, n = gridDim.x * k, r0 = sent * k;   // this sentence's rows [r0, r0 + k) of n
    const int cur = step & 1, nxt = cur ^ 1;
    int32_t* cnt = counters + 8 * sent;
    top_p += (long long)r0 * k; top_i += (long long)r0 * k;
    const float* sc_in = scores + cur * n + r0;
    float* sc_out = scores + nxt * n + r0;
    const int32_t* tk_in = tokens + ((long long)cur * n + r0) * maxlen;
    int32_t* tk_out = tokens + ((long long)nxt * n + r0) * maxlen;
    parents += r0; fin_parent += r0; next_w += r0;
    out_tokens += (long long)r0 * maxlen; out_len += r0; out_score += r0;
    for (int j = lane; j < k; j += 32) { parents[j] = -1; fin_parent[j] = -1; }
    const int live_k = cnt[0], dead_k = cnt[1];
    if (cnt[2] != 0) {                                                // finished earlier: nothing moves any more
        if (lane == 0) beam_group_count(counters, host_counters);
        return;
    }
    const int n_keep = k - dead_k;
    const int ncand = live_k * k;
    for (int e = lane; e < k * k; e += 32) {
        float cost = INFINITY, rank = INFINITY;
        const int word = (e < ncand) ? top_i[e] : -1;
        s_word[e] = word;
        if (e < ncand) {
            const int r = e / k;
            if (word >= 0) {
                cost = sc_in[r] - logf(top_p[e]);                     // nats.py:976
                rank = cost;
                if (pen != nullptr && step > 0) rank = cost + pen[r0 + r] + pen[n + r0 + r] + pen[2 * n + r0 + r];     // :997
            }
        }
        s_cost[e] = cost;
        s_rank[e] = rank;
    }
    __syncwarp();
    // n_keep rounds of (value, index) argmin: the order of a stable argsort over the flattened [live_k, k] array
    int nsel = 0;
    for (int r = 0; r < n_keep; ++r) {
        float bv = INFINITY;
        int bi = 0x7fffffff;
        for (int e = lane; e < ncand; e += 32) {
            const float v = s_rank[e];
            if (v < bv || (v == bv && e < bi)) { bv = v; bi = e; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (bi == 0x7fffffff || s_word[bi] < 0) break;                // fewer valid candidates than n_keep
        if (lane == 0) { s_sel[r] = bi; s_rank[bi] = __int_as_float(0x7fc00000); }      // consumed: NaN never compares smaller or equal
        nsel = r + 1;
        __syncwarp();
    }
    int new_live = 0, nfin = cnt[3], ndead = dead_k, fin_now = 0;
    for (int r = 0; r < nsel; ++r) {                                  // rank order, as the reference's zip loop (:1010-1052)
        const int e = s_sel[r];
        const int ti = e / k, wi = s_word[e];
        const float ci = s_cost[e];
        if (wi == 0) {
            if (lane == 0) {
                out_tokens[(long long)nfin * maxlen + step] = 0; out_len[nfin] = step + 1; out_score[nfin] = ci;
                fin_parent[fin_now] = ti; s_slot[r] = nfin | (1 << 30);
            }
            ++nfin; ++ndead; ++fin_now;
        } else {
            if (lane == 0) {
                tk_out[(long long)new_live * maxlen + step] = wi; sc_out[new_live] = ci; parents[new_live] = ti;
                next_w[new_live] = wi; s_slot[r] = new_live;
            }
            ++new_live;
        }
    }
    __syncwarp();
    // the word histories of all selected candidates in one flat loop (independent loads, not one row after the other)
    for (int idx = lane; idx < nsel * step; idx += 32) {
        const int r = idx / step, t = idx - r * step;
        const int slot = s_slot[r], ti = s_sel[r] / k;
        int32_t* dst = (slot & (1 << 30)) ? out_tokens + (long long)(slot & ~(1 << 30)) * maxlen : tk_out + (long long)slot * maxlen;
        dst[t] = tk_in[(long long)ti * maxlen + t];
    }
    __syncwarp();
    if (lane == 0) {
        const int done = (new_live < 1 || ndead >= k) ? 1 : 0;
        cnt[0] = new_live; cnt[1] = ndead; cnt[3] = nfin; cnt[4] = step;
        if (done) cnt[2] = 1;
        if (host_counters != nullptr && gridDim.x == 1) {             // mapped pinned host memory: the host polls it, no copy
            volatile int32_t* h = host_counters;
            h[0] = new_live; h[1] = ndead; h[3] = nfin; h[4] = step; h[2] = done;
        }
        beam_group_count(counters, host_counters);
    }
}

// One launch for all the copies of a beam step (nats.py:1015-1023, 1040); blockIdx.x = row j of the group (sentence j / k,
// whose parents are local to its block of k rows), blockIdx.z selects the job:
//   0..2  history of the next step's row j <- history of its parent + the current vector (alpha; ctx and state when kept)
//   3     attention history of the hypotheses that retired in this step -> the sentence's result slot (assigned in order)
//   4     state / acc_ctx / acc_alpha rows of the next step <- f_next outputs of the parents (blockIdx.y = buffer)
struct BeamAdvance {
    const int32_t* parents; const int32_t* fin_parent; const int32_t* counters;
    const float* hist_src[3]; float* hist_dst[3]; const float* cur[3]; int dim[3];
    const float* row_src[3]; float* row_dst[3]; int row_dim[3];
    float* out_alpha;
    int k, len_cap, step;
};

__global__ void __launch_bounds__(256) beam_advance_kernel(const __grid_constant__ BeamAdvance a) {
    const int j = blockIdx.x, s = blockIdx.y, job = blockIdx.z;
    const int r0 = j - j % a.k;                                       // first row of j's sentence
    if (job < 4 && s > a.step) return;                                // the grid is at least 3 deep for job 4
    if (job < 3) {
        if (a.hist_src[job] == nullptr) return;
        if (a.parents[j] < 0) return;                                 // row not alive after this step
        const int par = r0 + a.parents[j];
        const int dim = a.dim[job];
        const float* from = (s < a.step) ? a.hist_src[job] + ((long long)par * a.len_cap + s) * dim : a.cur[job] + (long long)par * dim;
        float* to = a.hist_dst[job] + ((long long)j * a.len_cap + s) * dim;
        for (int t = threadIdx.x; t < dim; t += 256) to[t] = from[t];
    } else if (job == 3) {
        if (a.fin_parent[j] < 0) return;
        const int par = r0 + a.fin_parent[j];
        int nf_before = a.counters[8 * (r0 / a.k) + 3];
        for (int q = 0; q < a.k; ++q)                                 // count this step's retirements
            if (a.fin_parent[r0 + q] >= 0) --nf_before;
        const int Tx = a.dim[0];
        const float* from = (s < a.step) ? a.hist_src[0] + ((long long)par * a.len_cap + s) * Tx : a.cur[0] + (long long)par * Tx;
        float* to = a.out_alpha + ((long long)(nf_before + j) * a.len_cap + s) * Tx;    // slot r0 + nf_before + (j - r0)
        for (int t = threadIdx.x; t < Tx; t += 256) to[t] = from[t];
    } else {
        if (s >= 3) return;
        if (a.parents[j] < 0) return;
        const int par = r0 + a.parents[j];
        const int n = a.row_dim[s];
        const float* src = a.row_src[s] + (long long)par * n;
        float* dst = a.row_dst[s] + (long long)j * n;
        for (int t = threadIdx.x; t < n; t += 256) dst[t] = src[t];
    }
}

// Output constraints on the next-word probabilities of the live rows (an addition beyond the reference), one warp per row
// of the group.  Row r holds `step` words in tokens[r] (tokens = the current parity's [n, maxlen] rows).  With
// no_repeat = N >= 1, for every start j in [0, step - N] whose N-1 words equal the row's last N-1 words, word
// tokens[r][j + N - 1] gets probability 0: no hypothesis contains an N-gram twice.  While step < min_len, word 0 (EOS)
// gets probability 0.  mask_unk writes entry 1 = 1e-20 (nats.py:975) BEFORE the bans, so a banned UNK ends at 0.
// Idle rows are skipped: beam rows by the counters, sampling rows by row_done (NULL for beam search).
__global__ void __launch_bounds__(32) beam_constrain_kernel(float* __restrict__ probs, int V, const int32_t* __restrict__ tokens,
                                                            int maxlen, int step, int k, const int32_t* __restrict__ counters,
                                                            const int32_t* __restrict__ row_done, int no_repeat, int min_len,
                                                            int mask_unk) {
    extern __shared__ int32_t s_hist[];                               // the row's `step` words
    const int row = blockIdx.x, lane = threadIdx.x;
    if (beam_row_idle(counters, k, row) || (row_done != nullptr && row_done[row] != 0)) return;
    float* p = probs + (long long)row * V;
    const int32_t* tk = tokens + (long long)row * maxlen;
    for (int t = lane; t < step; t += 32) s_hist[t] = tk[t];
    if (mask_unk && lane == 0) p[1] = 1e-20f;
    __syncwarp();                                                     // orders the history and the UNK store before the bans
    if (step < min_len && lane == 0) p[0] = 0.f;
    if (no_repeat < 1 || step < no_repeat) return;
    const int sfx = step - no_repeat + 1;                             // first word of the row's (N-1)-word suffix
    for (int j = lane; j < sfx; j += 32) {
        bool hit = true;
        for (int q = 0; q < no_repeat - 1 && hit; ++q) hit = s_hist[j + q] == s_hist[sfx + q];
        const int w = s_hist[j + no_repeat - 1];
        if (hit && w >= 0 && w < V) p[w] = 0.f;                       // several lanes may ban the same word: same store
    }
}

}  // namespace

int beam_constrain(cudaStream_t st, float* probs, int V, const int32_t* tokens, int maxlen, int step, int n_src, int k,
                   const int32_t* counters, int no_repeat, int min_len, int mask_unk) {
    NATS_REQUIRE(k >= 1 && n_src >= 1 && (long long)n_src * k <= 65535 && step >= 0 && step < maxlen, "beam_constrain shape");
    NATS_REQUIRE(no_repeat >= 0 && min_len >= 0, "beam constraints must be >= 0");
    NATS_REQUIRE(maxlen <= kBeamConstrainMaxLen, "beam constraints need maxlen <= 12288");
    const int n = n_src * k;
    ProfScope ps(st, K_BEAM);
    beam_constrain_kernel<<<n, 32, (size_t)step * sizeof(int32_t), st>>>(probs, V, tokens + (long long)(step & 1) * n * maxlen,
                                                                      maxlen, step, k, counters, nullptr, no_repeat, min_len,
                                                                      mask_unk);
    NATS_LAUNCH_OK();
    return 0;
}

int sample_constrain(cudaStream_t st, float* probs, int V, const int32_t* tokens, int maxlen, int step, int n,
                     const int32_t* row_done, int no_repeat, int min_len) {
    NATS_REQUIRE(n >= 1 && n <= 65535 && step >= 0 && step < maxlen, "sample_constrain shape");
    NATS_REQUIRE(no_repeat >= 0 && min_len >= 0, "sampling constraints must be >= 0");
    NATS_REQUIRE(maxlen <= kBeamConstrainMaxLen, "sampling constraints need maxlen <= 12288");
    ProfScope ps(st, K_SAMPLE);
    beam_constrain_kernel<<<n, 32, (size_t)step * sizeof(int32_t), st>>>(probs, V, tokens, maxlen, step, 1, nullptr, row_done,
                                                                      no_repeat, min_len, 0);
    NATS_LAUNCH_OK();
    return 0;
}

namespace {

// Bookkeeping of one sampling step (an addition beyond the reference), one CTA per source s of the group, rows
// [s R, s R + R).  A row that is not done takes its word v = pick[q]: tokens[q][step] = v, cost[q] -= log probs[q][v] (the
// f_next probability, as beam search's stored cost), out_alpha[q][step] = its attention row, next_w[q] = v; v = 0 ends
// the row with out_len[q] = step + 1.  Rows never branch, so nothing is gathered.  counters[8 + s] = finished rows of
// source s; the last CTA to arrive (ticket counters[1], kept 0) writes the group's total to counters[0] and mirrors it
// into host_counters[0] (pinned host memory the host polls; NULL = off).
__global__ void __launch_bounds__(256) sample_advance_kernel(const int32_t* __restrict__ pick, const float* __restrict__ probs,
                                                             int V, const float* __restrict__ alphaT, int Tx, int R, int maxlen,
                                                             int step, int32_t* __restrict__ done, int32_t* __restrict__ tokens,
                                                             float* __restrict__ cost, int32_t* __restrict__ out_len,
                                                             float* __restrict__ out_alpha, long long* __restrict__ next_w,
                                                             int32_t* counters, int32_t* host_counters) {
    __shared__ int red[8];
    const int s = blockIdx.x, tid = threadIdx.x, S = gridDim.x;
    const long long q0 = (long long)s * R;
    for (long long e = tid; e < (long long)R * Tx; e += 256) {         // attention rows of the rows still open
        const long long q = q0 + e / Tx, t = e % Tx;
        if (done[q] == 0) out_alpha[(q * maxlen + step) * Tx + t] = alphaT[q * Tx + t];
    }
    __syncthreads();                                                  // every read of `done` above precedes the updates
    int nd = 0;
    for (int j = tid; j < R; j += 256) {
        const long long q = q0 + j;
        if (done[q] == 0) {
            const int v = pick[q];
            tokens[q * maxlen + step] = v;
            cost[q] = cost[q] - logf(probs[q * V + v]);
            next_w[q] = v;
            if (v == 0) { done[q] = 1; out_len[q] = step + 1; }
        }
        nd += done[q] != 0 ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nd += __shfl_xor_sync(0xffffffffu, nd, o);
    if ((tid & 31) == 0) red[tid >> 5] = nd;
    __syncthreads();
    if (tid != 0) return;
    nd = 0;
    for (int w = 0; w < 8; ++w) nd += red[w];
    counters[8 + s] = nd;
    __threadfence();
    if (atomicAdd(&counters[1], 1) != S - 1) return;
    int total = 0;
    for (int u = 0; u < S; ++u) total += *(volatile int32_t*)&counters[8 + u];
    counters[1] = 0;
    counters[0] = total;
    if (host_counters != nullptr) {
        *(volatile int32_t*)&host_counters[0] = total;
        __threadfence_system();
    }
}

}  // namespace

int sample_advance(cudaStream_t st, const int32_t* pick, const float* probs, int V, const float* alphaT, int Tx, int n_src,
                   int R, int maxlen, int step, int32_t* done, int32_t* tokens, float* cost, int32_t* out_len, float* out_alpha,
                   long long* next_w, int32_t* counters, int32_t* host_counters) {
    NATS_REQUIRE(n_src >= 1 && R >= 1 && (long long)n_src * R <= 65535 && step >= 0 && step < maxlen && Tx >= 1,
                 "sample_advance shape");
    ProfScope ps(st, K_SAMPLE);
    sample_advance_kernel<<<n_src, 256, 0, st>>>(pick, probs, V, alphaT, Tx, R, maxlen, step, done, tokens, cost, out_len,
                                                 out_alpha, next_w, counters, host_counters);
    NATS_LAUNCH_OK();
    return 0;
}

int beam_select(cudaStream_t st, const float* top_p, const int32_t* top_i, const float* pen, int n_src, int k, int maxlen,
                int step, int32_t* counters, float* scores, int32_t* tokens, int32_t* parents, long long* next_w,
                int32_t* out_tokens, int32_t* out_len, float* out_score, int32_t* fin_parent, int32_t* host_counters) {
    NATS_REQUIRE(k >= 1 && k <= kMaxBeam && step >= 0 && step < maxlen, "beam_select shape (beam <= 32)");
    NATS_REQUIRE(n_src >= 1 && n_src <= 65535, "beam group size");
    ProfScope ps(st, K_BEAM);
    beam_select_kernel<<<n_src, 32, 0, st>>>(top_p, top_i, pen, k, maxlen, step, counters, scores, tokens, parents, next_w,
                                         out_tokens, out_len, out_score, fin_parent, host_counters);
    NATS_LAUNCH_OK();
    return 0;
}

int beam_advance(cudaStream_t st, const int32_t* parents, const int32_t* fin_parent, const int32_t* counters, int n_src,
                 int k, int len_cap, int step, int Tx, int C, int D, const float* state_o, float* state_n, const float* acc_ctx_o,
                 float* acc_ctx_n, const float* acc_alpha_o, float* acc_alpha_n, const float* cur_alpha, const float* cur_ctx,
                 const float* cur_state, const float* hist_alpha_src, float* hist_alpha_dst, const float* hist_ctx_src,
                 float* hist_ctx_dst, const float* hist_state_src, float* hist_state_dst, float* out_alpha) {
    NATS_REQUIRE(k >= 1 && n_src >= 1 && step >= 0 && step < len_cap, "beam_advance shape");
    ProfScope ps(st, K_BEAM);
    BeamAdvance a;
    memset(&a, 0, sizeof(a));
    a.parents = parents; a.fin_parent = fin_parent; a.counters = counters;
    a.hist_src[0] = hist_alpha_src; a.hist_dst[0] = hist_alpha_dst; a.cur[0] = cur_alpha; a.dim[0] = Tx;
    a.hist_src[1] = hist_ctx_src;   a.hist_dst[1] = hist_ctx_dst;   a.cur[1] = cur_ctx;   a.dim[1] = C;
    a.hist_src[2] = hist_ctx_src != nullptr ? hist_state_src : nullptr; a.hist_dst[2] = hist_state_dst; a.cur[2] = cur_state; a.dim[2] = D;
    a.row_src[0] = state_o;     a.row_dst[0] = state_n;     a.row_dim[0] = D;
    a.row_src[1] = acc_ctx_o;   a.row_dst[1] = acc_ctx_n;   a.row_dim[1] = C;
    a.row_src[2] = acc_alpha_o; a.row_dst[2] = acc_alpha_n; a.row_dim[2] = Tx;
    a.out_alpha = out_alpha; a.k = k; a.len_cap = len_cap; a.step = step;
    const int gy = step + 1 < 3 ? 3 : step + 1;
    beam_advance_kernel<<<dim3(n_src * k, gy, 5), 256, 0, st>>>(a);
    NATS_LAUNCH_OK();
    return 0;
}

namespace {

// One CTA per hypothesis row.  Round r selects the largest probability that comes strictly after the previous pick in
// the total order (value descending, index ascending): no marking, no copy of the row, any vocabulary size; the row
// (120 KB at |V| = 30000) is re-read from L1/L2 K times.
__global__ void __launch_bounds__(256) beam_topk_kernel(const float* __restrict__ probs, int V, int K, int mask_unk,
                                                        float* __restrict__ out_p, int32_t* __restrict__ out_idx) {
    __shared__ float s_v[8];
    __shared__ int s_i[8];
    __shared__ float s_pv;
    __shared__ int s_pi;
    const float* row = probs + (long long)blockIdx.x * V;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float pv = INFINITY;
    int pi = -1;
    for (int r = 0; r < K; ++r) {
        float bv = -1.f;
        int bi = 0x7fffffff;
        for (int i = tid; i < V; i += 256) {
            float v = __ldg(row + i);
            if (mask_unk && i == 1) v = 1e-20f;                        // nats.py:975: next_p[:,1] = 1e-20
            if (!(v > 0.f)) v = 0.f;                                     // NaN / negatives count as 0 (never win)
            const bool after = (v < pv) || (v == pv && i > pi);
            if (after && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { s_v[warp] = bv; s_i[warp] = bi; }
        __syncthreads();
        if (tid == 0) {
            float v = s_v[0];
            int i = s_i[0];
#pragma unroll
            for (int w = 1; w < 8; ++w)
                if (s_v[w] > v || (s_v[w] == v && s_i[w] < i)) { v = s_v[w]; i = s_i[w]; }
            if (i == 0x7fffffff) { v = 0.f; i = -1; }                    // fewer than K candidates
            out_p[(long long)blockIdx.x * K + r] = v;
            out_idx[(long long)blockIdx.x * K + r] = i;
            s_pv = v; s_pi = i;
        }
        __syncthreads();
        pv = s_pv; pi = s_pi;
        if (pi < 0) {                                                    // exhausted: fill the rest
            if (tid == 0)
                for (int q = r + 1; q < K; ++q) { out_p[(long long)blockIdx.x * K + q] = 0.f; out_idx[(long long)blockIdx.x * K + q] = -1; }
            break;
        }
    }
}

// Beam-search shapes (a handful of rows, |V| <= 32768): a cluster of 8 CTAs per row.  Every lane holds 8 entries of the
// row in REGISTERS (one read of the row instead of K); each warp picks its own K best with shuffles only, warp 0 merges
// the CTA's 16 x K candidates, and the first warp of the cluster's first CTA merges the 8 x K survivors through
// distributed shared memory.  A candidate is ONE 64-bit key, (bits of the probability) << 32 | ~index: probabilities are
// >= +0 (anything else -- NaN, negatives -- counts as 0, in both kernels), so unsigned key order IS "value descending,
// index ascending", the selection is branch-free, and key 0 means "no candidate".
constexpr int kTopCluster = 8, kTopThreads = 512, kTopPer = 8, kTopMaxK = 32, kTopWarps = kTopThreads / 32;

__device__ __forceinline__ unsigned long long cand_key(float v, int i) {
    return ((unsigned long long)__float_as_uint(v) << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
}

// The K largest keys a warp holds in registers, in descending order; emit(r, key) runs on lane 0 for r = 0..K-1 (key 0
// once the candidates run out).
template <int NPER, class Emit>
__device__ __forceinline__ void warp_select_topk(const unsigned long long (&key)[NPER], int K, int lane, Emit emit) {
    unsigned long long prev = ~0ull;
    for (int r = 0; r < K; ++r) {
        unsigned long long best = 0ull;
#pragma unroll
        for (int q = 0; q < NPER; ++q) {
            const unsigned long long c = key[q] < prev ? key[q] : 0ull;
            best = c > best ? c : best;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other > best ? other : best;
        }
        if (best == 0ull) {
            if (lane == 0)
                for (int q = r; q < K; ++q) emit(q, 0ull);
            return;
        }
        if (lane == 0) emit(r, best);
        prev = best;
    }
}

__global__ void __cluster_dims__(kTopCluster, 1, 1) __launch_bounds__(kTopThreads)
    beam_topk_cluster_kernel(const float* __restrict__ probs, int V, int K, int mask_unk, float* __restrict__ out_p,
                             int32_t* __restrict__ out_idx) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ unsigned long long w_k[kTopWarps * kTopMaxK];
    __shared__ unsigned long long c_k[kTopMaxK];
    const int seg = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* row = probs + (long long)blockIdx.y * V;
    const int seglen = (V + kTopCluster - 1) / kTopCluster;
    const int base = seg * seglen, end = min(V, base + seglen);
    {
        unsigned long long x[kTopPer];
#pragma unroll
        for (int k = 0; k < kTopPer; ++k) {
            const int i = base + k * kTopThreads + tid;
            float v = (i < end) ? __ldg(row + i) : 0.f;
            if (mask_unk && i == 1) v = 1e-20f;                          // nats.py:975
            if (!(v > 0.f)) v = 0.f;
            x[k] = (i < end) ? cand_key(v, i) : 0ull;
        }
        warp_select_topk<kTopPer>(x, K, lane, [&](int r, unsigned long long c) { w_k[warp * K + r] = c; });
    }
    __syncthreads();
    if (warp == 0) {
        unsigned long long m[kTopWarps * kTopMaxK / 32];
#pragma unroll
        for (int q = 0; q < kTopWarps * kTopMaxK / 32; ++q) {
            const int j = lane + 32 * q;
            m[q] = (j < kTopWarps * K) ? w_k[j] : 0ull;
        }
        warp_select_topk<kTopWarps * kTopMaxK / 32>(m, K, lane, [&](int r, unsigned long long c) { c_k[r] = c; });
    }
    cluster.sync();
    if (seg == 0 && warp == 0) {
        unsigned long long m[kTopCluster * kTopMaxK / 32];
#pragma unroll
        for (int q = 0; q < kTopCluster * kTopMaxK / 32; ++q) {
            const int j = lane + 32 * q;                                 // candidate j = (cta j / K, rank j % K)
            m[q] = (j < kTopCluster * K) ? cluster.map_shared_rank(c_k, j / K)[j % K] : 0ull;
        }
        float* op = out_p + (long long)blockIdx.y * K;
        int32_t* oi = out_idx + (long long)blockIdx.y * K;
        warp_select_topk<kTopCluster * kTopMaxK / 32>(m, K, lane, [&](int r, unsigned long long c) {
            op[r] = __uint_as_float((unsigned)(c >> 32));                // key 0 -> (0, -1): the pad of short rows
            oi[r] = c ? (int)(0xffffffffu - (unsigned)c) : -1;
        });
    }
    cluster.sync();                                                      // remote reads done before any CTA exits
}

}  // namespace

int beam_topk(cudaStream_t st, const float* probs, int n, int V, int K, int mask_unk, float* out_p, int32_t* out_idx) {
    NATS_REQUIRE(n >= 1 && V >= 1 && K >= 1, "beam_topk shape");
    static const int force_simple = [] { const char* e = getenv("NATS_TOPK_SIMPLE"); return e && atoi(e) != 0; }();
    if (!force_simple && K <= kTopMaxK && V <= kTopCluster * kTopThreads * kTopPer && n <= 65535) {
        beam_topk_cluster_kernel<<<dim3(kTopCluster, n), kTopThreads, 0, st>>>(probs, V, K, mask_unk, out_p, out_idx);
        NATS_LAUNCH_OK();
        return 0;
    }
    beam_topk_kernel<<<n, 256, 0, st>>>(probs, V, K, mask_unk, out_p, out_idx);
    NATS_LAUNCH_OK();
    return 0;
}

}  // namespace nats
