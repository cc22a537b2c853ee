// ops.cuh -- host wrappers of the non-GEMM kernels of libnats_b200.  Internal (not part of the C ABI).
#pragma once
#include "common.cuh"

namespace nats {

// ------------------------------------------------------------------ embedding (nats.py:700-701, 730-734, 827-829)
// out[i,:] = Wemb[id_i,:] with id_i = ids[i - shift] (i >= shift) or "none" (i < shift); id < 0 or >= V -> zeros.
int gather_rows(cudaStream_t st, const float* Wemb, const int64_t* ids, int n_rows, int W, int V, int shift,
                float* out);
// dWemb[id_i,:] += src[i,:]  (same index rule; rows with no id are skipped)
int scatter_add_rows(cudaStream_t st, float* dWemb, const int64_t* ids, int n_rows, int W, int V, int shift,
                     const float* src);

// ------------------------------------------------------------------ GRU cell epilogues (nats.py:336-356, 505-518, 551-565)
struct GateFwd {
    const float* part;      // split-K slabs of h_prev.[U|Ux]: element (s,b,n) at part[s*part_stride + b*3D + n]
    int nsplit;             // 0 = h_prev is zero (first step)
    long long part_stride;
    const float* xproj;     // mode 0: [B,3D] input projection incl. biases (row stride 3D)
    const float* part2;     // mode 1: slabs of ctx.[W_1|Wx_1]
    int nsplit2;
    long long part2_stride;
    const float* bias;      // mode 1: [3D] = [b_1 | bx_1]
    const float* h_prev;    // [B,D] with row stride ld_hprev; NULL = zeros
    int ld_hprev;
    const float* mask;      // [B] or NULL (= ones)
    float* h_out;           // [B,D] row stride ld_hout
    int ld_hout;
    float* r; float* u; float* c; float* p;   // [B,D] save slots or NULL
    float* ctxsum;          // optional running sum_t mask*h  (row stride ld_ctxsum), or NULL
    int ld_ctxsum;
};
// mode 0: encoder GRU / decoder GRU_2 (candidate bias outside the reset gate);
// mode 1: decoder GRU_1 (bias bx_1 inside the reset gate, context products in part2)
int gru_gates_fwd(cudaStream_t st, const GateFwd* groups, int ngroups, int B, int D, int mode);

struct GateBwd {
    const float* dh_a; int ld_a;          // dense addends of d h_t (NULL = none)
    const float* dh_b; int ld_b;
    const float* part;  int nsplit;  long long part_stride;  int part_ld;    // slabs [s][B][part_ld]
    const float* part2; int nsplit2; long long part2_stride; int part2_ld;
    const float* mean_grad; int ld_mean;  // optional: dh += mask[b]*coef[b]*mean_grad[b, j]  (ctx-mean path)
    const float* coef;                    // [B] (1 / sum_t mask)
    const float* r; const float* u; const float* c; const float* p;   // saved [B,D]
    const float* h_prev; int ld_hprev;    // NULL = zeros
    const float* mask;                    // [B] or NULL
    float* dG;                            // [B,3D] = [dg_r | dg_u | dp ]    (products with the recurrent input)
    float* dGx;                           // [B,3D] = [dg_r | dg_u | dpc]    (input side)
    float* dh_elem;                       // [B,D]  elementwise part of d h_{t-1}
};
int gru_gates_bwd(cudaStream_t st, const GateBwd* groups, int ngroups, int B, int D);

// ------------------------------------------------------------------ persistent tensor-core encoder recurrence (enc_tc.cu)
struct EncTcFwdArgs {
    const float* Ucat[2]; const float* xproj[2]; const float* mask; float* cc;
    float* r[2]; float* u[2]; float* c[2]; float* p[2];      // NULL = do not save
    float* ctxsum;
    unsigned* bar; long long bar_ints;                        // counters (zeroed by the call)
    float* scratch; long long scratch_floats;                 // residual side buffer + K-partial slabs
    unsigned long long* dbg;                                  // optional phase stamps (NULL = off)
    int Tx, n, D;
};
struct EncTcBwdArgs {
    const float* Ucat[2]; const float* dcc; const float* mean_grad; const float* coef; const float* mask; const float* cc;
    const float* r[2]; const float* u[2]; const float* c[2]; const float* p[2];
    float* dG[2]; float* dGx[2];
    unsigned* bar; long long bar_ints; float* scratch; long long scratch_floats;
    unsigned long long* dbg;
    int Tx, n, D;
};
bool enc_tc_eligible(const nats_ctx* ctx, int n, int D, int pass);   // pass: 0 forward, 1 backward
void enc_tc_enable(int on);                                          // 0 off, 1 both passes (default), 2 forward only, 3 backward only
int enc_tc_setup(const nats_ctx* ctx);
long long enc_tc_scratch_floats(int n, int D);     // upper bounds, independent of the device
long long enc_tc_counter_ints();
int enc_tc_fwd(const nats_ctx* ctx, cudaStream_t st, const EncTcFwdArgs& a);
int enc_tc_bwd(const nats_ctx* ctx, cudaStream_t st, const EncTcBwdArgs& a);
void tma_gemm_set_ts(int on);
int tma_gemm_get_ts();
void gates_trace(int on);
void attention_set_cc_keep(int mode);

// ------------------------------------------------------------------ small elementwise / reductions
int tanh_inplace(cudaStream_t st, float* x, long long n);
// out[n,N] = act(sum_p x_p[n,K_p].W_p[K_p,N] + sum_p bias_p): few rows, narrow output (ops_readout.cu); unused parts K = 0
struct NarrowProj {
    const float* x[3]; long long ldx[3];
    const float* W[3]; long long ldw[3];
    const float* bias[3];
    int K[3];
    int n, N;
    float* out; long long ldo;
    int act_tanh;
};
int narrow_proj_setup(const nats_ctx* ctx);   // one-time kernel attribute (shared-memory opt-in)
bool narrow_proj_eligible(const NarrowProj& a);
int narrow_proj(cudaStream_t st, const NarrowProj& a);
// dst[i] = g[i] * (1 - y[i]^2)
int dtanh(cudaStream_t st, const float* g, const float* y, float* dst, long long n);
// dst[b,j] = (a[b,j] + sum_s part[s][b][j]) * (1 - y[b,j]^2)   (d init_state path)
int sum_parts_dtanh(cudaStream_t st, const float* a, const float* part, int nsplit, long long part_stride,
                    const float* y, float* dst, int B, int D);
// xlen[b] = sum_t mask[t*B+b] (mask NULL -> Tx);  inv[b] = 1/xlen[b]
int mask_lengths(cudaStream_t st, const float* mask, int Tx, int B, float* xlen, float* inv);
// out[b,c] = sum[b,c] * inv[b]
int scale_rows(cudaStream_t st, const float* src, const float* inv, int B, int C, float* out);
// out[n] (+)= sum_k X[k*ld + n]                  (bias gradients)
int colsum(cudaStream_t st, const float* X, long long K, int N, int ld, float* out, int accumulate, float* scratch);
// the same column sums written to three outputs
int colsum3(cudaStream_t st, const float* X, long long K, int N, int ld, float* out, float* out2, float* out3, int accumulate,
            float* scratch);
// out[n] (+)= sum_k X[k*ld+n] * Y[k*ld+n]        (d U_con, d W_con)
int colsum_prod(cudaStream_t st, const float* X, const float* Y, long long K, int N, int ld, float* out,
                int accumulate, float* scratch);
// cost[b] = sum_t rowcost[t*B+b];   *total (device scalar) = scale * sum_b weight[b] * cost[b]   (weight NULL = ones)
int cost_reduce(cudaStream_t st, const float* rowcost, int Ty, int B, float* cost, float scale, const float* weight,
                float* total);

// ------------------------------------------------------------------ attention + distraction (nats.py:527-546, 569-570)
struct AttFwd {
    const float* pctx; long long pctx_tstride, pctx_bstride;  // element (t,b,a) at pctx[t*ts + b*bs + a]
    const float* cc;   long long cc_tstride, cc_bstride;      // element (t,b,c)
    int cc_keep;               // L2 evict_last fraction mode for the cc stream (0 none, 1..4 = 25..100 %)
    const float* ps_part; int ps_nsplit; long long ps_stride; // slabs of h1.W_att  [s][n][A]
    float* ps_save;            // [n,A] or NULL
    const float* acc_alpha_in; // [n,Tx]
    const float* acc_ctx_in;   // [n,C]
    const float* xmask;        // [Tx,n] (element t*n+b) or NULL
    int rows_per_src;          // row b reads source b / rows_per_src (0 = 1; a zero cc batch stride: all rows share one)
    const int32_t* src_len;    // [sources] valid positions of each source (alpha = 0 at t >= len) or NULL (= Tx)
    const float* ymask;        // [n] step mask m_ or NULL (= ones)
    const float* D_wei; const float* U_att; const float* c_att; const float* U_con; const float* W_con;
    float* escore;             // [n,Tx] scratch
    float* alpha_out;          // [n,Tx]
    float* acc_alpha_out;      // [n,Tx]
    float* craw_out;           // [n,C] or NULL
    float* ctx_out;            // [n,C]
    float* acc_ctx_out;        // [n,C]
    int Tx, n, A, C;
};
int attention_fwd(const nats_ctx* ctx, cudaStream_t st, const AttFwd& a);
int attention_setup(const nats_ctx* ctx);   // one-time kernel attributes

struct AttBwd {
    const float* pctx; const float* cc;           // training layouts [Tx,B,A], [Tx,B,C]
    int cc_keep;
    const float* dctx_a;                          // [B,C] readout contribution
    const float* dctx_part; int dctx_nsplit; long long dctx_stride;   // slabs [s][B][C] of dG1x.W1cat^T
    const float* dacc_ctx_in; float* dacc_ctx_out; // [B,C]
    float* dacc_alpha;                            // [B,Tx] in/out
    const float* ymask;                           // [B]
    const float* ctx; const float* craw; const float* acc_ctx; // saved [B,C]
    const float* alpha; const float* acc_alpha;   // saved [B,Tx]
    const float* ps;                              // saved [B,A]
    const float* D_wei; const float* U_att; const float* U_con; const float* W_con;
    float* dq; float* dcraw;                      // [B,C] outputs (kept for the post-loop products)
    float* dalpha;                                // [B,Tx] scratch
    float* dps;                                   // [B,A] output
    float* dpctx;                                 // [Tx,B,A] accumulated over steps
    float* gatt_part;                             // [B, 2A+1] accumulated over steps
    float* dot_part;                              // scratch [B, ceil(Tx/16)]
    float* soft_part;                             // scratch [B, ceil(Tx/16), 3A+1]
    int Tx, B, A, C;
};
int attention_bwd(const nats_ctx* ctx, cudaStream_t st, const AttBwd& a);

// ------------------------------------------------------------------ readout (nats.py:763-770, 861-864)
// per row r: lse[r] = logsumexp(logits[r,:]); rowcost[r] = (lse[r] - logits[r, y[r]]) * ymask[r]
int nll_rows(cudaStream_t st, const float* logits, int rows, int V, const int64_t* y, const float* ymask,
             float* lse, float* rowcost);
// logits[r,v] <- (exp(logits[r,v]-lse[r]) - [v==y[r]]) * ymask[r] * scale (* weight[r % B] unless weight is NULL)
int dlogits_inplace(cudaStream_t st, float* logits, int rows, int V, const int64_t* y, const float* ymask,
                    const float* lse, float scale, const float* weight, int B);
// probs[r,:] = softmax(logits[r,:]); sample[r] ~ multinomial(probs[r,:]) (counter-based RNG)
int softmax_sample_rows(cudaStream_t st, const float* logits, int rows, int V, float* probs, int64_t* sample,
                        uint64_t seed, uint64_t step);
// filtered sampling of one word per row that is not done (row_done[r] != 0 skips row r; NULL = every row): UNK banned
// when mask_unk, EOS when ban_eos (probs itself is not changed), temperature, top-k (0 = off), top-p (1 = off), draw with
// uniform01(seed, step, row_base + r); pick [rows]; see ops_readout.cu and nats_sample_step_many in include/nats_b200.h
int sample_filter(cudaStream_t st, const float* probs, int rows, int V, const int32_t* row_done, int mask_unk, int ban_eos,
                  float temperature, int top_k, float top_p, uint64_t seed, int step, uint64_t row_base, int32_t* pick);

// ------------------------------------------------------------------ optimiser (nats.py:1106-1206, 1326-1353)
int grad_clip(const nats_ctx* ctx, cudaStream_t st, long long n, const float* params, float* grads, float decay_c,
              float clip_c, float* stats);
int adadelta_grad_shared(cudaStream_t st, long long n, const float* zg, float* rg2, float rho);
int adadelta_update(cudaStream_t st, long long n, float* p, const float* zg, float* ru2, const float* rg2,
                    float rho, float eps);
int adam_update(cudaStream_t st, long long n, float* p, const float* g, float* m, float* v, long long step);
int rmsprop_grad_shared(cudaStream_t st, long long n, const float* zg, float* rg, float* rg2);
int rmsprop_update(cudaStream_t st, long long n, float* p, const float* zg, float* ud, const float* rg,
                   const float* rg2);

// ------------------------------------------------------------------ beam search (nats.py:982-995, 1015-1023)
// counters (NULL = every row): beam_select's [S][8] counters; rows i with i % k >= live_k of sentence i / k are skipped
int beam_distraction_scores(cudaStream_t st, const float* hist_alpha, const float* hist_ctx, const float* hist_state,
                            int len_cap, int hist_len, int live_k, int Tx, int C, int D, const float* cur_alpha,
                            const float* cur_ctx, const float* cur_state, float kl, float cf, float sf,
                            const int32_t* counters, int k, float* scratch, float* out);
// per row the K largest probabilities (descending; ties by ascending index); entry 1 counts as 1e-20 when mask_unk
int beam_topk(cudaStream_t st, const float* probs, int n, int V, int K, int mask_unk, float* out_p, int32_t* out_idx);
int beam_reorder_append(cudaStream_t st, const float* src, float* dst, const float* cur, const int32_t* parent,
                        int n_new, int len_cap, int hist_len, int dim);
// n-gram blocking and minimum length on the live rows' probs [n_src*k, V] before beam_topk (tokens: beam_select's ping-pong
// [2, n_src*k, maxlen] histories, read at parity step & 1); entry 1 = 1e-20 first when mask_unk: see ops_beam.cu
constexpr int kBeamConstrainMaxLen = 12288;   // a row's history is staged in (at most 48 KB of) shared memory
int beam_constrain(cudaStream_t st, float* probs, int V, const int32_t* tokens, int maxlen, int step, int n_src, int k,
                   const int32_t* counters, int no_repeat, int min_len, int mask_unk);
// the same bans on the n rows of a sampling group (tokens [n, maxlen]: each row's own words; rows with row_done[r] != 0
// are skipped); the sampling step passes min_len = 0 and leaves the EOS and UNK bans to sample_filter
int sample_constrain(cudaStream_t st, float* probs, int V, const int32_t* tokens, int maxlen, int step, int n,
                     const int32_t* row_done, int no_repeat, int min_len);
// bookkeeping of one sampling step for a group of n_src sources x R rows (pick -> tokens, cost, lengths, attention,
// next_w, the group's count of finished rows): see ops_beam.cu
int sample_advance(cudaStream_t st, const int32_t* pick, const float* probs, int V, const float* alphaT, int Tx, int n_src,
                   int R, int maxlen, int step, int32_t* done, int32_t* tokens, float* cost, int32_t* out_len, float* out_alpha,
                   long long* next_w, int32_t* counters, int32_t* host_counters);
// device-resident bookkeeping of one beam step (nats.py:976-1066) for a group of n_src sentences x k rows: see ops_beam.cu
int beam_select(cudaStream_t st, const float* top_p, const int32_t* top_i, const float* pen, int n_src, int k, int maxlen,
                int step, int32_t* counters, float* scores, int32_t* tokens, int32_t* parents, long long* next_w,
                int32_t* out_tokens, int32_t* out_len, float* out_score, int32_t* fin_parent, int32_t* host_counters);
int beam_advance(cudaStream_t st, const int32_t* parents, const int32_t* fin_parent, const int32_t* counters, int n_src,
                 int k, int len_cap, int step, int Tx, int C, int D, const float* state_o, float* state_n, const float* acc_ctx_o,
                 float* acc_ctx_n, const float* acc_alpha_o, float* acc_alpha_n, const float* cur_alpha, const float* cur_ctx,
                 const float* cur_state, const float* hist_alpha_src, float* hist_alpha_dst, const float* hist_ctx_src,
                 float* hist_ctx_dst, const float* hist_state_src, float* hist_state_dst, float* out_alpha);

// ------------------------------------------------------------------ ROUGE of token-id rows (ops_rouge.cu)
constexpr int kRougeMaxCap = NATS_ROUGE_MAX_CAP;   // ref_cap + cand_cap: both rows and the LCS diagonals in shared memory
// out [3, n]: ROUGE-1, ROUGE-2 and ROUGE-L F of candidate row r against reference row r / rows_per_ref (nats_rouge_f)
int rouge_f(cudaStream_t st, const int32_t* cand, int cand_cap, const int32_t* cand_len, int n, const int32_t* ref,
            int ref_cap, const int32_t* ref_len, int rows_per_ref, float* out);

}  // namespace nats
