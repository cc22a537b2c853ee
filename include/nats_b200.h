/*
 * nats_b200.h -- C ABI of libnats_b200.so: the H100 (sm_90a) implementation of the hot path of
 * lukecq1231/nats (scripts/nats.py).
 *
 * The reference has no FFI layer: its operator boundary is the set of compiled `theano.function`
 * callables (f_init, f_next, f_log_probs, f_cost, f_grad_shared, f_update -- nats.py:817, 871, 1320, 1336,
 * 1160, 1170) plus the `tparams` dict of shared variables (nats.py:72-77).  Each entry point below names the
 * reference construct it replaces.  A maintainer of the reference binds these with ctypes (see
 * INTEGRATION.md); nats_b200/nats.py is exactly that binding.
 *
 * Conventions
 *   - Plain C: pointers, sizes, a cudaStream_t passed as void*.  No torch / C++ types.
 *   - Every data pointer is a DEVICE pointer (host code stages inputs; the host-side shim owns the copies).
 *   - Layouts are the reference's: time-major [T, B, feat], float32, token ids int64 (nats.py:237-240).
 *   - Parameters / gradients / optimiser state live in ONE flat float32 buffer each, in the packed device
 *     layout described by nats_param_layout() (gate and candidate matrices of every GRU are stored side by
 *     side as [rows, 3*dim] so one GEMM serves both; nats.py:283-300 keeps them as separate tensors).
 *   - Nothing allocates, nothing synchronises the host: the caller passes a workspace sized by the
 *     *_workspace_bytes() queries, and all work is enqueued on `stream` (CUDA-graph capturable).
 *   - Return value: 0 = ok, non-zero = error; nats_last_error() returns a message (thread-local).
 *   - One host thread per context (the reference is single-threaded per process, gen.py:78-85).
 */
#ifndef NATS_B200_H
#define NATS_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* all entry points below are exported; everything else in the library has hidden visibility */
#pragma GCC visibility push(default)

#define NATS_NUM_PARAMS 43          /* nats.py:613-654 */
#define NATS_GRAD_TAIL 32           /* extra floats after the parameter area of a gradient buffer:
                                       [0] = sum_b cost_b * scale (so one allreduce carries cost + grads) */
#define NATS_ROUGE_MAX_CAP 4096     /* nats_rouge_f: largest ref_cap + cand_cap */

typedef struct nats_ctx nats_ctx_t; /* opaque: device id, SM count, small device scratch */

typedef struct {
    int32_t n_words;   /* V : options['n_words']  */
    int32_t dim_word;  /* W : options['dim_word'] */
    int32_t dim;       /* D : options['dim']      */
    int32_t dim_att;   /* A : options['dim_att']  */
} nats_dims_t;

/* One reference-named tensor inside the flat buffer: element (r, c) lives at offset + r*ld + c. */
typedef struct {
    char name[32];     /* reference key, e.g. "encoder_U" */
    int64_t offset;    /* in floats from the start of the flat buffer */
    int32_t rows, cols, ld;
    int32_t ndim;      /* 1 or 2: rank of the reference tensor (vectors have rows == 1) */
} nats_param_view_t;

const char* nats_last_error(void);
int nats_version(void);

int nats_ctx_create(int device, nats_ctx_t** out);
int nats_ctx_destroy(nats_ctx_t* ctx);

/* replaces: init_params key order / zipp / unzip / itemlist (nats.py:31-46, 613-654).
 * Fills views[NATS_NUM_PARAMS] in the reference order; *total_floats = size of a parameter buffer (a multiple
 * of 32 floats; padding stays zero).  Gradient buffers need total_floats + NATS_GRAD_TAIL floats. */
int nats_param_layout(const nats_dims_t* dims, nats_param_view_t* views, int64_t* total_floats);

/* ---------------------------------------------------------------- training graph (build_model) ---- */
/* Workspace for one (Tx, Ty, B) problem: saved activations for the backward + scratch. */
int64_t nats_train_workspace_bytes(const nats_dims_t* dims, int Tx, int Ty, int B);

/* replaces: f_log_probs (nats.py:1320) = build_model forward (nats.py:658-772).
 * x [Tx,B] i64, x_mask [Tx,B] f32, y [Ty,B] i64, y_mask [Ty,B] f32  ->  cost [B] f32 (per-sample NLL).
 * Leaves in `ws` everything nats_train_bwd needs. */
int nats_train_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                   const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                   int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float* cost);

/* replaces: tensor.grad(cost.mean(), wrt=itemlist(tparams)) (nats.py:1323, 1340), hand-written reverse mode.
 * Must follow nats_train_fwd on the same ws / inputs.  Overwrites grads[0 .. total_floats + NATS_GRAD_TAIL):
 * grads = d( scale * sum_b cost_b ) / d params (scale = 1/B_global), grads[total_floats] = scale*sum_b cost_b. */
int nats_train_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                   const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                   int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float scale, float* grads);

/* nats_train_bwd in two halves, for overlapping the data-parallel all-reduce with the backward itself (SURVEY 8(e)):
 *   _begin  = zero grads, cost tail, readout + decoder-scan backward: on return (in stream order) the slice
 *             grads[nats_grad_split(dims) .. total_floats + NATS_GRAD_TAIL) -- ff_state, decoder, readout parameters and
 *             the cost slot, ~65 % of the buffer -- is FINAL and may be all-reduced while _finish runs;
 *   _finish = encoder backward (both recurrences + their weight gradients + the source-side Wemb scatter): completes
 *             grads[0 .. nats_grad_split(dims)) = Wemb, encoder, encoder_r.
 * _begin followed by _finish == nats_train_bwd. */
int64_t nats_grad_split(const nats_dims_t* dims);
int nats_train_bwd_begin(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                         const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                         int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float scale, float* grads);
int nats_train_bwd_finish(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                          const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                          int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float scale, float* grads);

/* Per-sample weighted backward (an addition beyond the reference; self-critical training weighs each sampled summary by
 * its reward's advantage, some weights negative).  The arguments of nats_train_bwd / nats_train_bwd_begin plus
 * weight [B] (device float32; NULL is an error: the unweighted calls are the way to train without weights):
 *   grads = d( scale * sum_b weight[b] * cost_b ) / d params,   grads[total_floats] = scale * sum_b weight[b] * cost_b.
 * The backward is linear in d logits, so the weight enters only there (row t*B + b of d logits is scaled by weight[b]) and
 * in the cost tail; every product after it is the unweighted one.  nats_train_bwd_finish completes either half unchanged,
 * and nats_train_fwd's per-sample cost stays the unweighted NLL.  A weight that is a power of two (or its negative) scales
 * every gradient by exactly that factor, except the Wemb scatter, whose float atomics have no fixed order. */
int nats_train_bwd_weighted(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                            const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                            int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float scale, const float* weight,
                            float* grads);
int nats_train_bwd_begin_weighted(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                                  const int64_t* x, const float* x_mask, const int64_t* y, const float* y_mask,
                                  int Tx, int Ty, int B, void* ws, int64_t ws_bytes, float scale, const float* weight,
                                  float* grads);

/* Finer-grained pieces of the same graph (SURVEY 8(b)); all operate on the same workspace. */
int nats_encoder_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                     const int64_t* x, const float* x_mask /* NULL = all ones */, int Tx, int Ty, int B,
                     void* ws, int64_t ws_bytes);                       /* nats.py:700-724 */
int nats_decoder_scan_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                          const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                          void* ws, int64_t ws_bytes);                  /* nats.py:730-742 */
int nats_readout_nll_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                         const int64_t* y, const float* y_mask, int Tx, int Ty, int B,
                         void* ws, int64_t ws_bytes, float* cost);      /* nats.py:753-770 */
int nats_readout_nll_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                         const int64_t* y, const float* y_mask, int Tx, int Ty, int B,
                         void* ws, int64_t ws_bytes, float scale, float* grads);
int nats_decoder_scan_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                          const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                          void* ws, int64_t ws_bytes, float* grads);
int nats_encoder_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                     const int64_t* x, const float* x_mask, const int64_t* y, int Tx, int Ty, int B,
                     void* ws, int64_t ws_bytes, float* grads);

/* Read-only views into a training workspace (for tests / alignment dumps): name in
 * {"ctx","init_state","dec_h","dec_ctx","dec_alpha","pctx","logits","dcc","dmean"}; returns device pointer or NULL.
 * "dcc" [Tx,B,2D] = d cost / d ctx from the decoder and "dmean" [B,2D] = d cost / d ctx_mean (not yet divided by the
 * source length): the gradient the encoder backward reads, valid after nats_train_bwd_begin. */
const float* nats_train_ws_view(const nats_dims_t* dims, int Tx, int Ty, int B, void* ws, const char* name);

/* ---------------------------------------------------------------- sampler graph (build_sampler) ---- */
int64_t nats_sampler_workspace_bytes(const nats_dims_t* dims, int Tx, int n);

/* replaces: f_init (nats.py:789-817).  x [Tx,n] i64 -> init_state [n,D], ctx [Tx,n,C]; additionally returns
 * pctx [Tx,n,A] = ctx.Wc_att + b_att (nats.py:493-494) so that f_next need not recompute it every step.
 * x_mask [Tx,n] (NULL = the reference's f_init: no mask): encodes SEVERAL sentences of different lengths in one call,
 * exactly as the training encoder does (nats.py:700-724, masked GRU steps, masked mean for init_state); rows t >= length
 * of column i of ctx / pctx are then padding and must be cut by the caller. */
int nats_sampler_init(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                      const int64_t* x, const float* x_mask, int Tx, int n, void* ws, int64_t ws_bytes,
                      float* init_state, float* ctx_out, float* pctx_out);

/* replaces: f_next (nats.py:821-871) = embed (y<0 -> zeros) + one _step_slice (nats.py:498-572, mask == 1,
 * no context mask) + readout softmax (nats.py:850-861) + multinomial sample (nats.py:864).
 * ctx element (t, i, c) is read at ctx_in[t*ctx_tstride + i*ctx_bstride + c] (bstride 0 = all n hypotheses
 * share one source, i.e. numpy.tile(ctx0,[live_k,1]) of nats.py:958 without the copy).  pctx likewise
 * (pctx_in may be NULL: then it is recomputed from ctx as the reference does).
 * Outputs in the reference order (nats.py:870): probs [n,V], sample [n] i64, state' [n,D], alphaT [n,Tx],
 * ctxs [n,C], acc_ctx' [n,C], acc_alpha' [n,Tx]. */
int nats_sampler_next(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                      const int64_t* y, const float* ctx_in, int64_t ctx_tstride, int64_t ctx_bstride,
                      const float* pctx_in, int64_t pctx_tstride, int64_t pctx_bstride,
                      const float* state, const float* acc_ctx, const float* acc_alpha, int Tx, int n,
                      uint64_t rng_seed, uint64_t rng_step, void* ws, int64_t ws_bytes,
                      float* probs, int64_t* sample, float* state_out, float* alphaT, float* ctxs,
                      float* acc_ctx_out, float* acc_alpha_out);

/* ---------------------------------------------------------------- gradient clip + optimisers ------ */
/* replaces: L2 term (nats.py:1326-1332) and global-norm clip (nats.py:1344-1353) on the flat buffer:
 * grads += 2*decay_c*params (if decay_c>0); g2 = sum grads^2; if clip_c>0 and g2>clip_c^2: grads *= clip_c/sqrt(g2).
 * stats[0] = g2 (pre-clip), stats[1] = sum params^2 (only if decay_c>0).  n = total_floats. */
int nats_grad_clip(nats_ctx_t* ctx, void* stream, int64_t n, const float* params, float* grads,
                   float decay_c, float clip_c, float* stats /* device, >= 4 floats */);

/* replaces: adadelta (nats.py:1145-1173). grad_shared: rg2 <- rho rg2 + (1-rho) g^2 (zg IS the grads buffer);
 * update: ud = -sqrt(ru2+eps)/sqrt(rg2+eps)*zg; ru2 <- rho ru2 + (1-rho) ud^2; p <- p + ud. */
int nats_adadelta_grad_shared(nats_ctx_t* ctx, void* stream, int64_t n, const float* zg, float* rg2, float rho);
int nats_adadelta_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* zg,
                         float* ru2, const float* rg2, float rho, float eps);
/* replaces: adam (nats.py:1106-1142); step = value of i before the update (0-based). */
int nats_adam_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* g,
                     float* m, float* v, int64_t step);
/* replaces: rmsprop (nats.py:1176-1206). */
int nats_rmsprop_grad_shared(nats_ctx_t* ctx, void* stream, int64_t n, const float* zg, float* rg, float* rg2);
int nats_rmsprop_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* zg,
                        float* ud, const float* rg, const float* rg2);

/* ---------------------------------------------------------------- beam-search distraction --------- */
/* replaces: the SciPy loop of gen_sample (nats.py:982-995).  Histories are [k_cap, len_cap, dim] arrays of
 * which rows [0, live_k) x [0, hist_len) are valid.  out [3, live_k]:
 *   out[0,i] = -kl_factor   * min_s KL(alpha_hist[i,s] || alpha_cur[i])   (scipy.stats.entropy semantics)
 *   out[1,i] =  ctx_factor  * max_s (1 - cos(ctx_hist[i,s],   ctx_cur[i]))
 *   out[2,i] =  state_factor* max_s (1 - cos(state_hist[i,s], state_cur[i]))
 * scratch: >= 3*live_k*hist_len floats. */
int nats_beam_distraction_scores(nats_ctx_t* ctx, void* stream,
                                 const float* hist_alpha, const float* hist_ctx, const float* hist_state,
                                 int len_cap, int hist_len, int live_k, int Tx, int C, int D,
                                 const float* cur_alpha, const float* cur_ctx, const float* cur_state,
                                 float kl_factor, float ctx_factor, float state_factor,
                                 float* scratch, float* out);

/* replaces: the full argsort over live_k*|V| candidate scores of nats.py:997-999.  Penalties and hypothesis scores are
 * constant per row, so the global best (k - dead_k) candidates are among each row's (k - dead_k) most probable words:
 * out_p[i, 0:k] / out_idx[i, 0:k] = the k largest probs[i, :] in descending order (ties: lower index first; -1 pads);
 * mask_unk != 0 treats entry 1 as 1e-20 (nats.py:975, use_unk=False); NaN or negative entries count as 0. */
int nats_beam_topk(nats_ctx_t* ctx, void* stream, const float* probs /* [n, n_words] */, int n, int n_words, int k,
                   int mask_unk, float* out_p /* [n,k] */, int32_t* out_idx /* [n,k] */);

/* replaces: the history copies of nats.py:1015-1023: for every new hypothesis j (parent[j] = trans index)
 * dst[j, 0:hist_len] = src[parent[j], 0:hist_len]; dst[j, hist_len] = cur[parent[j]].  dim = row width. */
int nats_beam_reorder_append(nats_ctx_t* ctx, void* stream, const float* src, float* dst, const float* cur,
                             const int32_t* parent, int n_new, int len_cap, int hist_len, int dim);

/* Device-resident bookkeeping of one beam step (replaces the host loop of nats.py:1001-1066): called after
 * nats_sampler_next ran on k rows (rows >= live_k are ignored), nats_beam_topk with K = k, and -- for step > 0 with a
 * distraction factor on -- nats_beam_distraction_scores with live_k = k.
 *   nats_beam_select : candidate costs hyp_score - log p (nats.py:976), re-ranking with the penalties pen [3,k] or NULL
 *     (:997-999, stored cost un-penalised :1004), the k - dead_k best in flattened-argsort order, then in rank order:
 *     word 0 retires the hypothesis into out_tokens / out_len / out_score (:1037-1041), any other word makes the next
 *     live row.  counters (device int32[8]) = {live_k, dead_k, done, finished, last effective step, sentences done (0 or 1), -, -}; scores [2,k] and tokens [2,k,maxlen] are
 *     ping-pong buffers indexed by step parity; parents [k] (-1 = row unused), next_w [k] (input y of the next step),
 *     fin_parent [k] (parents of the hypotheses retired in this step, compacted, -1 padded) are outputs.
 *   nats_beam_advance: state / acc_ctx / acc_alpha rows of the next step <- outputs of nats_sampler_next gathered by
 *     parents (:1015-1023); histories (alpha always, ctx / state when hist_ctx_src != NULL) <- history of the parent + the
 *     current vectors; out_alpha [k,len_cap,Tx] receives the attention history of the hypotheses retired in this step.
 *     host_counters (NULL = off): page-locked HOST memory the device can address (cudaHostAlloc under unified addressing),
 *     int32[8]; the kernel stores the six counters there as well, so the host polls `done` without any copy.
 * The host reads `done` one or two steps late to stop early and copies the result buffers once at the end. */
int nats_beam_select(nats_ctx_t* ctx, void* stream, const float* top_p, const int32_t* top_i, const float* pen,
                     int k, int maxlen, int step, int32_t* counters, float* scores, int32_t* tokens, int32_t* parents,
                     int64_t* next_w, int32_t* out_tokens, int32_t* out_len, float* out_score, int32_t* fin_parent,
                     int32_t* host_counters);
int nats_beam_advance(nats_ctx_t* ctx, void* stream, const int32_t* parents, const int32_t* fin_parent,
                      const int32_t* counters, int k, int len_cap, int step, int Tx, int C, int D,
                      const float* state_o, float* state_n, const float* acc_ctx_o, float* acc_ctx_n,
                      const float* acc_alpha_o, float* acc_alpha_n,
                      const float* cur_alpha, const float* cur_ctx, const float* cur_state,
                      const float* hist_alpha_src, float* hist_alpha_dst, const float* hist_ctx_src, float* hist_ctx_dst,
                      const float* hist_state_src, float* hist_state_dst, float* out_alpha);

/* One beam-search step in ONE call (what nats.py:957-1066 does per iteration of `for ii in xrange(maxlen)`):
 * nats_sampler_next on k rows of one source (zero batch stride, no multinomial draw) -> for step > 0 with a distraction
 * factor on, nats_beam_distraction_scores -> nats_beam_topk (K = k) -> nats_beam_select -> nats_beam_advance, all on
 * `stream`.  The struct carries the arguments of those five calls for one ping-pong parity (`*_in` buffers are read,
 * `*_out` / `*_next` written; the caller swaps them every step); hist_ctx_* / hist_state_* / pen / scratch are NULL when
 * all three factors are 0.  Exists because five foreign-function calls per step cost the host more than the step costs
 * the GPU. */
typedef struct nats_beam_step {
    const float* params;                 /* flat parameter buffer */
    const int64_t* next_w;               /* [k] previous words (-1 = BOS); nats_beam_select writes the next ones here */
    const float* ctx; const float* pctx; /* [Tx, 2*dim], [Tx, dim_att] of the ONE source sentence */
    int32_t Tx, k, maxlen, use_unk;
    void* ws; int64_t ws_bytes;          /* nats_sampler_workspace_bytes(dims, Tx, k) */
    /* f_next: state in, outputs */
    const float* state_in; const float* acc_ctx_in; const float* acc_alpha_in;
    float* probs; float* state_out; float* alphaT; float* ctxs; float* acc_ctx_out; float* acc_alpha_out;
    /* distraction penalties (nats.py:981-999) */
    float kl_factor, ctx_factor, state_factor;
    const float* hist_alpha_in; const float* hist_ctx_in; const float* hist_state_in;
    float* scratch; float* pen;
    /* selection + bookkeeping */
    float* top_p; int32_t* top_i;
    int32_t* counters; float* scores; int32_t* tokens; int32_t* parents; int32_t* fin_parent;
    int32_t* out_tokens; int32_t* out_len; float* out_score; float* out_alpha; int32_t* host_counters;
    /* rows of the next step */
    float* state_next; float* acc_ctx_next; float* acc_alpha_next;
    float* hist_alpha_out; float* hist_ctx_out; float* hist_state_out;
} nats_beam_step_t;
int nats_beam_step(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const nats_beam_step_t* a, int step);

/* One beam step for a GROUP of S source sentences with k rows each, in one call: the weights are read once for all S*k
 * rows and one chain of kernels runs instead of S.  Every sentence is searched exactly as by nats_beam_step on its own
 * (the sentences only share launches), and all of them step in lockstep.  nats_beam_step is the S = 1 case with the
 * source layout [Tx, C].  Row r = s*k + j is row j of sentence s; `beam` holds the fields of nats_beam_step_t with these
 * layouts (n = S*k):
 *   ctx [Tx, S, 2*dim], pctx [Tx, S, dim_att]: exactly what nats_sampler_init with x_mask writes for the S sentences
 *     (Tx = the longest source); src_len [S] (device int32): valid positions of each source.  Attention weights at
 *     t >= src_len[s] are exactly 0 (the training graph's x_mask, nats.py:538-540), which equals f_next on the unpadded
 *     source.  alphaT / acc_alpha / the attention histories are Tx wide, with zeros past src_len[s];
 *   ws: nats_sampler_workspace_bytes(dims, Tx, n);
 *   next_w [n]; state_* [n, dim]; probs [n, n_words]; alphaT, acc_alpha_* [n, Tx]; ctxs, acc_ctx_* [n, 2*dim];
 *   hist_alpha_* [n, maxlen, Tx], hist_ctx_* [n, maxlen, 2*dim], hist_state_* [n, maxlen, dim]; scratch >= 3*n*maxlen
 *     floats, pen [3, n]; top_p / top_i [n, k];
 *   counters [S, 8] (sentence s: {live_k, dead_k, done, finished, last effective step, -, -, -}; the caller sets every
 *     sentence to {1, 0, 0, 0, -1, 0, 0, 0}); counters[5] of sentence 0 = number of sentences that are done, counters[6]
 *     of sentence 0 is used by the kernel and must start at 0;
 *   scores [2, n], tokens [2, n, maxlen], parents [n], fin_parent [n] (parents are row indices within the sentence);
 *   out_tokens [S, k, maxlen], out_len [S, k], out_score [S, k], out_alpha [S, k, maxlen, Tx]: sentence s's retired
 *     hypotheses in slots [0, counters[8*s + 3]);
 *   host_counters (NULL = off): page-locked host memory, int32[8]; [5] receives the number of sentences that are done
 *     (for S = 1 also words 0..4), so the host polls one flag for the whole group.
 * A sentence that is done stays untouched while the others go on.
 * Output constraints (additions beyond the reference; 0 = off, and with both 0 the step is exactly the one above).  At
 * step ii a live row holds the words y_0 .. y_{ii-1} (no BOS, no EOS), and its next-word probabilities are changed before
 * the per-row top-k:
 *   no_repeat_ngram = N >= 1: for every j in [0, ii-N] with y_j .. y_{j+N-2} == y_{ii-N+1} .. y_{ii-1}, word y_{j+N-1}
 *     gets probability 0 (N = 1: every word already in the row), so no hypothesis contains the same N-gram twice;
 *   min_len = L: while ii < L, word 0 (EOS) gets probability 0, so every retired hypothesis has >= L words before EOS.
 *   With use_unk == 0, entry 1 is set to 1e-20 first, so a banned UNK gets 0.  A banned word's candidate cost is +inf,
 *   like a word whose probability underflows; scores and the distraction re-ranking are otherwise unchanged.  A row with
 *   fewer than k admissible words may still select +inf candidates.  The constraints act on beam search only.
 * Errors: k < 1 or k > 32, S < 1, NULL src_len or buffers, no_repeat_ngram < 0 or min_len < 0, a constraint on with
 * maxlen > 12288. */
typedef struct nats_beam_step_many {
    nats_beam_step_t beam;               /* Tx = longest source, k = rows per sentence */
    int32_t n_src;                       /* S */
    const int32_t* src_len;              /* [S] device */
    int32_t no_repeat_ngram;             /* N: block repeated N-grams (0 = off) */
    int32_t min_len;                     /* L: no EOS before L words (0 = off) */
} nats_beam_step_many_t;
int nats_beam_step_many(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const nats_beam_step_many_t* a, int step);

/* Filtered sampling (an addition beyond the reference): one step draws the next word of n = S*R independent rows, R
 * samples of each of S sources, in one call: nats_sampler_next on all n rows (row r = s*R + j attends to source s, as in
 * nats_beam_step_many; no multinomial draw) -> the bans when a constraint is on -> the filtered draw -> the bookkeeping.
 * Rows never branch, so nothing is gathered: the caller swaps the state / acc_ctx / acc_alpha ping-pong buffers (`*_out` of
 * step ii is `*_in` of step ii + 1).  Layouts (n = S*R):
 *   ctx [Tx, S, 2*dim], pctx [Tx, S, dim_att], src_len [S] (device int32): as for nats_beam_step_many;
 *   ws: nats_sampler_workspace_bytes(dims, Tx, n); next_w [n] (int64; -1 = BOS before step 0; receives the drawn words);
 *   state_* [n, dim] (state_in of step 0: each source's init_state on its R rows), acc_ctx_* [n, 2*dim] and acc_alpha_*
 *     [n, Tx] (zeros at step 0), probs [n, n_words], alphaT [n, Tx], ctxs [n, 2*dim]: f_next's outputs;
 *   pick [n] (int32 scratch), done [n] (int32, zeros at step 0), tokens [n, maxlen] (int32), cost [n] (float, zeros at
 *     step 0), out_len [n] (int32, maxlen at step 0), out_alpha [n, maxlen, Tx];
 *   counters [8 + S] (int32, zeros at step 0): [0] finished rows of the group, [1] used by the kernel, [8 + s] finished
 *     rows of source s; host_counters (NULL = off): page-locked host memory, int32[8]; [0] receives counters[0], so the
 *     host polls one flag for the whole group.
 * Row r is the global row q = row_base + r (row_base = (index of the group's first source) * R), and at step ii a row that
 * is not done does:
 *   1. p = its f_next probabilities.  A word is banned when it is UNK (1) and use_unk == 0, EOS (0) while ii < min_len, or
 *      it would complete an N-gram the row already contains (no_repeat_ngram = N, the rule of nats_beam_step_many).
 *   2. Banned words get weight 0, every other word w_v = (p_v / p_max)^(1/T), p_max the largest admissible p (T = 1:
 *      w = p exactly).
 *   3. Sorted order: w descending, ties by lower index first.  top_k = K >= 1 keeps the first K words with w > 0; top_p =
 *      P < 1 then keeps the shortest prefix of those whose weight sum is >= P x their total.  (The kernel sums these
 *      weights in 2^-40 fixed point of the largest weight, exact and independent of order: below n_words * 2^-40 of it.)
 *   4. u = uniform01(seed, ii, q) (the counter-based splitmix64 uniform of nats_sampler_next), Z = the kept total: the word
 *      is the smallest kept v with u*Z < sum of the kept w up to v in vocabulary order (rounding: the last kept word).  A
 *      word of weight 0 is never drawn.  When (p_v / p_max)^(1/T) underflows to 0 in float32 (small T), fewer words may
 *      carry weight than top_k asks for: then all of them are kept.  With no admissible word the row ends with word 0.
 *   5. tokens[q][ii] = v, cost[q] += -log p_v (the unfiltered f_next probability, as beam search's stored cost),
 *      out_alpha[q][ii] = its attention row; word 0 ends the row with out_len[q] = ii + 1 (EOS included).  A row forced to
 *      end also pays -log p_0 of its unfiltered probability: the EOS and UNK bans act in the draw, probs keeps f_next's
 *      values except the n-gram bans' zeros (which never hit EOS).
 * A row's draws depend only on (seed, step, q) and its own words: not on the group, its size or the other rows.  Every
 * reduction has a fixed order, so a repeated call gives the same bits.
 * Errors: temperature <= 0 or NaN, top_k < 0, top_p outside (0, 1] or NaN, R < 1, S < 1, S*R > 65535, negative
 * constraints, a constraint on with maxlen > 12288, NULL buffers. */
typedef struct nats_sample_step_many {
    const float* params;                 /* flat parameter buffer */
    int64_t* next_w;                     /* [n] */
    const float* ctx; const float* pctx; /* [Tx, S, 2*dim], [Tx, S, dim_att] */
    const int32_t* src_len;              /* [S] device */
    int32_t Tx, n_src, n_samples, maxlen; /* Tx = longest source, S, R, steps */
    int32_t use_unk, top_k, no_repeat_ngram, min_len;
    float temperature, top_p;
    uint64_t seed, row_base;
    void* ws; int64_t ws_bytes;
    const float* state_in; const float* acc_ctx_in; const float* acc_alpha_in;
    float* state_out; float* acc_ctx_out; float* acc_alpha_out;
    float* probs; float* alphaT; float* ctxs;
    int32_t* pick; int32_t* done; int32_t* tokens; float* cost; int32_t* out_len; float* out_alpha;
    int32_t* counters; int32_t* host_counters;
} nats_sample_step_many_t;
int nats_sample_step_many(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const nats_sample_step_many_t* a, int step);

/* ---------------------------------------------------------------- rewards ----------------------- */
/* ROUGE of token ids (an addition beyond the reference; the reward of self-critical training): out [3, n] (device float32)
 * = the ROUGE-1, ROUGE-2 and ROUGE-L F of candidate row r against reference row r / rows_per_ref, n = n_ref * rows_per_ref.
 *   cand [n, cand_cap] int32 with cand_len [n], ref [n_ref, ref_cap] int32 with ref_len [n_ref] (all device arrays).
 *   A row's words are its first min(len, cap) entries (len clamped to [0, cap]) up to the first 0 (EOS, excluded).
 *   UNK (1) matches nothing, UNK included, but counts in the lengths.  Hits: ROUGE-N, the clipped counts
 *   sum_g min(c_ref(g), c_cand(g)) of ROUGE.pl (N = 1, 2); ROUGE-L, the length of the longest common subsequence.
 *   F = (float)(2 h) / (float)(m + c), h the hits, m and c the reference's and the candidate's n-gram counts
 *   max(0, len - N + 1) (ROUGE-L: the lengths); F = 0 when h = 0.  This is ROUGE.pl's P R / (0.5 P + 0.5 R) (alpha 0.5)
 *   without its 5-decimal rounding.  Counting is integer, so the result does not depend on the launch.
 * Errors: NULL arguments, n_ref < 1, rows_per_ref < 1, n != n_ref * rows_per_ref, a cap < 1,
 * ref_cap + cand_cap > NATS_ROUGE_MAX_CAP. */
int nats_rouge_f(nats_ctx_t* ctx, void* stream, const int32_t* cand, int cand_cap, const int32_t* cand_len, int n,
                 const int32_t* ref, int ref_cap, const int32_t* ref_len, int n_ref, int rows_per_ref, float* out);

/* ---------------------------------------------------------------- diagnostics ------------------- */
/* The library's internal GEMM engine, exposed for the parity tests: C = op(A).op(B) (+bias) (+C), row-major,
 * path 0 = exact-fp32 FFMA kernels, path 1 = wgmma 3xTF32 kernel with software loaders, path 2 = wgmma 3xTF32 kernel
 * fed by TMA (needs 16-byte aligned operands, leading dimensions multiple of 4), path 3 = the TMA-fed kernel with the
 * 128-row operand split in registers (its default for skinny products); any other path is an error.  splitk > 1
 * writes splitk slabs of M*ldc floats to C (the consumer kernels sum them); batch > 1 uses the given strides. */
int nats_debug_gemm(nats_ctx_t* ctx, void* stream, int path, int transA, int transB, int M, int N, int K,
                    const float* A, int lda, const float* B, int ldb, float* C, int ldc, const float* bias,
                    int accumulate, int splitk, int batch, int64_t strideA, int64_t strideB, int64_t strideC);

/* Per-kernel-class timing with CUDA events on the launch stream (eager launches only; keep it off while a step
 * is captured into a CUDA graph).  nats_profile_read synchronises the device and returns, per class, the summed
 * milliseconds, algorithmic flops / bytes declared at the launch sites, and the number of launches. */
int nats_profile_enable(nats_ctx_t* ctx, int on);
int nats_profile_num_classes(void);
const char* nats_profile_class_name(int cls);
int nats_profile_read(nats_ctx_t* ctx, int n_classes, double* ms, double* flops, double* bytes, int64_t* launches);

#pragma GCC visibility pop

#ifdef __cplusplus
}
#endif
#endif /* NATS_B200_H */
