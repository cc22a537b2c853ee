// api.cu -- the C ABI of libnats_b200.so (declared in include/nats_b200.h).
#include <stdarg.h>
#include <stdlib.h>

#include <vector>

#include "model.cuh"

namespace nats {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace nats

// ------------------------------------------------------------------ per-kernel-class profiler (prof.cuh)
namespace nats {
namespace {
struct ProfRec { int cls; double flops, bytes; };
struct ProfState {
    bool on = false;
    std::vector<cudaEvent_t> ev;     // pairs: 2*i = start, 2*i+1 = stop
    std::vector<ProfRec> recs;
};
ProfState g_prof;
const char* kNames[K_COUNT] = {
    "gemm_big_nn", "gemm_big_nt", "gemm_big_tn", "gemm_big_tt", "gemm_mid_nn", "gemm_mid_nt", "gemm_mid_tn",
    "gemm_mid_tt", "gemm_smallm_nn", "gemm_smallm_nt", "gemm_smallm_tn", "gemm_smallm_tt", "gru_gates_fwd",
    "gru_gates_bwd", "att_scores", "att_context", "att_bwd_ctx", "att_bwd_dalpha", "att_bwd_softmax", "nll_rows",
    "dlogits", "softmax_sample", "colsum", "reduce_splits", "embedding", "elementwise", "optimizer", "beam",
    "memset", "tc_gemm_3xtf32", "tc_gemm_3xtf32_skinny", "enc_tc_fwd", "enc_tc_bwd"};
}  // namespace
const char* kclass_name(int cls) { return (cls >= 0 && cls < K_COUNT) ? kNames[cls] : "?"; }
bool prof_enabled() { return g_prof.on; }
void prof_begin(cudaStream_t st, int cls, double flops, double bytes) {
    const size_t i = g_prof.recs.size();
    while (g_prof.ev.size() < 2 * (i + 1)) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) { g_prof.on = false; return; }
        g_prof.ev.push_back(e);
    }
    g_prof.recs.push_back(ProfRec{cls, flops, bytes});
    cudaEventRecord(g_prof.ev[2 * i], st);
}
void prof_end(cudaStream_t st) {
    if (g_prof.recs.empty()) return;
    cudaEventRecord(g_prof.ev[2 * (g_prof.recs.size() - 1) + 1], st);
}
}  // namespace nats

namespace nats {
static int g_pdl = 1;
int pdl_enabled() { return g_pdl; }
void pdl_set(int on) { g_pdl = on; }
}  // namespace nats

using namespace nats;

namespace {

int check_dims(const nats_dims_t* d) {
    NATS_REQUIRE(d != nullptr, "dims");
    NATS_REQUIRE(d->n_words >= 2 && d->dim_word >= 1 && d->dim >= 1 && d->dim_att >= 1, "dims must be positive");
    NATS_REQUIRE(d->dim_att <= 256, "dim_att <= 256");
    return 0;
}

struct ViewDef { const char* name; int64_t off; int rows, cols, ld, ndim; };

}  // namespace

extern "C" {

const char* nats_last_error(void) { return g_err; }
int nats_version(void) { return 101; }

int nats_ctx_create(int device, nats_ctx_t** out) {
    NATS_REQUIRE(out != nullptr, "out");
    NATS_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    NATS_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("libnats_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
        return 3;
    }
    nats_ctx* c = new nats_ctx;
    c->device = device;
    c->num_sms = prop.multiProcessorCount;
    c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
    c->dev_scratch = nullptr;
    NATS_CUDA_OK(cudaMalloc(&c->dev_scratch, kCtxScratchFloats * sizeof(float)));
    int r = attention_setup(c);
    if (r == 0) r = narrow_proj_setup(c);
    if (r == 0) r = tc_gemm_setup();
    if (r == 0) r = tma_gemm_setup();
    if (r == 0) r = enc_tc_setup(c);
    enc_tc_enable(getenv("NATS_ENC_TC") ? atoi(getenv("NATS_ENC_TC")) : 1);      // 0: per-step encoder path, 2 / 3: forward / backward only
    attention_set_cc_keep(getenv("NATS_CC_KEEP") ? atoi(getenv("NATS_CC_KEEP")) : 0);
    tma_gemm_set_ts(getenv("NATS_TS") ? atoi(getenv("NATS_TS")) : 1);
    if (getenv("NATS_TRACE_GATES")) gates_trace(atoi(getenv("NATS_TRACE_GATES")));
    pdl_set(getenv("NATS_PDL") ? atoi(getenv("NATS_PDL")) : 1);
    gemm_set_tensor_cores(getenv("NATS_TC") ? atoi(getenv("NATS_TC")) : 2);
    if (r != 0) { cudaFree(c->dev_scratch); delete c; return r; }
    *out = c;
    return 0;
}

int nats_ctx_destroy(nats_ctx_t* ctx) {
    if (!ctx) return 0;
    if (ctx->dev_scratch) cudaFree(ctx->dev_scratch);
    delete ctx;
    return 0;
}

int nats_param_layout(const nats_dims_t* dims, nats_param_view_t* views, int64_t* total_floats) {
    NATS_TRY(check_dims(dims));
    const ParamOff o = param_offsets(*dims);
    const int V = dims->n_words, W = dims->dim_word, D = dims->dim, A = dims->dim_att, C = 2 * D, D3 = 3 * D;
    const ViewDef defs[NATS_NUM_PARAMS] = {
        {"Wemb", o.Wemb, V, W, W, 2},
        {"encoder_W", o.enc[0].Wcat, W, 2 * D, D3, 2},
        {"encoder_b", o.enc[0].bcat, 1, 2 * D, D3, 1},
        {"encoder_U", o.enc[0].Ucat, D, 2 * D, D3, 2},
        {"encoder_Wx", o.enc[0].Wcat + 2 * D, W, D, D3, 2},
        {"encoder_bx", o.enc[0].bcat + 2 * D, 1, D, D3, 1},
        {"encoder_Ux", o.enc[0].Ucat + 2 * D, D, D, D3, 2},
        {"encoder_r_W", o.enc[1].Wcat, W, 2 * D, D3, 2},
        {"encoder_r_b", o.enc[1].bcat, 1, 2 * D, D3, 1},
        {"encoder_r_U", o.enc[1].Ucat, D, 2 * D, D3, 2},
        {"encoder_r_Wx", o.enc[1].Wcat + 2 * D, W, D, D3, 2},
        {"encoder_r_bx", o.enc[1].bcat + 2 * D, 1, D, D3, 1},
        {"encoder_r_Ux", o.enc[1].Ucat + 2 * D, D, D, D3, 2},
        {"ff_state_W", o.ff_state_W, C, D, D, 2},
        {"ff_state_b", o.ff_state_b, 1, D, D, 1},
        {"decoder_W", o.dec.Wcat, W, 2 * D, D3, 2},
        {"decoder_U", o.dec.Ucat, D, 2 * D, D3, 2},
        {"decoder_b", o.dec.bcat, 1, 2 * D, D3, 1},
        {"decoder_Wx", o.dec.Wcat + 2 * D, W, D, D3, 2},
        {"decoder_Ux", o.dec.Ucat + 2 * D, D, D, D3, 2},
        {"decoder_bx", o.dec.bcat + 2 * D, 1, D, D3, 1},
        {"decoder_U_1", o.U1cat, D, 2 * D, D3, 2},
        {"decoder_W_1", o.W1cat, C, 2 * D, D3, 2},
        {"decoder_b_1", o.b1cat, 1, 2 * D, D3, 1},
        {"decoder_Wx_1", o.W1cat + 2 * D, C, D, D3, 2},
        {"decoder_Ux_1", o.U1cat + 2 * D, D, D, D3, 2},
        {"decoder_bx_1", o.b1cat + 2 * D, 1, D, D3, 1},
        {"decoder_W_att", o.W_att, D, A, A, 2},
        {"decoder_Wc_att", o.Wc_att, C, A, A, 2},
        {"decoder_b_att", o.b_att, 1, A, A, 1},
        {"decoder_U_att", o.U_att, A, 1, 1, 2},
        {"decoder_c_att", o.c_att, 1, 1, 1, 1},
        {"decoder_W_con", o.W_con, C, 1, 1, 2},
        {"decoder_U_con", o.U_con, C, 1, 1, 2},
        {"decoder_D_wei", o.D_wei, 1, A, A, 2},
        {"ff_logit_lstm_W", o.lstm_W, D, W, W, 2},
        {"ff_logit_lstm_b", o.lstm_b, 1, W, W, 1},
        {"ff_logit_prev_W", o.prev_W, W, W, W, 2},
        {"ff_logit_prev_b", o.prev_b, 1, W, W, 1},
        {"ff_logit_ctx_W", o.ctxr_W, C, W, W, 2},
        {"ff_logit_ctx_b", o.ctxr_b, 1, W, W, 1},
        {"ff_logit_W", o.logit_W, W, V, V, 2},
        {"ff_logit_b", o.logit_b, 1, V, V, 1},
    };
    if (views) {
        for (int i = 0; i < NATS_NUM_PARAMS; ++i) {
            memset(&views[i], 0, sizeof(views[i]));
            strncpy(views[i].name, defs[i].name, sizeof(views[i].name) - 1);
            views[i].offset = defs[i].off;
            views[i].rows = defs[i].rows; views[i].cols = defs[i].cols; views[i].ld = defs[i].ld;
            views[i].ndim = defs[i].ndim;
        }
    }
    if (total_floats) *total_floats = o.total;
    return 0;
}

// ------------------------------------------------------------------------------------------ debug
int nats_debug_gemm(nats_ctx_t* ctx, void* stream, int path, int transA, int transB, int M, int N, int K,
                    const float* A, int lda, const float* B, int ldb, float* C, int ldc, const float* bias,
                    int accumulate, int splitk, int batch, int64_t strideA, int64_t strideB, int64_t strideC) {
    NATS_REQUIRE(ctx && A && B && C, "null argument");
    GemmProblem p = gemm_problem(A, lda, B, ldb, C, ldc, M, N, K);
    p.bias = bias; p.accumulate = accumulate; p.batch = batch < 1 ? 1 : batch;
    p.strideA = strideA; p.strideB = strideB; p.strideC = strideC;
    if (splitk > 1) gemm_set_split(p, splitk, (long long)M * ldc);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (path == 1) return tc_gemm_launch(st, &p, 1, transA != 0, transB != 0);
    if (path == 2 || path == 3) {        // 3 = TMA-fed with the 128-row operand through registers (skinny shapes)
        NATS_REQUIRE(tma_gemm_eligible(&p, 1), "operands not TMA-compatible (alignment)");
        const int keep_ts = tma_gemm_get_ts();
        tma_gemm_set_ts(path == 3 ? 1 : 0);
        const int r = tma_gemm_launch(st, &p, 1, transA != 0, transB != 0);
        tma_gemm_set_ts(keep_ts);
        return r;
    }
    const int keep = gemm_get_tensor_cores();
    gemm_set_tensor_cores(0);
    const int r = gemm_launch(st, &p, 1, transA != 0, transB != 0, GEMM_CFG_AUTO);
    gemm_set_tensor_cores(keep);
    return r;
}

// ------------------------------------------------------------------------------------------ profiling
int nats_profile_enable(nats_ctx_t* ctx, int on) {
    (void)ctx;
    g_prof.recs.clear();
    g_prof.on = on != 0;
    return 0;
}
int nats_profile_num_classes(void) { return K_COUNT; }
const char* nats_profile_class_name(int cls) { return kclass_name(cls); }
int nats_profile_read(nats_ctx_t* ctx, int n_classes, double* ms, double* flops, double* bytes, int64_t* launches) {
    (void)ctx;
    NATS_REQUIRE(n_classes >= K_COUNT && ms && flops && bytes && launches, "profile_read buffers");
    NATS_CUDA_OK(cudaDeviceSynchronize());
    for (int i = 0; i < n_classes; ++i) { ms[i] = 0; flops[i] = 0; bytes[i] = 0; launches[i] = 0; }
    for (size_t i = 0; i < g_prof.recs.size(); ++i) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, g_prof.ev[2 * i], g_prof.ev[2 * i + 1]) != cudaSuccess) continue;
        const ProfRec& r = g_prof.recs[i];
        ms[r.cls] += t; flops[r.cls] += r.flops; bytes[r.cls] += r.bytes; launches[r.cls] += 1;
    }
    g_prof.recs.clear();
    return 0;
}

// ------------------------------------------------------------------------------------------ training
int64_t nats_train_workspace_bytes(const nats_dims_t* dims, int Tx, int Ty, int B) {
    if (check_dims(dims) != 0 || Tx < 1 || Ty < 1 || B < 1) return -1;
    return carve_train(*dims, Tx, Ty, B, nullptr).bytes;
}

#define NATS_TRAIN_PROLOGUE()                                                                      \
    NATS_REQUIRE(ctx != nullptr, "ctx");                                                           \
    NATS_TRY(check_dims(dims));                                                                    \
    NATS_REQUIRE(Tx >= 1 && Ty >= 1 && B >= 1, "shape");                                           \
    NATS_REQUIRE(ws != nullptr, "workspace");                                                      \
    const TrainWS w = carve_train(*dims, Tx, Ty, B, ws);                                           \
    NATS_REQUIRE(ws_bytes >= w.bytes, "workspace too small (see nats_train_workspace_bytes)");     \
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream)

int nats_encoder_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                     const float* x_mask, int Tx, int Ty, int B, void* ws, int64_t ws_bytes) {
    NATS_TRAIN_PROLOGUE();
    return train_encoder_fwd(ctx, st, *dims, params, x, x_mask, Tx, B, w);
}

int nats_decoder_scan_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                          const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B, void* ws,
                          int64_t ws_bytes) {
    NATS_TRAIN_PROLOGUE();
    return train_decoder_fwd(ctx, st, *dims, params, y, x_mask, y_mask, Tx, Ty, B, w);
}

int nats_readout_nll_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                         const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws, int64_t ws_bytes,
                         float* cost) {
    NATS_TRAIN_PROLOGUE();
    return train_readout_fwd(ctx, st, *dims, params, y, y_mask, Ty, B, w, cost);
}

int nats_readout_nll_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                         const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws, int64_t ws_bytes,
                         float scale, float* grads) {
    NATS_TRAIN_PROLOGUE();
    return train_readout_bwd(ctx, st, *dims, params, y, y_mask, Ty, B, w, scale, grads);
}

int nats_decoder_scan_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params,
                          const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B, void* ws,
                          int64_t ws_bytes, float* grads) {
    NATS_TRAIN_PROLOGUE();
    return train_decoder_bwd(ctx, st, *dims, params, y, x_mask, y_mask, Tx, Ty, B, w, grads);
}

int nats_encoder_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                     const float* x_mask, const int64_t* y, int Tx, int Ty, int B, void* ws, int64_t ws_bytes,
                     float* grads) {
    NATS_TRAIN_PROLOGUE();
    return train_encoder_bwd(ctx, st, *dims, params, x, x_mask, y, Tx, Ty, B, w, grads);
}

int nats_train_fwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                   const float* x_mask, const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws,
                   int64_t ws_bytes, float* cost) {
    NATS_TRAIN_PROLOGUE();
    NATS_REQUIRE(x && x_mask && y && y_mask && cost && params, "null argument");
    NATS_TRY(train_encoder_fwd(ctx, st, *dims, params, x, x_mask, Tx, B, w));
    NATS_TRY(train_decoder_fwd(ctx, st, *dims, params, y, x_mask, y_mask, Tx, Ty, B, w));
    NATS_TRY(train_readout_fwd(ctx, st, *dims, params, y, y_mask, Ty, B, w, cost));
    return 0;
}

int64_t nats_grad_split(const nats_dims_t* dims) {
    if (check_dims(dims) != 0) return -1;
    return param_offsets(*dims).ff_state_W;      // [Wemb | encoder | encoder_r] come first in the flat layout
}

int nats_train_bwd_begin(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                         const float* x_mask, const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws,
                         int64_t ws_bytes, float scale, float* grads) {
    NATS_TRAIN_PROLOGUE();
    NATS_REQUIRE(x && x_mask && y && y_mask && grads && params, "null argument");
    const ParamOff o = param_offsets(*dims);
    NATS_CUDA_OK(memset_async(st, grads, 0, (size_t)(o.total + NATS_GRAD_TAIL) * sizeof(float)));
    NATS_TRY(cost_reduce(st, w.rowcost, Ty, B, nullptr, scale, grads + o.total));
    NATS_TRY(train_readout_bwd(ctx, st, *dims, params, y, y_mask, Ty, B, w, scale, grads));
    NATS_TRY(train_decoder_bwd(ctx, st, *dims, params, y, x_mask, y_mask, Tx, Ty, B, w, grads));
    return 0;
}

int nats_train_bwd_finish(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                          const float* x_mask, const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws,
                          int64_t ws_bytes, float scale, float* grads) {
    (void)scale; (void)y_mask;
    NATS_TRAIN_PROLOGUE();
    NATS_REQUIRE(x && x_mask && y && grads && params, "null argument");
    return train_encoder_bwd(ctx, st, *dims, params, x, x_mask, y, Tx, Ty, B, w, grads);
}

int nats_train_bwd(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                   const float* x_mask, const int64_t* y, const float* y_mask, int Tx, int Ty, int B, void* ws,
                   int64_t ws_bytes, float scale, float* grads) {
    NATS_TRY(nats_train_bwd_begin(ctx, stream, dims, params, x, x_mask, y, y_mask, Tx, Ty, B, ws, ws_bytes, scale, grads));
    return nats_train_bwd_finish(ctx, stream, dims, params, x, x_mask, y, y_mask, Tx, Ty, B, ws, ws_bytes, scale, grads);
}

const float* nats_train_ws_view(const nats_dims_t* dims, int Tx, int Ty, int B, void* ws, const char* name) {
    if (check_dims(dims) != 0 || !ws || !name) return nullptr;
    const TrainWS w = carve_train(*dims, Tx, Ty, B, ws);
    if (!strcmp(name, "ctx")) return w.cc;
    if (!strcmp(name, "init_state")) return w.init_state;
    if (!strcmp(name, "dec_h")) return w.d_h2;
    if (!strcmp(name, "dec_ctx")) return w.d_ctx;
    if (!strcmp(name, "dec_alpha")) return w.d_alpha;
    if (!strcmp(name, "pctx")) return w.pctx;
    if (!strcmp(name, "logits")) return w.logits;
    if (!strcmp(name, "dcc")) return w.dcc;
    if (!strcmp(name, "dmean")) return w.dmean;
    return nullptr;
}

// ------------------------------------------------------------------------------------------ sampler
int64_t nats_sampler_workspace_bytes(const nats_dims_t* dims, int Tx, int n) {
    if (check_dims(dims) != 0 || Tx < 1 || n < 1) return -1;
    return carve_sampler(*dims, Tx, n, nullptr).bytes;
}

int nats_sampler_init(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* x,
                      const float* x_mask, int Tx, int n, void* ws, int64_t ws_bytes, float* init_state, float* ctx_out,
                      float* pctx_out) {
    NATS_REQUIRE(ctx && ws && params && x && init_state && ctx_out, "null argument");
    NATS_TRY(check_dims(dims));
    NATS_REQUIRE(Tx >= 1 && n >= 1, "shape");
    const SamplerWS w = carve_sampler(*dims, Tx, n, ws);
    NATS_REQUIRE(ws_bytes >= w.bytes, "workspace too small (see nats_sampler_workspace_bytes)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EncBufs e;
    memset(&e, 0, sizeof(e));
    e.emb_x = w.emb_x;
    e.xproj[0] = w.xproj[0]; e.xproj[1] = w.xproj[1];
    e.cc = ctx_out; e.ctxsum = w.ctxsum; e.xlen = w.xlen; e.xinv = w.xinv; e.ctx_mean = w.ctx_mean;
    e.init_state = init_state; e.part_a = w.part_a;
    e.gemm_scratch = w.gemm_scratch; e.gemm_scratch_floats = w.gemm_scratch_floats;
    e.enc_scratch = w.enc_scratch; e.enc_scratch_floats = w.enc_scratch_floats;
    e.enc_counters = w.enc_counters; e.enc_counter_ints = w.enc_counter_ints;
    NATS_TRY(encoder_forward(ctx, st, *dims, params, x, x_mask, Tx, n, e));       // NULL: no masks (nats.py:801-804, 810)
    if (pctx_out) {
        const ParamOff o = param_offsets(*dims);
        const int A = dims->dim_att, C = 2 * dims->dim;
        GemmProblem p = gemm_problem(ctx_out, C, params + o.Wc_att, A, pctx_out, A, Tx * n, A, C);
        p.bias = params + o.b_att;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    }
    return 0;
}

}  // extern "C"

namespace {

// f_next on n rows; row b attends to source b / rows_per_src of ctx_in / pctx_in (element (t, s, c) at
// t * tstride + s * bstride + c), of which src_len[s] positions are valid (NULL: all Tx)
int sampler_next(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* y,
                 const float* ctx_in, int64_t ctx_tstride, int64_t ctx_bstride, const float* pctx_in,
                 int64_t pctx_tstride, int64_t pctx_bstride, int rows_per_src, const int32_t* src_len, const float* state,
                 const float* acc_ctx, const float* acc_alpha, int Tx, int n, uint64_t rng_seed, uint64_t rng_step, void* ws,
                 int64_t ws_bytes, float* probs, int64_t* sample, float* state_out, float* alphaT, float* ctxs,
                 float* acc_ctx_out, float* acc_alpha_out) {
    NATS_REQUIRE(ctx && ws && params && y && ctx_in && state && acc_ctx && acc_alpha, "null argument");
    NATS_REQUIRE(probs && state_out && alphaT && ctxs && acc_ctx_out && acc_alpha_out, "null output");
    NATS_TRY(check_dims(dims));
    NATS_REQUIRE(Tx >= 1 && n >= 1, "shape");
    const SamplerWS w = carve_sampler(*dims, Tx, n, ws);
    NATS_REQUIRE(ws_bytes >= w.bytes, "workspace too small (see nats_sampler_workspace_bytes)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const ParamOff o = param_offsets(*dims);
    const int W = dims->dim_word, D = dims->dim, A = dims->dim_att, V = dims->n_words, C = 2 * D, D3 = 3 * D;

    // previous word embedding, -1 -> zeros (nats.py:827-829), and its projections (nats.py:487-491)
    NATS_TRY(gather_rows(st, params + o.Wemb, y, n, W, V, 0, w.emb_y));
    {
        GemmProblem p = gemm_problem(w.emb_y, W, params + o.dec.Wcat, D3, w.xproj_y, D3, n, D3, W);
        p.bias = params + o.dec.bcat;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    }
    const float* pctx = pctx_in;
    long long pts = pctx_tstride, pbs = pctx_bstride;
    if (!pctx) {   // the reference recomputes pctx_ inside every f_next call (nats.py:493-494)
        GemmProblem p;
        if (ctx_bstride == 0) {
            p = gemm_problem(ctx_in, (int)ctx_tstride, params + o.Wc_att, A, w.pctx, A, Tx, A, C);
            pts = A; pbs = 0;
        } else {
            NATS_REQUIRE(ctx_bstride == C && ctx_tstride == (int64_t)n * C, "pctx recompute needs a dense [Tx,n,C] context");
            p = gemm_problem(ctx_in, C, params + o.Wc_att, A, w.pctx, A, Tx * n, A, C);
            pts = (long long)n * A; pbs = A;
        }
        p.bias = params + o.b_att;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
        pctx = w.pctx;
    }
    DecStep s;
    memset(&s, 0, sizeof(s));
    s.n = n; s.Tx = Tx;
    s.h_prev = state; s.xproj = w.xproj_y;
    s.ymask = nullptr; s.xmask = nullptr;                       // mask=None, no context mask (nats.py:472-473, 538)
    s.rows_per_src = rows_per_src; s.src_len = src_len;         // a source's padding gets alpha = 0 (the x_mask of nats.py:538-540)
    s.pctx = pctx; s.pctx_ts = pts; s.pctx_bs = pbs;
    s.cc = ctx_in; s.cc_ts = ctx_tstride; s.cc_bs = ctx_bstride;
    s.acc_alpha_in = acc_alpha; s.acc_ctx_in = acc_ctx;
    s.h1 = w.h1; s.ps_save = w.ps; s.escore = w.escore;
    s.alpha_out = alphaT; s.acc_alpha_out = acc_alpha_out; s.craw_out = w.craw; s.ctx_out = ctxs;
    s.acc_ctx_out = acc_ctx_out; s.h2 = state_out;
    s.part_a = w.part_a; s.part_b = w.part_b; s.part_c = w.part_c; s.part_d = w.part_d;
    NATS_TRY(decoder_step_forward(ctx, st, *dims, params, s));

    // readout (nats.py:850-861)
    NarrowProj np;
    memset(&np, 0, sizeof(np));
    np.x[0] = state_out; np.ldx[0] = D; np.W[0] = params + o.lstm_W; np.ldw[0] = W; np.bias[0] = params + o.lstm_b; np.K[0] = D;
    np.x[1] = w.emb_y;   np.ldx[1] = W; np.W[1] = params + o.prev_W; np.ldw[1] = W; np.bias[1] = params + o.prev_b; np.K[1] = W;
    np.x[2] = ctxs;      np.ldx[2] = C; np.W[2] = params + o.ctxr_W; np.ldw[2] = W; np.bias[2] = params + o.ctxr_b; np.K[2] = C;
    np.n = n; np.N = W; np.out = w.L; np.ldo = W; np.act_tanh = 1;
    GemmProblem p;
    if (narrow_proj_eligible(np)) {
        NATS_TRY(narrow_proj(st, np));                          // one launch: three products + biases + tanh, exact fp32
    } else {
        p = gemm_problem(state_out, D, params + o.lstm_W, W, w.L, W, n, W, D);
        p.bias = params + o.lstm_b;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
        p = gemm_problem(w.emb_y, W, params + o.prev_W, W, w.L, W, n, W, W);
        p.bias = params + o.prev_b; p.accumulate = 1;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
        p = gemm_problem(ctxs, C, params + o.ctxr_W, W, w.L, W, n, W, C);
        p.bias = params + o.ctxr_b; p.accumulate = 1;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
        NATS_TRY(tanh_inplace(st, w.L, (long long)n * W));
    }
    p = gemm_problem(w.L, W, params + o.logit_W, V, w.logits, V, n, V, W);
    p.bias = params + o.logit_b;
    NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    NATS_TRY(softmax_sample_rows(st, w.logits, n, V, probs, sample, rng_seed, rng_step));
    return 0;
}

}  // namespace

extern "C" {

int nats_sampler_next(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const float* params, const int64_t* y,
                      const float* ctx_in, int64_t ctx_tstride, int64_t ctx_bstride, const float* pctx_in,
                      int64_t pctx_tstride, int64_t pctx_bstride, const float* state, const float* acc_ctx,
                      const float* acc_alpha, int Tx, int n, uint64_t rng_seed, uint64_t rng_step, void* ws,
                      int64_t ws_bytes, float* probs, int64_t* sample, float* state_out, float* alphaT, float* ctxs,
                      float* acc_ctx_out, float* acc_alpha_out) {
    // a zero batch stride: one source shared by all n rows; otherwise one source per row
    return sampler_next(ctx, stream, dims, params, y, ctx_in, ctx_tstride, ctx_bstride, pctx_in, pctx_tstride, pctx_bstride,
                        ctx_bstride == 0 ? n : 1, nullptr, state, acc_ctx, acc_alpha, Tx, n, rng_seed, rng_step, ws, ws_bytes,
                        probs, sample, state_out, alphaT, ctxs, acc_ctx_out, acc_alpha_out);
}

// ------------------------------------------------------------------------------------------ optimiser
int nats_grad_clip(nats_ctx_t* ctx, void* stream, int64_t n, const float* params, float* grads, float decay_c,
                   float clip_c, float* stats) {
    NATS_REQUIRE(ctx && grads && stats, "null argument");
    NATS_REQUIRE(!(decay_c > 0.f) || params, "params needed for decay");
    return grad_clip(ctx, reinterpret_cast<cudaStream_t>(stream), n, params, grads, decay_c, clip_c, stats);
}
int nats_adadelta_grad_shared(nats_ctx_t* ctx, void* stream, int64_t n, const float* zg, float* rg2, float rho) {
    (void)ctx;
    return adadelta_grad_shared(reinterpret_cast<cudaStream_t>(stream), n, zg, rg2, rho);
}
int nats_adadelta_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* zg, float* ru2,
                         const float* rg2, float rho, float eps) {
    (void)ctx;
    return adadelta_update(reinterpret_cast<cudaStream_t>(stream), n, params, zg, ru2, rg2, rho, eps);
}
int nats_adam_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* g, float* m, float* v,
                     int64_t step) {
    (void)ctx;
    return adam_update(reinterpret_cast<cudaStream_t>(stream), n, params, g, m, v, step);
}
int nats_rmsprop_grad_shared(nats_ctx_t* ctx, void* stream, int64_t n, const float* zg, float* rg, float* rg2) {
    (void)ctx;
    return rmsprop_grad_shared(reinterpret_cast<cudaStream_t>(stream), n, zg, rg, rg2);
}
int nats_rmsprop_update(nats_ctx_t* ctx, void* stream, int64_t n, float* params, const float* zg, float* ud,
                        const float* rg, const float* rg2) {
    (void)ctx;
    return rmsprop_update(reinterpret_cast<cudaStream_t>(stream), n, params, zg, ud, rg, rg2);
}

// ------------------------------------------------------------------------------------------ beam search
int nats_beam_distraction_scores(nats_ctx_t* ctx, void* stream, const float* hist_alpha, const float* hist_ctx,
                                 const float* hist_state, int len_cap, int hist_len, int live_k, int Tx, int C, int D,
                                 const float* cur_alpha, const float* cur_ctx, const float* cur_state, float kl_factor,
                                 float ctx_factor, float state_factor, float* scratch, float* out) {
    (void)ctx;
    return beam_distraction_scores(reinterpret_cast<cudaStream_t>(stream), hist_alpha, hist_ctx, hist_state, len_cap,
                                   hist_len, live_k, Tx, C, D, cur_alpha, cur_ctx, cur_state, kl_factor, ctx_factor,
                                   state_factor, nullptr, 0, scratch, out);
}
int nats_beam_topk(nats_ctx_t* ctx, void* stream, const float* probs, int n, int n_words, int k, int mask_unk,
                   float* out_p, int32_t* out_idx) {
    (void)ctx;
    return beam_topk(reinterpret_cast<cudaStream_t>(stream), probs, n, n_words, k, mask_unk, out_p, out_idx);
}

int nats_beam_reorder_append(nats_ctx_t* ctx, void* stream, const float* src, float* dst, const float* cur,
                             const int32_t* parent, int n_new, int len_cap, int hist_len, int dim) {
    (void)ctx;
    return beam_reorder_append(reinterpret_cast<cudaStream_t>(stream), src, dst, cur, parent, n_new, len_cap, hist_len,
                               dim);
}

int nats_beam_select(nats_ctx_t* ctx, void* stream, const float* top_p, const int32_t* top_i, const float* pen, int k,
                     int maxlen, int step, int32_t* counters, float* scores, int32_t* tokens, int32_t* parents,
                     int64_t* next_w, int32_t* out_tokens, int32_t* out_len, float* out_score, int32_t* fin_parent,
                     int32_t* host_counters) {
    (void)ctx;
    NATS_REQUIRE(top_p && top_i && counters && scores && tokens && parents && next_w && out_tokens && out_len && out_score &&
                     fin_parent, "null argument");
    return beam_select(reinterpret_cast<cudaStream_t>(stream), top_p, top_i, pen, 1, k, maxlen, step, counters, scores, tokens,
                       parents, reinterpret_cast<long long*>(next_w), out_tokens, out_len, out_score, fin_parent, host_counters);
}

int nats_beam_advance(nats_ctx_t* ctx, void* stream, const int32_t* parents, const int32_t* fin_parent,
                      const int32_t* counters, int k, int len_cap, int step, int Tx, int C, int D, const float* state_o,
                      float* state_n, const float* acc_ctx_o, float* acc_ctx_n, const float* acc_alpha_o, float* acc_alpha_n,
                      const float* cur_alpha, const float* cur_ctx, const float* cur_state, const float* hist_alpha_src,
                      float* hist_alpha_dst, const float* hist_ctx_src, float* hist_ctx_dst, const float* hist_state_src,
                      float* hist_state_dst, float* out_alpha) {
    (void)ctx;
    NATS_REQUIRE(parents && fin_parent && counters && state_o && state_n && acc_ctx_o && acc_ctx_n && acc_alpha_o &&
                     acc_alpha_n && cur_alpha && hist_alpha_src && hist_alpha_dst && out_alpha, "null argument");
    NATS_REQUIRE(hist_ctx_src == nullptr || (hist_ctx_dst && hist_state_src && hist_state_dst && cur_ctx && cur_state),
                 "context / state histories come together");
    return beam_advance(reinterpret_cast<cudaStream_t>(stream), parents, fin_parent, counters, 1, k, len_cap, step, Tx, C, D,
                        state_o, state_n, acc_ctx_o, acc_ctx_n, acc_alpha_o, acc_alpha_n, cur_alpha, cur_ctx, cur_state,
                        hist_alpha_src, hist_alpha_dst, hist_ctx_src, hist_ctx_dst, hist_state_src, hist_state_dst, out_alpha);
}

}  // extern "C"

namespace {

// One beam step of a group of n_src sentences x k rows (nats.py:957-1066 for each sentence): f_next on all rows, each
// attending to its own source (ctx [Tx, n_src, C]; n_src = 1 with src_len NULL is the single-sentence layout [Tx, C]),
// distraction scores of the live rows, per-row top-k, one selection warp per sentence, one gather launch.
int beam_step_group(nats_ctx_t* ctx, cudaStream_t st, const nats_dims_t* dims, const nats_beam_step_t* a, int n_src,
                    const int32_t* src_len, int step) {
    NATS_REQUIRE(ctx && dims && a, "null argument");
    NATS_REQUIRE(a->k >= 1 && a->k <= 32 && a->maxlen >= 1 && step >= 0 && step < a->maxlen, "beam step shape (1 <= k <= 32)");
    NATS_REQUIRE(n_src >= 1 && (long long)n_src * a->k <= 65535, "beam group size");
    NATS_TRY(check_dims(dims));
    const int D = dims->dim, C = 2 * D, A = dims->dim_att, V = dims->n_words, k = a->k, Tx = a->Tx, n = n_src * k;
    void* stream = reinterpret_cast<void*>(st);
    const int64_t cbs = n_src == 1 ? 0 : C, pbs = n_src == 1 ? 0 : A;
    NATS_TRY(sampler_next(ctx, stream, dims, a->params, a->next_w, a->ctx, (int64_t)n_src * C, cbs, a->pctx, (int64_t)n_src * A,
                          pbs, k, src_len, a->state_in, a->acc_ctx_in, a->acc_alpha_in, Tx, n, 0, 0, a->ws, a->ws_bytes,
                          a->probs, nullptr, a->state_out, a->alphaT, a->ctxs, a->acc_ctx_out, a->acc_alpha_out));
    const bool distract = a->kl_factor > 0.f || a->ctx_factor > 0.f || a->state_factor > 0.f;
    const bool use_pen = distract && step > 0;
    if (use_pen) {
        NATS_REQUIRE(a->hist_ctx_in && a->hist_state_in && a->scratch && a->pen, "distraction buffers");
        NATS_TRY(beam_distraction_scores(st, a->hist_alpha_in, a->hist_ctx_in, a->hist_state_in, a->maxlen, step, n, Tx, C, D,
                                         a->alphaT, a->ctxs, a->state_out, a->kl_factor, a->ctx_factor, a->state_factor,
                                         a->counters, k, a->scratch, a->pen));
    }
    NATS_REQUIRE(a->probs && a->top_p && a->top_i && a->counters && a->scores && a->tokens && a->parents && a->next_w &&
                     a->out_tokens && a->out_len && a->out_score && a->fin_parent, "null argument");
    NATS_REQUIRE(a->state_next && a->acc_ctx_next && a->acc_alpha_next && a->hist_alpha_in && a->hist_alpha_out && a->out_alpha,
                 "null argument");
    NATS_REQUIRE(!distract || (a->hist_ctx_out && a->hist_state_out), "distraction histories");
    NATS_TRY(beam_topk(st, a->probs, n, V, k, a->use_unk ? 0 : 1, a->top_p, a->top_i));
    NATS_TRY(beam_select(st, a->top_p, a->top_i, use_pen ? a->pen : nullptr, n_src, k, a->maxlen, step, a->counters, a->scores,
                         a->tokens, a->parents, reinterpret_cast<long long*>(const_cast<int64_t*>(a->next_w)), a->out_tokens,
                         a->out_len, a->out_score, a->fin_parent, a->host_counters));
    NATS_TRY(beam_advance(st, a->parents, a->fin_parent, a->counters, n_src, k, a->maxlen, step, Tx, C, D, a->state_out,
                          a->state_next, a->acc_ctx_out, a->acc_ctx_next, a->acc_alpha_out, a->acc_alpha_next, a->alphaT, a->ctxs,
                          a->state_out, a->hist_alpha_in, a->hist_alpha_out, distract ? a->hist_ctx_in : nullptr,
                          a->hist_ctx_out, a->hist_state_in, a->hist_state_out, a->out_alpha));
    return 0;
}

}  // namespace

extern "C" {

int nats_beam_step(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const nats_beam_step_t* a, int step) {
    return beam_step_group(ctx, reinterpret_cast<cudaStream_t>(stream), dims, a, 1, nullptr, step);
}

int nats_beam_step_many(nats_ctx_t* ctx, void* stream, const nats_dims_t* dims, const nats_beam_step_many_t* a, int step) {
    NATS_REQUIRE(a != nullptr, "null argument");
    NATS_REQUIRE(a->n_src >= 1, "n_src >= 1");
    NATS_REQUIRE(a->src_len != nullptr, "src_len");
    return beam_step_group(ctx, reinterpret_cast<cudaStream_t>(stream), dims, &a->beam, a->n_src, a->src_len, step);
}


}  // extern "C"
