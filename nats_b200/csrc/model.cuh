// model.cuh -- orchestration of the hot path on top of gemm + ops (internal).
#pragma once
#include "common.cuh"
#include "gemm.cuh"
#include "ops.cuh"
#include "workspace.cuh"

namespace nats {

struct EncBufs {
    float* emb_x;
    float* xproj[2];
    float* r[2]; float* u[2]; float* c[2]; float* p[2];   // NULL = do not save (sampler)
    float* cc;            // [Tx, n, C] dense
    float* ctxsum; float* xlen; float* xinv; float* ctx_mean; float* init_state;
    float* part_a;
    float* gemm_scratch; long long gemm_scratch_floats;
    float* enc_scratch; long long enc_scratch_floats;      // persistent encoder kernel (enc_tc.cu): NULL = per-step path
    unsigned* enc_counters; long long enc_counter_ints;
};
// bi-GRU encoder + masked mean + ff_state (nats.py:700-724 / 795-813)
int encoder_forward(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                    const int64_t* x, const float* x_mask, int Tx, int n, const EncBufs& e);

struct DecStep {
    int n, Tx;
    const float* h_prev;      // [n,D]
    const float* xproj;       // [n,3D]
    const float* ymask;       // [n] or NULL
    const float* xmask;       // [Tx,n] or NULL
    int rows_per_src;         // row b attends to source b / rows_per_src (0 = 1); see AttFwd
    const int32_t* src_len;   // [sources] or NULL (= Tx)
    const float* pctx; long long pctx_ts, pctx_bs;
    const float* cc; long long cc_ts, cc_bs;
    const float* acc_alpha_in; const float* acc_ctx_in;
    float* h1; float* r1; float* u1; float* c1; float* p1;     // r1..p1 NULL = no save
    float* ps_save; float* escore;
    float* alpha_out; float* acc_alpha_out; float* craw_out; float* ctx_out; float* acc_ctx_out;
    float* r2; float* u2; float* c2; float* p2; float* h2;
    float* part_a; float* part_b; float* part_c; float* part_d;
};
// one _step_slice (nats.py:498-572)
int decoder_step_forward(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                         const DecStep& s);

int train_encoder_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* x, const float* x_mask, int Tx, int B, const TrainWS& w);
int train_decoder_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                      const TrainWS& w);
int train_readout_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* y_mask, int Ty, int B, const TrainWS& w, float* cost);
int train_readout_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* y_mask, int Ty, int B, const TrainWS& w, float scale,
                      const float* weight /* [B] or NULL */, float* grads);
int train_decoder_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                      const TrainWS& w, float* grads);
int train_encoder_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* x, const float* x_mask, const int64_t* y, int Tx, int Ty, int B,
                      const TrainWS& w, float* grads);

}  // namespace nats
