// workspace.cuh -- flat parameter layout (packed, H100-native) and workspace carving.  Host-side only.
#pragma once
#include "common.cuh"
#include "gemm.cuh"
#include "ops.cuh"

namespace nats {

// Offsets (in floats) of the packed blocks inside the flat parameter / gradient buffer.
//   *_Wcat [W,3D] = [ X_W | X_Wx ]   *_bcat [3D] = [ X_b | X_bx ]   *_Ucat [D,3D] = [ X_U | X_Ux ]
//   dec_U1cat [D,3D] = [ U_1 | Ux_1 ]   dec_W1cat [C,3D] = [ W_1 | Wx_1 ]   dec_b1cat [3D] = [ b_1 | bx_1 ]
// (reference keeps these as separate tensors, nats.py:283-300, 392-420)
struct GruOff { int64_t Wcat, bcat, Ucat; };
struct ParamOff {
    int64_t Wemb;
    GruOff enc[2];
    int64_t ff_state_W, ff_state_b;
    GruOff dec;
    int64_t U1cat, W1cat, b1cat;
    int64_t W_att, Wc_att, b_att, U_att, c_att, W_con, U_con, D_wei;
    int64_t lstm_W, lstm_b, prev_W, prev_b, ctxr_W, ctxr_b, logit_W, logit_b;
    int64_t total;
};

inline ParamOff param_offsets(const nats_dims_t& d) {
    const int64_t V = d.n_words, W = d.dim_word, D = d.dim, A = d.dim_att, C = 2 * D;
    ParamOff o;
    int64_t off = 0;
    auto take = [&](int64_t n) { int64_t r = off; off += round_up64(n, 32); return r; };
    o.Wemb = take(V * W);
    for (int i = 0; i < 2; ++i) {
        o.enc[i].Wcat = take(W * 3 * D);
        o.enc[i].bcat = take(3 * D);
        o.enc[i].Ucat = take(D * 3 * D);
    }
    o.ff_state_W = take(C * D);
    o.ff_state_b = take(D);
    o.dec.Wcat = take(W * 3 * D);
    o.dec.bcat = take(3 * D);
    o.dec.Ucat = take(D * 3 * D);
    o.U1cat = take(D * 3 * D);
    o.W1cat = take(C * 3 * D);
    o.b1cat = take(3 * D);
    o.W_att = take(D * A);
    o.Wc_att = take(C * A);
    o.b_att = take(A);
    o.U_att = take(A);
    o.c_att = take(1);
    o.W_con = take(C);
    o.U_con = take(C);
    o.D_wei = take(A);
    o.lstm_W = take(D * W);
    o.lstm_b = take(W);
    o.prev_W = take(W * W);
    o.prev_b = take(W);
    o.ctxr_W = take(C * W);
    o.ctxr_b = take(W);
    o.logit_W = take(W * V);
    o.logit_b = take(V);
    o.total = off;
    return o;
}

constexpr int kStepMaxSplit = kGemmMaxSplit;

struct Carver {
    char* base;
    int64_t off;
    template <class T>
    T* take(int64_t n) {
        off = round_up64(off, 256);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += n * (int64_t)sizeof(T);
        return p;
    }
    float* f(int64_t n) { return take<float>(n); }
};

// Saved activations + scratch of one training problem (Tx, Ty, B).  Layouts: row index = t*B + b.
struct TrainWS {
    // ---- encoder (nats.py:700-724)
    float* emb_x;        // [Tx*B, W]            Wemb[x]
    float* xproj[2];     // [Tx*B, 3D]           emb.Wcat + bcat, indexed by source position (both directions)
    float* enc_r[2];     // [Tx*B, D] each: reset gate / update gate / candidate / h_prev.Ux, indexed by position
    float* enc_u[2];
    float* enc_c[2];
    float* enc_p[2];
    float* cc;           // [Tx*B, C]            context = [h_fwd | h_bwd]  (nats.py:713), written in place
    float* ctxsum;       // [B, C]               sum_t mask*ctx
    float* xlen;         // [B]                  sum_t mask
    float* xinv;         // [B]                  1 / xlen
    float* ctx_mean;     // [B, C]
    float* init_state;   // [B, D]
    float* part_a;       // [kStepMaxSplit, 2, B, 3D]   split-K slabs of the recurrent products (shared scratch)
    float* part_b;       // [kStepMaxSplit, B, 3D]
    float* part_c;       // [kStepMaxSplit, B, max(3D,C)]
    float* part_d;       // [kStepMaxSplit, B, A]
    // ---- decoder (nats.py:730-742)
    float* embs;         // [Ty*B, W]            shifted target embedding
    float* xproj_y;      // [Ty*B, 3D]
    float* pctx;         // [Tx*B, A]
    float* escore;       // [B, Tx]              scratch: attention energies of the current step
    float* d_h1;         // [Ty*B, D]
    float* d_r1; float* d_u1; float* d_c1; float* d_p1;   // [Ty*B, D]
    float* d_ps;         // [Ty*B, A]
    float* d_alpha;      // [Ty, B, Tx]
    float* d_accalpha;   // [Ty+1, B, Tx]        acc_alpha BEFORE step t at slot t
    float* d_craw;       // [Ty*B, C]
    float* d_ctx;        // [Ty*B, C]
    float* d_accctx;     // [(Ty+1)*B, C]
    float* d_r2; float* d_u2; float* d_c2; float* d_p2;   // [Ty*B, D]
    float* d_h2;         // [Ty*B, D]
    // ---- readout (nats.py:753-770)
    float* L;            // [Ty*B, W]            tanh(pre)
    float* logits;       // [Ty*B, V]            becomes d logits in the backward
    float* lse;          // [Ty*B]
    float* rowcost;      // [Ty*B]
    // ---- backward scratch
    float* dpre;         // [Ty*B, W]
    float* dh2_ro;       // [Ty*B, D]            d cost / d h2 through the readout
    float* dctx_ro;      // [Ty*B, C]
    float* dembs;        // [Ty*B, W]
    float* dG1;          // [Ty*B, 3D]  [dg2 | dp2]     (GRU_1: products with h1)
    float* dG1x;         // [Ty*B, 3D]  [dg2 | dpc2]    (GRU_1: products with ctx)
    float* dG2;          // [Ty*B, 3D]  [dg1 | dp1]     (GRU_2: products with h_)
    float* dG2x;         // [Ty*B, 3D]  [dg1 | dpc1]    (GRU_2: input side)
    float* dq;           // [Ty*B, C]
    float* dcraw;        // [Ty*B, C]
    float* dps;          // [Ty*B, A]
    float* dpctx;        // [Tx*B, A]
    float* dalpha;       // [B, Tx]
    float* dacc_alpha;   // [B, Tx]
    float* dacc_ctx;     // [2, B, C]   ping-pong
    float* dh_elem;      // [2, B, D]   elementwise part of d h_{t-1} (per direction for the encoder)
    float* dh1_elem;     // [B, D]
    float* gatt_part;    // [B, 2A+1]   per-sample partial sums of d U_att | d D_wei | d c_att over all steps
    float* att_dot_part; // [B, ceil(Tx/16)]           attention-backward scratch
    float* att_soft_part;// [B, ceil(Tx/16), 3A+1]
    float* dcc;          // [Tx*B, C]
    float* dinit;        // [B, D]
    float* dmean;        // [B, C]
    float* dGe[2];       // [Tx*B, 3D]  encoder [dg | dp]
    float* dGex[2];      // [Tx*B, 3D]  encoder [dg | dpc]
    float* demb_x;       // [Tx*B, W]
    float* gemm_scratch; // split-K slabs for gemm_auto
    int64_t gemm_scratch_floats;
    float* red_scratch;  // column-sum scratch: 64 * max(V, 3D, C) floats
    float* enc_scratch;  // persistent encoder kernels (enc_tc.cu): residual side buffer + K-partial words
    int64_t enc_scratch_floats;
    unsigned* enc_counters;
    int64_t enc_counter_ints;
    int64_t bytes;
};

inline TrainWS carve_train(const nats_dims_t& d, int Tx, int Ty, int B, void* base) {
    const int64_t W = d.dim_word, D = d.dim, A = d.dim_att, V = d.n_words, C = 2 * D;
    const int64_t XB = (int64_t)Tx * B, YB = (int64_t)Ty * B;
    TrainWS w;
    memset(&w, 0, sizeof(w));
    Carver c{reinterpret_cast<char*>(base), 0};
    w.emb_x = c.f(XB * W);
    for (int i = 0; i < 2; ++i) {
        w.xproj[i] = c.f(XB * 3 * D);
        w.enc_r[i] = c.f(XB * D); w.enc_u[i] = c.f(XB * D); w.enc_c[i] = c.f(XB * D); w.enc_p[i] = c.f(XB * D);
    }
    w.cc = c.f(XB * C);
    w.ctxsum = c.f(B * C); w.xlen = c.f(B); w.xinv = c.f(B); w.ctx_mean = c.f(B * C); w.init_state = c.f(B * D);
    w.part_a = c.f((int64_t)kStepMaxSplit * 2 * B * 3 * D);
    w.part_b = c.f((int64_t)kStepMaxSplit * B * 3 * D);
    w.part_c = c.f((int64_t)kStepMaxSplit * B * 3 * D);
    w.part_d = c.f((int64_t)kStepMaxSplit * B * (A > D ? A : D));
    w.embs = c.f(YB * W); w.xproj_y = c.f(YB * 3 * D); w.pctx = c.f(XB * A); w.escore = c.f((int64_t)B * Tx);
    w.d_h1 = c.f(YB * D);
    w.d_r1 = c.f(YB * D); w.d_u1 = c.f(YB * D); w.d_c1 = c.f(YB * D); w.d_p1 = c.f(YB * D);
    w.d_ps = c.f(YB * A);
    w.d_alpha = c.f(YB * Tx); w.d_accalpha = c.f((YB + B) * Tx);
    w.d_craw = c.f(YB * C); w.d_ctx = c.f(YB * C); w.d_accctx = c.f((YB + B) * C);
    w.d_r2 = c.f(YB * D); w.d_u2 = c.f(YB * D); w.d_c2 = c.f(YB * D); w.d_p2 = c.f(YB * D);
    w.d_h2 = c.f(YB * D);
    w.L = c.f(YB * W); w.logits = c.f(YB * V); w.lse = c.f(YB); w.rowcost = c.f(YB);
    w.dpre = c.f(YB * W); w.dh2_ro = c.f(YB * D); w.dctx_ro = c.f(YB * C); w.dembs = c.f(YB * W);
    w.dG1 = c.f(YB * 3 * D); w.dG1x = c.f(YB * 3 * D); w.dG2 = c.f(YB * 3 * D); w.dG2x = c.f(YB * 3 * D);
    w.dq = c.f(YB * C); w.dcraw = c.f(YB * C); w.dps = c.f(YB * A); w.dpctx = c.f(XB * A);
    w.dalpha = c.f((int64_t)B * Tx); w.dacc_alpha = c.f((int64_t)B * Tx); w.dacc_ctx = c.f(2 * B * C);
    w.dh_elem = c.f(2 * B * D); w.dh1_elem = c.f(B * D);
    w.gatt_part = c.f(B * (2 * A + 1));
    w.att_dot_part = c.f((int64_t)B * ((Tx + 15) / 16));
    w.att_soft_part = c.f((int64_t)B * ((Tx + 15) / 16) * (3 * A + 1));
    w.dcc = c.f(XB * C); w.dinit = c.f(B * D); w.dmean = c.f(B * C);
    for (int i = 0; i < 2; ++i) { w.dGe[i] = c.f(XB * 3 * D); w.dGex[i] = c.f(XB * 3 * D); }
    w.demb_x = c.f(XB * W);
    w.gemm_scratch_floats = 16LL << 20;      // split-K slabs: up to 4 x [D,3D] at D = 1000 (the deep d[U|Ux] products)
    w.gemm_scratch = c.f(w.gemm_scratch_floats);
    { int64_t mx = V; if (3 * D > mx) mx = 3 * D; w.red_scratch = c.f(64 * mx); }
    w.enc_scratch_floats = enc_tc_scratch_floats(B, (int)D);
    w.enc_scratch = c.f(w.enc_scratch_floats);
    w.enc_counter_ints = enc_tc_counter_ints();
    w.enc_counters = c.take<unsigned>(w.enc_counter_ints);
    w.bytes = round_up64(c.off, 256);
    return w;
}

// Sampler workspace (f_init / f_next), n hypotheses / sentences.
struct SamplerWS {
    float* emb_x;       // [Tx*n, W]
    float* xproj[2];    // [Tx*n, 3D]
    float* ctxsum;      // [n, C]
    float* ctx_mean;    // [n, C]
    float* xlen; float* xinv;   // [n]
    float* part_a;      // [kStepMaxSplit, 2, n, 3D]
    float* part_b;      // [kStepMaxSplit, n, 3D]
    float* part_c;      // [kStepMaxSplit, n, 3D]
    float* part_d;      // [kStepMaxSplit, n, max(A, D)]
    float* emb_y;       // [n, W]
    float* xproj_y;     // [n, 3D]
    float* pctx;        // [Tx*n, A]   (only when f_next must recompute it)
    float* escore;      // [n, Tx]
    float* h1;          // [n, D]
    float* ps;          // [n, A]
    float* craw;        // [n, C]
    float* L;           // [n, W]
    float* logits;      // [n, V]
    float* gemm_scratch;
    int64_t gemm_scratch_floats;
    float* enc_scratch;
    int64_t enc_scratch_floats;
    unsigned* enc_counters;
    int64_t enc_counter_ints;
    int64_t bytes;
};

inline SamplerWS carve_sampler(const nats_dims_t& d, int Tx, int n, void* base) {
    const int64_t W = d.dim_word, D = d.dim, A = d.dim_att, V = d.n_words, C = 2 * D;
    const int64_t XB = (int64_t)Tx * n;
    SamplerWS w;
    memset(&w, 0, sizeof(w));
    Carver c{reinterpret_cast<char*>(base), 0};
    w.emb_x = c.f(XB * W);
    for (int i = 0; i < 2; ++i) w.xproj[i] = c.f(XB * 3 * D);
    w.ctxsum = c.f(n * C); w.ctx_mean = c.f(n * C); w.xlen = c.f(n); w.xinv = c.f(n);
    w.part_a = c.f((int64_t)kStepMaxSplit * 2 * n * 3 * D);
    w.part_b = c.f((int64_t)kStepMaxSplit * n * 3 * D);
    w.part_c = c.f((int64_t)kStepMaxSplit * n * 3 * D);
    w.part_d = c.f((int64_t)kStepMaxSplit * n * (A > D ? A : D));
    w.emb_y = c.f(n * W); w.xproj_y = c.f(n * 3 * D); w.pctx = c.f(XB * A); w.escore = c.f((int64_t)n * Tx);
    w.h1 = c.f(n * D); w.ps = c.f(n * A); w.craw = c.f(n * C); w.L = c.f(n * W); w.logits = c.f(n * V);
    w.gemm_scratch_floats = 4LL << 20;
    w.gemm_scratch = c.f(w.gemm_scratch_floats);
    w.enc_scratch_floats = enc_tc_scratch_floats(n, (int)D);
    w.enc_scratch = c.f(w.enc_scratch_floats);
    w.enc_counter_ints = enc_tc_counter_ints();
    w.enc_counters = c.take<unsigned>(w.enc_counter_ints);
    w.bytes = round_up64(c.off, 256);
    return w;
}

}  // namespace nats
