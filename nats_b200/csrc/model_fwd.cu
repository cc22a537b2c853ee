// model_fwd.cu -- forward orchestration: encoder, decoder step / scan, readout.
#include "model.cuh"

namespace nats {

// ------------------------------------------------------------------------------------------------
// encoder: embedding gather, input projections of both directions (one grouped GEMM), then Tx recurrent
// recurrent steps: ONE persistent wgmma launch for both directions (enc_tc.cu) or, for shapes it does not take,
// per-step launches where forward step s and backward step s share a grouped GEMM + a 2-group gate kernel.
// States are written straight into the concatenated context [Tx, n, 2D] (nats.py:713 needs no copy), the
// masked sum for ctx_mean (nats.py:717) is accumulated by the gate kernel.
// ------------------------------------------------------------------------------------------------
int encoder_forward(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                    const int64_t* x, const float* x_mask, int Tx, int n, const EncBufs& e) {
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, V = d.n_words, C = 2 * D, D3 = 3 * D;
    const long long XB = (long long)Tx * n;
    NATS_TRY(gather_rows(st, params + o.Wemb, x, (int)XB, W, V, 0, e.emb_x));          // nats.py:700-701
    {
        GemmProblem pr[2];
        for (int dir = 0; dir < 2; ++dir) {                                              // nats.py:328-332
            pr[dir] = gemm_problem(e.emb_x, W, params + o.enc[dir].Wcat, D3, e.xproj[dir], D3, (int)XB, D3, W);
            pr[dir].bias = params + o.enc[dir].bcat;
        }
        NATS_TRY(gemm_launch(st, pr, 2, false, false, GEMM_CFG_AUTO));
    }
    NATS_CUDA_OK(memset_async(st, e.ctxsum, 0, (size_t)n * C * sizeof(float)));
    const int S = gemm_pick_split(ctx, n, D3, D, 2);
    const int cfg = gemm_step_cfg(n);
    const long long strideP = 2LL * n * D3;
    if (enc_tc_eligible(ctx, n, D, 0) && e.enc_scratch != nullptr) {
        // the whole recurrence of both directions in ONE persistent weight-stationary wgmma launch (enc_tc.cu)
        EncTcFwdArgs pa;
        memset(&pa, 0, sizeof(pa));
        for (int dir = 0; dir < 2; ++dir) {
            pa.Ucat[dir] = params + o.enc[dir].Ucat; pa.xproj[dir] = e.xproj[dir];
            pa.r[dir] = e.r[dir]; pa.u[dir] = e.u[dir]; pa.c[dir] = e.c[dir]; pa.p[dir] = e.p[dir];
        }
        pa.mask = x_mask; pa.cc = e.cc; pa.ctxsum = e.ctxsum;
        pa.bar = e.enc_counters; pa.bar_ints = e.enc_counter_ints;
        pa.scratch = e.enc_scratch; pa.scratch_floats = e.enc_scratch_floats;
        pa.Tx = Tx; pa.n = n; pa.D = D;
        NATS_TRY(enc_tc_fwd(ctx, st, pa));
    } else {
        // per-step path (shapes the persistent kernel does not take): grouped product of both directions + gate kernel
        for (int s = 0; s < Tx; ++s) {
            const int pf = s, pb = Tx - 1 - s;      // source positions handled by the forward / backward direction
            if (s > 0) {                                                                     // nats.py:337, 345
                GemmProblem q[2];
                q[0] = gemm_problem(e.cc + (long long)(pf - 1) * n * C, C, params + o.enc[0].Ucat, D3, e.part_a, D3, n, D3, D);
                q[1] = gemm_problem(e.cc + (long long)(pb + 1) * n * C + D, C, params + o.enc[1].Ucat, D3,
                                    e.part_a + (long long)n * D3, D3, n, D3, D);
                gemm_set_split(q[0], S, strideP);
                gemm_set_split(q[1], S, strideP);
                NATS_TRY(gemm_launch(st, q, 2, false, false, cfg));
            }
            GateFwd g[2];
            memset(g, 0, sizeof(g));
            for (int dir = 0; dir < 2; ++dir) {
                const int pos = dir == 0 ? pf : pb;
                const int prev = dir == 0 ? pf - 1 : pb + 1;
                g[dir].part = e.part_a + (long long)dir * n * D3;
                g[dir].nsplit = s > 0 ? S : 0;
                g[dir].part_stride = strideP;
                g[dir].xproj = e.xproj[dir] + (long long)pos * n * D3;
                g[dir].h_prev = s > 0 ? e.cc + (long long)prev * n * C + dir * D : nullptr;
                g[dir].ld_hprev = C;
                g[dir].mask = x_mask ? x_mask + (long long)pos * n : nullptr;
                g[dir].h_out = e.cc + (long long)pos * n * C + dir * D;
                g[dir].ld_hout = C;
                if (e.r[dir]) {
                    const long long so = (long long)pos * n * D;
                    g[dir].r = e.r[dir] + so; g[dir].u = e.u[dir] + so; g[dir].c = e.c[dir] + so; g[dir].p = e.p[dir] + so;
                }
                g[dir].ctxsum = e.ctxsum + dir * D;
                g[dir].ld_ctxsum = C;
            }
            NATS_TRY(gru_gates_fwd(st, g, 2, n, D, 0));
        }
    }
    NATS_TRY(mask_lengths(st, x_mask, Tx, n, e.xlen, e.xinv));
    NATS_TRY(scale_rows(st, e.ctxsum, e.xinv, n, C, e.ctx_mean));                        // nats.py:717 / 810
    GemmProblem pi = gemm_problem(e.ctx_mean, C, params + o.ff_state_W, D, e.init_state, D, n, D, C);
    pi.bias = params + o.ff_state_b;
    NATS_TRY(gemm_auto(ctx, st, pi, false, false, e.gemm_scratch, e.gemm_scratch_floats));
    NATS_TRY(tanh_inplace(st, e.init_state, (long long)n * D));                          // nats.py:723-724
    return 0;
}

// ------------------------------------------------------------------------------------------------
// one decoder step (nats.py:498-572): 7 launches
//   GEMM h_.[U|Ux] -> gates(GRU_2) -> grouped GEMM {h1.[U_1|Ux_1], h1.W_att} -> scores -> context(+distraction)
//   -> GEMM ctx.[W_1|Wx_1] -> gates(GRU_1)
// ------------------------------------------------------------------------------------------------
int decoder_step_forward(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                         const DecStep& s) {
    const ParamOff o = param_offsets(d);
    const int D = d.dim, A = d.dim_att, C = 2 * D, D3 = 3 * D, n = s.n;
    const int cfg = gemm_step_cfg(n);
    const int S1 = gemm_pick_split(ctx, n, D3, D);
    const int S2 = gemm_pick_split(ctx, n, D3, C);
    const long long sp3 = (long long)n * D3;
    {   // GRU_2 recurrent product (nats.py:505, 512)
        GemmProblem q = gemm_problem(s.h_prev, D, params + o.dec.Ucat, D3, s.part_b, D3, n, D3, D);
        gemm_set_split(q, S1, sp3);
        NATS_TRY(gemm_launch(st, &q, 1, false, false, cfg));
        GateFwd g;
        memset(&g, 0, sizeof(g));
        g.part = s.part_b; g.nsplit = S1; g.part_stride = sp3;
        g.xproj = s.xproj;
        g.h_prev = s.h_prev; g.ld_hprev = D;
        g.mask = s.ymask;
        g.h_out = s.h1; g.ld_hout = D;
        g.r = s.r1; g.u = s.u1; g.c = s.c1; g.p = s.p1;
        NATS_TRY(gru_gates_fwd(st, &g, 1, n, D, 0));
    }
    {   // products with h1: GRU_1 recurrent part (nats.py:551, 558) and the attention query (nats.py:527)
        GemmProblem q[2];
        q[0] = gemm_problem(s.h1, D, params + o.U1cat, D3, s.part_c, D3, n, D3, D);
        gemm_set_split(q[0], S1, sp3);
        q[1] = gemm_problem(s.h1, D, params + o.W_att, A, s.part_d, A, n, A, D);
        gemm_set_split(q[1], S1, (long long)n * A);
        NATS_TRY(gemm_launch(st, q, 2, false, false, cfg));
    }
    {
        AttFwd a;
        memset(&a, 0, sizeof(a));
        a.pctx = s.pctx; a.pctx_tstride = s.pctx_ts; a.pctx_bstride = s.pctx_bs;
        a.cc = s.cc; a.cc_tstride = s.cc_ts; a.cc_bstride = s.cc_bs;
        a.ps_part = s.part_d; a.ps_nsplit = S1; a.ps_stride = (long long)n * A;
        a.ps_save = s.ps_save;
        a.acc_alpha_in = s.acc_alpha_in; a.acc_ctx_in = s.acc_ctx_in;
        a.xmask = s.xmask; a.ymask = s.ymask;
        a.rows_per_src = s.rows_per_src; a.src_len = s.src_len;
        a.D_wei = params + o.D_wei; a.U_att = params + o.U_att; a.c_att = params + o.c_att;
        a.U_con = params + o.U_con; a.W_con = params + o.W_con;
        a.escore = s.escore;
        a.alpha_out = s.alpha_out; a.acc_alpha_out = s.acc_alpha_out;
        a.craw_out = s.craw_out; a.ctx_out = s.ctx_out; a.acc_ctx_out = s.acc_ctx_out;
        a.Tx = s.Tx; a.n = n; a.A = A; a.C = C;
        NATS_TRY(attention_fwd(ctx, st, a));
    }
    {   // GRU_1 (nats.py:551-565)
        GemmProblem q = gemm_problem(s.ctx_out, C, params + o.W1cat, D3, s.part_a, D3, n, D3, C);
        gemm_set_split(q, S2, sp3);
        NATS_TRY(gemm_launch(st, &q, 1, false, false, cfg));
        GateFwd g;
        memset(&g, 0, sizeof(g));
        g.part = s.part_c; g.nsplit = S1; g.part_stride = sp3;
        g.part2 = s.part_a; g.nsplit2 = S2; g.part2_stride = sp3;
        g.bias = params + o.b1cat;
        g.h_prev = s.h1; g.ld_hprev = D;
        g.mask = s.ymask;
        g.h_out = s.h2; g.ld_hout = D;
        g.r = s.r2; g.u = s.u2; g.c = s.c2; g.p = s.p2;
        NATS_TRY(gru_gates_fwd(st, &g, 1, n, D, 1));
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// training graph, forward (nats.py:658-772)
// ------------------------------------------------------------------------------------------------
int train_encoder_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* x, const float* x_mask, int Tx, int B, const TrainWS& w) {
    EncBufs e;
    memset(&e, 0, sizeof(e));
    e.emb_x = w.emb_x;
    for (int i = 0; i < 2; ++i) {
        e.xproj[i] = w.xproj[i];
        e.r[i] = w.enc_r[i]; e.u[i] = w.enc_u[i]; e.c[i] = w.enc_c[i]; e.p[i] = w.enc_p[i];
    }
    e.cc = w.cc; e.ctxsum = w.ctxsum; e.xlen = w.xlen; e.xinv = w.xinv; e.ctx_mean = w.ctx_mean;
    e.init_state = w.init_state; e.part_a = w.part_a;
    e.gemm_scratch = w.gemm_scratch; e.gemm_scratch_floats = w.gemm_scratch_floats;
    e.enc_scratch = w.enc_scratch; e.enc_scratch_floats = w.enc_scratch_floats;
    e.enc_counters = w.enc_counters; e.enc_counter_ints = w.enc_counter_ints;
    return encoder_forward(ctx, st, d, params, x, x_mask, Tx, B, e);
}

int train_decoder_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                      const TrainWS& w) {
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, A = d.dim_att, V = d.n_words, C = 2 * D, D3 = 3 * D;
    const long long XB = (long long)Tx * B, YB = (long long)Ty * B;
    // shifted target embedding (nats.py:730-734) and its projections (nats.py:487-491)
    NATS_TRY(gather_rows(st, params + o.Wemb, y, (int)YB, W, V, B, w.embs));
    {
        GemmProblem p = gemm_problem(w.embs, W, params + o.dec.Wcat, D3, w.xproj_y, D3, (int)YB, D3, W);
        p.bias = params + o.dec.bcat;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    }
    {   // projected context (nats.py:493-494)
        GemmProblem p = gemm_problem(w.cc, C, params + o.Wc_att, A, w.pctx, A, (int)XB, A, C);
        p.bias = params + o.b_att;
        NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    }
    NATS_CUDA_OK(memset_async(st, w.d_accalpha, 0, (size_t)B * Tx * sizeof(float)));   // nats.py:599-603
    NATS_CUDA_OK(memset_async(st, w.d_accctx, 0, (size_t)B * C * sizeof(float)));
    for (int t = 0; t < Ty; ++t) {
        const long long rD = (long long)t * B * D, rC = (long long)t * B * C, rT = (long long)t * B * Tx;
        DecStep s;
        memset(&s, 0, sizeof(s));
        s.n = B; s.Tx = Tx;
        s.h_prev = t == 0 ? w.init_state : w.d_h2 + rD - (long long)B * D;
        s.xproj = w.xproj_y + (long long)t * B * D3;
        s.ymask = y_mask + (long long)t * B;
        s.xmask = x_mask;
        s.pctx = w.pctx; s.pctx_ts = (long long)B * A; s.pctx_bs = A;
        s.cc = w.cc; s.cc_ts = (long long)B * C; s.cc_bs = C;
        s.acc_alpha_in = w.d_accalpha + rT; s.acc_alpha_out = w.d_accalpha + rT + (long long)B * Tx;
        s.acc_ctx_in = w.d_accctx + rC; s.acc_ctx_out = w.d_accctx + rC + (long long)B * C;
        s.h1 = w.d_h1 + rD; s.r1 = w.d_r1 + rD; s.u1 = w.d_u1 + rD; s.c1 = w.d_c1 + rD; s.p1 = w.d_p1 + rD;
        s.ps_save = w.d_ps + (long long)t * B * A;
        s.escore = w.escore;
        s.alpha_out = w.d_alpha + rT;
        s.craw_out = w.d_craw + rC; s.ctx_out = w.d_ctx + rC;
        s.r2 = w.d_r2 + rD; s.u2 = w.d_u2 + rD; s.c2 = w.d_c2 + rD; s.p2 = w.d_p2 + rD; s.h2 = w.d_h2 + rD;
        s.part_a = w.part_a; s.part_b = w.part_b; s.part_c = w.part_c; s.part_d = w.part_d;
        NATS_TRY(decoder_step_forward(ctx, st, d, params, s));
    }
    return 0;
}

int train_readout_fwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* y_mask, int Ty, int B, const TrainWS& w, float* cost) {
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, V = d.n_words, C = 2 * D;
    const int YB = Ty * B;
    // pre = h.Wl + bl + emb.Wp + bp + ctx.Wc + bc  (nats.py:753-758), L = tanh(pre) (nats.py:759)
    GemmProblem p = gemm_problem(w.d_h2, D, params + o.lstm_W, W, w.L, W, YB, W, D);
    p.bias = params + o.lstm_b;
    NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    p = gemm_problem(w.embs, W, params + o.prev_W, W, w.L, W, YB, W, W);
    p.bias = params + o.prev_b; p.accumulate = 1;
    NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    p = gemm_problem(w.d_ctx, C, params + o.ctxr_W, W, w.L, W, YB, W, C);
    p.bias = params + o.ctxr_b; p.accumulate = 1;
    NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    NATS_TRY(tanh_inplace(st, w.L, (long long)YB * W));
    // logits (nats.py:760-761), log-softmax + NLL (nats.py:763-770)
    p = gemm_problem(w.L, W, params + o.logit_W, V, w.logits, V, YB, V, W);
    p.bias = params + o.logit_b;
    NATS_TRY(gemm_auto(ctx, st, p, false, false, w.gemm_scratch, w.gemm_scratch_floats));
    NATS_TRY(nll_rows(st, w.logits, YB, V, y, y_mask, w.lse, w.rowcost));
    NATS_TRY(cost_reduce(st, w.rowcost, Ty, B, cost, 1.f, nullptr));
    return 0;
}

}  // namespace nats
