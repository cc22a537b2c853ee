// model_bwd.cu -- hand-written reverse mode of the training graph (what tensor.grad, nats.py:1340, derives
// through the two encoder scans and the decoder scan).  Mirrors oracle/nats_oracle.py:model_bwd.
//
// Strategy: inside the time loops only the strictly sequential work is done (gate derivatives, the products
// that carry d h_{t-1}, the attention backward); every parameter gradient that is a sum over time is deferred
// to ONE large product after the loop ([rows = T*B] deep), using the per-step gate derivatives saved in
// dG* buffers.  All reductions have a fixed order (split-K slabs, per-sample partials): no float atomics
// except the embedding scatter-add.
#include "model.cuh"

namespace nats {

namespace {
inline int ga(const nats_ctx* ctx, cudaStream_t st, const TrainWS& w, GemmProblem p, bool ta, bool tb) {
    return gemm_auto(ctx, st, p, ta, tb, w.gemm_scratch, w.gemm_scratch_floats);
}
}  // namespace

// ------------------------------------------------------------------ readout (nats.py:753-770)
int train_readout_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* y_mask, int Ty, int B, const TrainWS& w, float scale,
                      float* G) {
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, V = d.n_words, C = 2 * D;
    const int YB = Ty * B;
    NATS_TRY(dlogits_inplace(st, w.logits, YB, V, y, y_mask, w.lse, scale));
    // ff_logit: dW = L^T dlogits, db = colsum, dL = dlogits W^T
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.L, W, w.logits, V, G + o.logit_W, V, W, V, YB), true, false));
    NATS_TRY(colsum(st, w.logits, YB, V, V, G + o.logit_b, 0, w.red_scratch));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.logits, V, params + o.logit_W, V, w.dpre, W, YB, W, V), false, true));
    NATS_TRY(dtanh(st, w.dpre, w.L, w.dpre, (long long)YB * W));
    // the three input transforms
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.d_h2, D, w.dpre, W, G + o.lstm_W, W, D, W, YB), true, false));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.embs, W, w.dpre, W, G + o.prev_W, W, W, W, YB), true, false));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.d_ctx, C, w.dpre, W, G + o.ctxr_W, W, C, W, YB), true, false));
    NATS_TRY(colsum3(st, w.dpre, YB, W, W, G + o.lstm_b, G + o.prev_b, G + o.ctxr_b, 0, w.red_scratch));   // one sum, three biases
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.dpre, W, params + o.lstm_W, W, w.dh2_ro, D, YB, D, W), false, true));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.dpre, W, params + o.ctxr_W, W, w.dctx_ro, C, YB, C, W), false, true));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.dpre, W, params + o.prev_W, W, w.dembs, W, YB, W, W), false, true));
    return 0;
}

// ------------------------------------------------------------------ decoder scan (nats.py:454-609)
int train_decoder_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* y, const float* x_mask, const float* y_mask, int Tx, int Ty, int B,
                      const TrainWS& w, float* G) {
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, A = d.dim_att, V = d.n_words, C = 2 * D, D3 = 3 * D;
    const long long XB = (long long)Tx * B, YB = (long long)Ty * B;
    const int cfg = gemm_step_cfg(B);
    const int SA = gemm_pick_split(ctx, B, D, D3);    // d h1   <- dG1 . U1cat^T      (slabs in part_b)
    const int SB = gemm_pick_split(ctx, B, C, D3);    // d ctx  <- dG1x . W1cat^T     (slabs in part_a)
    const int S4 = gemm_pick_split(ctx, B, D, D3);    // d h_   <- dG2 . Ucat^T       (slabs in part_c)
    const long long spD = (long long)B * D, spC = (long long)B * C;

    NATS_CUDA_OK(memset_async(st, w.dpctx, 0, (size_t)XB * A * sizeof(float)));
    NATS_CUDA_OK(memset_async(st, w.dacc_alpha, 0, (size_t)B * Tx * sizeof(float)));
    NATS_CUDA_OK(memset_async(st, w.dacc_ctx, 0, (size_t)2 * B * C * sizeof(float)));
    NATS_CUDA_OK(memset_async(st, w.gatt_part, 0, (size_t)B * (2 * A + 1) * sizeof(float)));

    for (int t = Ty - 1; t >= 0; --t) {
        const long long rD = (long long)t * B * D, rC = (long long)t * B * C, rT = (long long)t * B * Tx;
        const long long r3 = (long long)t * B * D3, rA = (long long)t * B * A;
        const float* ym = y_mask + (long long)t * B;
        const int pp = t & 1;
        {   // GRU_1 backward (nats.py:551-565)
            GateBwd g;
            memset(&g, 0, sizeof(g));
            g.dh_a = w.dh2_ro + rD; g.ld_a = D;
            if (t < Ty - 1) {
                g.dh_b = w.dh_elem; g.ld_b = D;
                g.part = w.part_c; g.nsplit = S4; g.part_stride = spD; g.part_ld = D;
            }
            g.r = w.d_r2 + rD; g.u = w.d_u2 + rD; g.c = w.d_c2 + rD; g.p = w.d_p2 + rD;
            g.h_prev = w.d_h1 + rD; g.ld_hprev = D;
            g.mask = ym;
            g.dG = w.dG1 + r3; g.dGx = w.dG1x + r3; g.dh_elem = w.dh1_elem;
            NATS_TRY(gru_gates_bwd(st, &g, 1, B, D));
        }
        {   // d h1 and d ctx through the GRU_1 products
            GemmProblem q[2];
            q[0] = gemm_problem(w.dG1 + r3, D3, params + o.U1cat, D3, w.part_b, D, B, D, D3);
            gemm_set_split(q[0], SA, spD);
            q[1] = gemm_problem(w.dG1x + r3, D3, params + o.W1cat, D3, w.part_a, C, B, C, D3);
            gemm_set_split(q[1], SB, spC);
            NATS_TRY(gemm_launch(st, q, 2, false, true, cfg));
        }
        {   // distraction + attention backward (nats.py:527-546, 569-570)
            AttBwd a;
            memset(&a, 0, sizeof(a));
            a.pctx = w.pctx; a.cc = w.cc;
            a.dctx_a = w.dctx_ro + rC;
            a.dctx_part = w.part_a; a.dctx_nsplit = SB; a.dctx_stride = spC;
            a.dacc_ctx_in = w.dacc_ctx + (long long)pp * B * C;
            a.dacc_ctx_out = w.dacc_ctx + (long long)(pp ^ 1) * B * C;
            a.dacc_alpha = w.dacc_alpha;
            a.ymask = ym;
            a.ctx = w.d_ctx + rC; a.craw = w.d_craw + rC; a.acc_ctx = w.d_accctx + rC;
            a.alpha = w.d_alpha + rT; a.acc_alpha = w.d_accalpha + rT;
            a.ps = w.d_ps + rA;
            a.D_wei = params + o.D_wei; a.U_att = params + o.U_att; a.U_con = params + o.U_con; a.W_con = params + o.W_con;
            a.dq = w.dq + rC; a.dcraw = w.dcraw + rC;
            a.dalpha = w.dalpha;
            a.dps = w.dps + rA;
            a.dpctx = w.dpctx;
            a.gatt_part = w.gatt_part;
            a.dot_part = w.att_dot_part; a.soft_part = w.att_soft_part;
            a.Tx = Tx; a.B = B; a.A = A; a.C = C;
            NATS_TRY(attention_bwd(ctx, st, a));
        }
        {   // d h1 += d ps . W_att^T  (nats.py:527)
            GemmProblem q = gemm_problem(w.dps + rA, A, params + o.W_att, A, w.part_d, D, B, D, A);
            NATS_TRY(gemm_launch(st, &q, 1, false, true, cfg));
        }
        {   // GRU_2 backward (nats.py:505-518)
            GateBwd g;
            memset(&g, 0, sizeof(g));
            g.dh_a = w.dh1_elem; g.ld_a = D;
            g.part = w.part_b; g.nsplit = SA; g.part_stride = spD; g.part_ld = D;
            g.part2 = w.part_d; g.nsplit2 = 1; g.part2_stride = spD; g.part2_ld = D;
            g.r = w.d_r1 + rD; g.u = w.d_u1 + rD; g.c = w.d_c1 + rD; g.p = w.d_p1 + rD;
            g.h_prev = t > 0 ? w.d_h2 + rD - spD : w.init_state; g.ld_hprev = D;
            g.mask = ym;
            g.dG = w.dG2 + r3; g.dGx = w.dG2x + r3; g.dh_elem = w.dh_elem;
            NATS_TRY(gru_gates_bwd(st, &g, 1, B, D));
        }
        {   // d h_{t-1} through the GRU_2 recurrent product
            GemmProblem q = gemm_problem(w.dG2 + r3, D3, params + o.dec.Ucat, D3, w.part_c, D, B, D, D3);
            gemm_set_split(q, S4, spD);
            NATS_TRY(gemm_launch(st, &q, 1, false, true, cfg));
        }
    }
    // d init_state -> pre-activation of ff_state (nats.py:723-724)
    NATS_TRY(sum_parts_dtanh(st, w.dh_elem, w.part_c, S4, spD, w.init_state, w.dinit, B, D));

    // ---- parameter gradients as deep products over all decoder steps
    {   // [U | Ux]: h_{t-1}^T dG2 ; the t = 0 row block pairs with init_state
        NATS_TRY(ga(ctx, st, w, gemm_problem(w.init_state, D, w.dG2, D3, G + o.dec.Ucat, D3, D, D3, B), true, false));
        if (Ty > 1) {
            GemmProblem p = gemm_problem(w.d_h2, D, w.dG2 + (long long)B * D3, D3, G + o.dec.Ucat, D3, D, D3, (Ty - 1) * B);
            p.accumulate = 1;
            NATS_TRY(ga(ctx, st, w, p, true, false));
        }
    }
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.embs, W, w.dG2x, D3, G + o.dec.Wcat, D3, W, D3, (int)YB), true, false));
    NATS_TRY(colsum(st, w.dG2x, YB, D3, D3, G + o.dec.bcat, 0, w.red_scratch));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.d_h1, D, w.dG1, D3, G + o.U1cat, D3, D, D3, (int)YB), true, false));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.d_ctx, C, w.dG1x, D3, G + o.W1cat, D3, C, D3, (int)YB), true, false));
    NATS_TRY(colsum(st, w.dG1, YB, D3, D3, G + o.b1cat, 0, w.red_scratch));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.d_h1, D, w.dps, A, G + o.W_att, A, D, A, (int)YB), true, false));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.cc, C, w.dpctx, A, G + o.Wc_att, A, C, A, (int)XB), true, false));
    NATS_TRY(colsum(st, w.dpctx, XB, A, A, G + o.b_att, 0, w.red_scratch));
    NATS_TRY(colsum_prod(st, w.dq, w.d_craw, YB, C, C, G + o.U_con, 0, w.red_scratch));
    NATS_TRY(colsum_prod(st, w.dq, w.d_accctx, YB, C, C, G + o.W_con, 0, w.red_scratch));
    NATS_TRY(colsum(st, w.gatt_part, B, A, 2 * A + 1, G + o.U_att, 0, w.red_scratch));
    NATS_TRY(colsum(st, w.gatt_part + A, B, A, 2 * A + 1, G + o.D_wei, 0, w.red_scratch));
    NATS_TRY(colsum(st, w.gatt_part + 2 * A, B, 1, 2 * A + 1, G + o.c_att, 0, w.red_scratch));

    // ---- d context: through pctx (nats.py:493) and through the weighted sums (nats.py:541)
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.dpctx, A, params + o.Wc_att, A, w.dcc, C, (int)XB, C, A), false, true));
    {   // dcc[:, b, :] += alpha_b^T [Tx,Ty] . dcraw_b [Ty,C]   -- one batched product instead of Ty rank-1 updates
        GemmProblem p = gemm_problem(w.d_alpha, B * Tx, w.dcraw, B * C, w.dcc, B * C, Tx, C, Ty);
        p.batch = B; p.strideA = Tx; p.strideB = C; p.strideC = C; p.accumulate = 1;
        NATS_TRY(gemm_launch(st, &p, 1, true, false, GEMM_CFG_AUTO));
    }
    // ---- d target embedding (nats.py:487-491, 730-734)
    {
        GemmProblem p = gemm_problem(w.dG2x, D3, params + o.dec.Wcat, D3, w.dembs, W, (int)YB, W, D3);
        p.accumulate = 1;
        NATS_TRY(ga(ctx, st, w, p, false, true));
        NATS_TRY(scatter_add_rows(st, G + o.Wemb, y, (int)YB, W, V, B, w.dembs));
    }
    // ---- ff_state (nats.py:717-724)
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.ctx_mean, C, w.dinit, D, G + o.ff_state_W, D, C, D, B), true, false));
    NATS_TRY(colsum(st, w.dinit, B, D, D, G + o.ff_state_b, 0, w.red_scratch));
    NATS_TRY(ga(ctx, st, w, gemm_problem(w.dinit, D, params + o.ff_state_W, D, w.dmean, C, B, C, D), false, true));
    return 0;
}

// ------------------------------------------------------------------ encoder (nats.py:305-374, 700-713)
int train_encoder_bwd(const nats_ctx* ctx, cudaStream_t st, const nats_dims_t& d, const float* params,
                      const int64_t* x, const float* x_mask, const int64_t* y, int Tx, int Ty, int B,
                      const TrainWS& w, float* G) {
    (void)y; (void)Ty;
    const ParamOff o = param_offsets(d);
    const int W = d.dim_word, D = d.dim, V = d.n_words, C = 2 * D, D3 = 3 * D;
    const long long XB = (long long)Tx * B;
    const int cfg = gemm_step_cfg(B);
    const int S = gemm_pick_split(ctx, B, D, D3, 2);
    const long long strideP = 2LL * B * D;
    const bool persistent = enc_tc_eligible(ctx, B, D, 1);
    if (persistent) {      // the whole reverse recurrence of both directions in ONE persistent wgmma launch (enc_tc.cu)
        EncTcBwdArgs pa;
        memset(&pa, 0, sizeof(pa));
        for (int dir = 0; dir < 2; ++dir) {
            pa.Ucat[dir] = params + o.enc[dir].Ucat;
            pa.r[dir] = w.enc_r[dir]; pa.u[dir] = w.enc_u[dir]; pa.c[dir] = w.enc_c[dir]; pa.p[dir] = w.enc_p[dir];
            pa.dG[dir] = w.dGe[dir]; pa.dGx[dir] = w.dGex[dir];
        }
        pa.dcc = w.dcc; pa.mean_grad = w.dmean; pa.coef = w.xinv; pa.mask = x_mask; pa.cc = w.cc;
        pa.bar = w.enc_counters; pa.bar_ints = w.enc_counter_ints;
        pa.scratch = w.enc_scratch; pa.scratch_floats = w.enc_scratch_floats;
        pa.Tx = Tx; pa.n = B; pa.D = D;
        NATS_TRY(enc_tc_bwd(ctx, st, pa));
    }
    for (int s = Tx - 1; s >= 0 && !persistent; --s) {
        const int pf = s, pb = Tx - 1 - s;
        GateBwd g[2];
        memset(g, 0, sizeof(g));
        for (int dir = 0; dir < 2; ++dir) {
            const int pos = dir == 0 ? pf : pb;
            const int prev = dir == 0 ? pf - 1 : pb + 1;
            const long long so = (long long)pos * B * D;
            g[dir].dh_a = w.dcc + (long long)pos * B * C + dir * D; g[dir].ld_a = C;
            if (s < Tx - 1) {
                g[dir].dh_b = w.dh_elem + (long long)dir * B * D; g[dir].ld_b = D;
                g[dir].part = w.part_a + (long long)dir * B * D; g[dir].nsplit = S;
                g[dir].part_stride = strideP; g[dir].part_ld = D;
            }
            g[dir].mean_grad = w.dmean + dir * D; g[dir].ld_mean = C; g[dir].coef = w.xinv;   // nats.py:717
            g[dir].r = w.enc_r[dir] + so; g[dir].u = w.enc_u[dir] + so; g[dir].c = w.enc_c[dir] + so;
            g[dir].p = w.enc_p[dir] + so;
            g[dir].h_prev = s > 0 ? w.cc + (long long)prev * B * C + dir * D : nullptr; g[dir].ld_hprev = C;
            g[dir].mask = x_mask + (long long)pos * B;
            g[dir].dG = w.dGe[dir] + (long long)pos * B * D3;
            g[dir].dGx = w.dGex[dir] + (long long)pos * B * D3;
            g[dir].dh_elem = w.dh_elem + (long long)dir * B * D;
        }
        NATS_TRY(gru_gates_bwd(st, g, 2, B, D));
        if (s > 0) {
            GemmProblem q[2];
            for (int dir = 0; dir < 2; ++dir) {
                const int pos = dir == 0 ? pf : pb;
                q[dir] = gemm_problem(w.dGe[dir] + (long long)pos * B * D3, D3, params + o.enc[dir].Ucat, D3,
                                      w.part_a + (long long)dir * B * D, D, B, D, D3);
                gemm_set_split(q[dir], S, strideP);
            }
            NATS_TRY(gemm_launch(st, q, 2, false, true, cfg));
        }
    }
    if (Tx > 1) {
        const int K = (Tx - 1) * B;
        // forward direction: h_{t-1} = cc[t-1, :, 0:D] pairs with dG[t]; backward: cc[p+1, :, D:2D] with dG[p]
        NATS_TRY(ga(ctx, st, w, gemm_problem(w.cc, C, w.dGe[0] + (long long)B * D3, D3, G + o.enc[0].Ucat, D3, D, D3, K),
                    true, false));
        NATS_TRY(ga(ctx, st, w, gemm_problem(w.cc + (long long)B * C + D, C, w.dGe[1], D3, G + o.enc[1].Ucat, D3, D, D3, K),
                    true, false));
    }
    for (int dir = 0; dir < 2; ++dir) {
        NATS_TRY(ga(ctx, st, w, gemm_problem(w.emb_x, W, w.dGex[dir], D3, G + o.enc[dir].Wcat, D3, W, D3, (int)XB),
                    true, false));
        NATS_TRY(colsum(st, w.dGex[dir], XB, D3, D3, G + o.enc[dir].bcat, 0, w.red_scratch));
        GemmProblem p = gemm_problem(w.dGex[dir], D3, params + o.enc[dir].Wcat, D3, w.demb_x, W, (int)XB, W, D3);
        p.accumulate = dir;
        NATS_TRY(ga(ctx, st, w, p, false, true));
    }
    NATS_TRY(scatter_add_rows(st, G + o.Wemb, x, (int)XB, W, V, 0, w.demb_x));      // both source gathers (nats.py:700, 706)
    return 0;
}

}  // namespace nats
