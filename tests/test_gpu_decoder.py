"""The decoder of the training step -- the conditional-GRU scan (7 launches per step, model_fwd.cu), the attention
forward and backward kernels (ops_att.cu), the readout and NLL (ops_readout.cu) and the decoder's deep weight-gradient
products (model_bwd.cu) -- against float64, case by case across the shapes where their plans change.

Each case drives the C ABI directly on its own workspace:
  * forward:  nats_train_fwd; the views `ctx`, `init_state`, `pctx`, `dec_h`, `dec_ctx`, `dec_alpha`, the cost, and a
    copy of `logits` (the backward overwrites it with d logits);
  * backward: nats_train_bwd_begin with scale 1/B; the gradient slice from nats_grad_split on (final at this point), the
    `Wemb` rows (only the target-side scatter so far) and the views `logits` (now d logits), `dcc` and `dmean`;
  * path:     the profiler's launch counts of the 3xTF32, FFMA and attention classes, against the recorded ones, so a
    plan change cannot quietly move a case to another kernel.

The reference is the float64 oracle fed the device's own encoder output (`ctx`, `init_state`), so the encoder's error is
not counted against the decoder: O.gru_cond_layer_fwd, the readout lines of O.model_fwd, the readout part of
O.model_bwd, O.gru_cond_layer_bwd and the ff_state part (_reference below).

Errors come in families with one bound each (FAMILIES).  test_bounds_reject_a_degraded_decoder (no GPU) runs the same
reference with weights truncated to their tf32 part, the way a kernel computes that drops a weight's lo term, and shows
that each bound is at most a quarter of the error of such a kernel:
  * per-step weights truncated (decoder_U / Ux / U_1 / Ux_1 / W_1 / Wx_1 / W_att): fails 'states' and 'products';
  * readout weights truncated (ff_logit_W, ff_logit_lstm_W, ff_logit_ctx_W): fails 'readout' and 'logits'."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import nats_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# What each case reaches (H100, 132 SMs).  Every case has ragged masks: column 0 at full Tx and Ty, column 1 with a
# source of length 1 and a target of about half the length, the rest random.
CASES = [
    # a one-step scan and a one-position softmax (alpha = 1, so d e = 0 exactly); W_att's products on FFMA (forward
    # N = A = 8 < 64, backward K = A = 8 < 32), which takes the grouped forward h1 . U_1cat product along
    dict(B=1, D=96, W=16, A=8, V=64, Tx=1, Ty=1),
    # Tx not a multiple of 16 or 32; odd V: the NLL and d logits row tails
    dict(B=5, D=100, W=32, A=100, V=1001, Tx=23, Ty=7),
    # C = 202, C % 4 != 0: att_context_kernel<0>, the scalar d alpha loop, the software-loader tc_gemm (no TMA)
    dict(B=4, D=101, W=20, A=40, V=300, Tx=37, Ty=9),
    # A = 256 (kMaxAk of the attention backward); the context kernel's tile ring wraps (5 blocks of 16 rows, 4 stages);
    # a batch of 33: the skinny per-step products' N tile is 64
    dict(B=33, D=256, W=32, A=256, V=500, Tx=70, Ty=12),
    # BASELINE config 2
    dict(B=64, D=500, W=100, A=100, V=4000, Tx=120, Ty=20),
    # batch 65-127: the per-step products leave the skinny kernel for tma_gemm_kernel_ws, weights on the 128-row side
    dict(B=80, D=256, W=32, A=64, V=500, Tx=40, Ty=10),
    # batch >= 128: the per-step products keep the batch rows on the 128-row side (not swapped)
    dict(B=128, D=256, W=32, A=100, V=500, Tx=24, Ty=10),
    # Ty >= 32: the batched dcc += alpha^T . dcraw product (K = Ty) on the tensor cores, roles swapped (Tx < 128)
    dict(B=6, D=200, W=32, A=48, V=500, Tx=40, Ty=35),
    # the same product with Tx = 136 >= 128: not swapped
    dict(B=3, D=200, W=32, A=48, V=500, Tx=136, Ty=35),
    # the config-3 decoder (D = 1000, V = 30000, Tx = 400, Ty = 30)
    dict(B=4, D=1000, W=100, A=100, V=30000, Tx=400, Ty=30),
]
for _c in CASES:
    _c['id'] = 'b%d_d%d_a%d_v%d_t%dx%d' % (_c['B'], _c['D'], _c['A'], _c['V'], _c['Tx'], _c['Ty'])
    _c['seed'] = 7919 * _c['B'] + 31 * _c['D'] + 7 * _c['Tx'] + _c['Ty']

READOUT = ('ff_logit_lstm_W', 'ff_logit_lstm_b', 'ff_logit_prev_W', 'ff_logit_prev_b', 'ff_logit_ctx_W',
           'ff_logit_ctx_b')
PRODUCTS = ('decoder_U', 'decoder_Ux', 'decoder_W', 'decoder_Wx', 'decoder_U_1', 'decoder_Ux_1', 'decoder_W_1',
            'decoder_Wx_1', 'ff_state_W')
ELEMENTWISE = ('decoder_b', 'decoder_bx', 'decoder_b_1', 'decoder_bx_1', 'decoder_U_con', 'decoder_W_con',
               'ff_state_b', 'ff_logit_b')
# gradients whose terms nearly cancel: every one sums the attention's d e (or d zp = d e . U_att . (1 - z^2)) over the
# source positions, and d e sums to exactly 0 over them (softmax), so whatever does not vary along the source cancels
CANCEL = ('decoder_b_att', 'decoder_W_att', 'decoder_c_att', 'decoder_U_att', 'decoder_D_wei', 'decoder_Wc_att')
STATE_VIEWS = ('dec_h', 'pctx', 'dec_ctx', 'dec_alpha')
# family -> its members.  'states' and 'attention': max abs error; 'kernels': the readout kernels on the device's own
# input (_kernel_errors); 'cancel': max_i |g_i - g*_i| / S_i (_reference); the rest ||g - g*|| / ||g*|| per tensor.
#  * 'states' is dec_h alone: the attention outputs hardly move when the per-step weights lose their lo term (W_att
#    feeds the scores only through the small query term), so they form 'attention', which no degradation must fail;
#  * 'logits' holds the logits and the ff_logit_W gradient, which a truncated readout moves only through L (2.3e-5),
#    too little for the bound of the other readout gradients;
#  * 'elementwise' holds the biases, the per-channel scales and ff_logit_b (a column sum of d logits).
FAMILIES = {'states': ('dec_h',), 'attention': ('pctx', 'dec_ctx', 'dec_alpha'), 'kernels': ('cost', 'dlogits', 'colsum'),
            'logits': ('logits', 'ff_logit_W'), 'readout': READOUT, 'products': PRODUCTS, 'elementwise': ELEMENTWISE,
            'inputs': ('Wemb', 'dcc', 'dmean'), 'cancel': CANCEL}
STEP_WEIGHTS = ('decoder_U', 'decoder_Ux', 'decoder_U_1', 'decoder_Ux_1', 'decoder_W_1', 'decoder_Wx_1', 'decoder_W_att')
READOUT_WEIGHTS = ('ff_logit_W', 'ff_logit_lstm_W', 'ff_logit_ctx_W')
# which families each degradation must fail
MUST_FAIL = {'step': ('states', 'products'), 'readout': ('readout', 'logits')}

# Measured on an H100 80GB HBM3 at a 700 W power limit: per case, each family's worst error (FAMILIES order).  NATS_TS=0
# gave the same bits as the default.  Before the near-cancelling tensors had their own bound, U_att, D_wei and Wc_att
# measured up to 2.1e-4, 2.0e-4 and 8.3e-5 as ||g - g*|| / ||g*||; scaled by their terms they sit at 3.7e-7 at most.
#                                          states   attention kernels  logits   readout  products elemwise inputs   cancel
MEASURED_COLUMNS = tuple(FAMILIES)
MEASURED = {
    'b1_d96_a8_v64_t1x1':                    (1.9e-8, 3.5e-9, 1.6e-8, 1.3e-7, 2.9e-7, 2.9e-7, 2.8e-7, 2.3e-7, 0.0),
    'b5_d100_a100_v1001_t23x7':              (2.4e-8, 3.6e-8, 6.3e-8, 1.6e-7, 2.6e-7, 5.9e-7, 3.8e-7, 3.4e-7, 3.7e-7),
    'b4_d101_a40_v300_t37x9':                (2.7e-8, 2.0e-8, 5.5e-8, 9.9e-8, 3.0e-7, 3.5e-7, 2.6e-7, 3.5e-7, 2.7e-7),
    'b33_d256_a256_v500_t70x12':             (3.3e-8, 5.6e-8, 1.4e-7, 4.6e-7, 5.1e-7, 1.1e-6, 7.3e-7, 8.0e-7, 1.8e-7),
    'b64_d500_a100_v4000_t120x20':           (4.7e-8, 9.8e-8, 1.4e-7, 4.9e-7, 1.3e-6, 2.2e-6, 1.4e-6, 1.4e-6, 3.7e-7),
    'b80_d256_a64_v500_t40x10':              (5.8e-8, 4.3e-8, 1.0e-7, 4.1e-7, 5.9e-7, 1.3e-6, 9.1e-7, 1.2e-6, 1.7e-7),
    'b128_d256_a100_v500_t24x10':            (5.2e-8, 7.1e-8, 1.2e-7, 3.8e-7, 6.1e-7, 1.4e-6, 1.0e-6, 1.3e-6, 1.8e-7),
    'b6_d200_a48_v500_t40x35':               (4.2e-8, 1.7e-8, 1.2e-7, 4.3e-7, 5.3e-7, 1.1e-6, 6.9e-7, 7.6e-7, 1.5e-7),
    'b3_d200_a48_v500_t136x35':              (3.3e-8, 2.1e-8, 9.6e-8, 3.8e-7, 4.8e-7, 1.0e-6, 7.9e-7, 1.0e-6, 1.2e-7),
    'b4_d1000_a100_v30000_t400x30':          (6.1e-8, 1.2e-7, 9.3e-8, 5.0e-7, 2.3e-6, 2.7e-6, 2.4e-6, 2.1e-6, 4.8e-7),
    'b33_d256_a256_v500_t70x12 NATS_TS=0':   (3.3e-8, 5.6e-8, 1.4e-7, 4.6e-7, 5.1e-7, 1.1e-6, 7.3e-7, 8.0e-7, 1.8e-7),
    'b64_d500_a100_v4000_t120x20 NATS_TS=0': (4.7e-8, 9.8e-8, 1.4e-7, 4.9e-7, 1.3e-6, 2.2e-6, 1.4e-6, 1.4e-6, 3.7e-7),
}

# About four times the worst measured value of each family.  A build whose skinny kernel dropped the weight lo term
# (A_lo . B_hi) failed every case (same card): dec_h off by up to 2.4e-5, the products by up to 3.3e-4.
BOUND = {'states': 2.5e-7, 'attention': 5e-7, 'kernels': 6e-7, 'logits': 2e-6, 'readout': 1e-5, 'products': 1e-5,
         'elementwise': 1e-5, 'inputs': 1e-5, 'cancel': 2e-6}
ALPHA_SUM = 6e-7        # |sum_t alpha - 1| of every alpha row (measured at most 1.6e-7)

# Launch counts per case over nats_train_fwd + nats_train_bwd_begin (classes with none left out).  What they show:
#  * b1: the FFMA gemm_smallm_nt launch of d h1 += d ps . W_att^T (K = A = 8), next to six skinny 3xTF32 products;
#  * b64 against b80 / b128: the per-step products move from tc_gemm_3xtf32_skinny (122 launches at 20 steps) to
#    tc_gemm_3xtf32 (112 / 99 launches at 10 steps);
#  * b6 against b3 (Ty = 35): one product, the batched alpha^T . dcraw, moves from the skinny kernel (Tx = 40,
#    swapped) to tc_gemm_3xtf32 (Tx = 136); the Ty < 32 cases run it on FFMA (gemm_*_tn);
#  * each att_* class launches once per decoder step.
LAUNCHES = {
    'b1_d96_a8_v64_t1x1': {'gemm_mid_tn': 8, 'gemm_smallm_nn': 8, 'gemm_smallm_nt': 7, 'gemm_smallm_tn': 4,
                           'att_scores': 1, 'att_context': 1, 'att_bwd_ctx': 1, 'att_bwd_dalpha': 1,
                           'att_bwd_softmax': 1, 'tc_gemm_3xtf32_skinny': 6},
    'b5_d100_a100_v1001_t23x7': {'gemm_mid_nn': 3, 'gemm_mid_nt': 3, 'gemm_mid_tn': 3, 'gemm_smallm_tn': 2,
                                 'att_scores': 7, 'att_context': 7, 'att_bwd_ctx': 7, 'att_bwd_dalpha': 7,
                                 'att_bwd_softmax': 7, 'tc_gemm_3xtf32': 7, 'tc_gemm_3xtf32_skinny': 52},
    'b4_d101_a40_v300_t37x9': {'gemm_mid_nn': 6, 'gemm_mid_nt': 5, 'gemm_mid_tn': 3, 'gemm_smallm_nn': 9,
                               'gemm_smallm_tn': 1, 'att_scores': 9, 'att_context': 9, 'att_bwd_ctx': 9,
                               'att_bwd_dalpha': 9, 'att_bwd_softmax': 9, 'tc_gemm_3xtf32': 4,
                               'tc_gemm_3xtf32_skinny': 90},
    'b33_d256_a256_v500_t70x12': {'gemm_mid_tn': 1, 'gemm_smallm_tn': 1, 'att_scores': 12, 'att_context': 12,
                                  'att_bwd_ctx': 12, 'att_bwd_dalpha': 12, 'att_bwd_softmax': 12,
                                  'tc_gemm_3xtf32': 14, 'tc_gemm_3xtf32_skinny': 84},
    'b64_d500_a100_v4000_t120x20': {'gemm_mid_tn': 1, 'att_scores': 20, 'att_context': 20, 'att_bwd_ctx': 20,
                                    'att_bwd_dalpha': 20, 'att_bwd_softmax': 20, 'tc_gemm_3xtf32': 25,
                                    'tc_gemm_3xtf32_skinny': 122},
    'b80_d256_a64_v500_t40x10': {'gemm_mid_tn': 1, 'gemm_smallm_tn': 1, 'att_scores': 10, 'att_context': 10,
                                 'att_bwd_ctx': 10, 'att_bwd_dalpha': 10, 'att_bwd_softmax': 10,
                                 'tc_gemm_3xtf32': 112, 'tc_gemm_3xtf32_skinny': 13},
    'b128_d256_a100_v500_t24x10': {'gemm_smallm_tn': 2, 'att_scores': 10, 'att_context': 10, 'att_bwd_ctx': 10,
                                   'att_bwd_dalpha': 10, 'att_bwd_softmax': 10, 'tc_gemm_3xtf32': 99,
                                   'tc_gemm_3xtf32_skinny': 10},
    'b6_d200_a48_v500_t40x35': {'gemm_mid_tn': 2, 'gemm_smallm_nn': 35, 'gemm_smallm_tn': 1, 'att_scores': 35,
                                'att_context': 35, 'att_bwd_ctx': 35, 'att_bwd_dalpha': 35, 'att_bwd_softmax': 35,
                                'tc_gemm_3xtf32': 9, 'tc_gemm_3xtf32_skinny': 191},
    'b3_d200_a48_v500_t136x35': {'gemm_mid_tn': 2, 'gemm_smallm_nn': 35, 'gemm_smallm_tn': 1, 'att_scores': 35,
                                 'att_context': 35, 'att_bwd_ctx': 35, 'att_bwd_dalpha': 35, 'att_bwd_softmax': 35,
                                 'tc_gemm_3xtf32': 10, 'tc_gemm_3xtf32_skinny': 190},
    'b4_d1000_a100_v30000_t400x30': {'gemm_big_tn': 2, 'gemm_mid_tn': 1, 'att_scores': 30, 'att_context': 30,
                                     'att_bwd_ctx': 30, 'att_bwd_dalpha': 30, 'att_bwd_softmax': 30,
                                     'tc_gemm_3xtf32': 23, 'tc_gemm_3xtf32_skinny': 182},
}
COUNTED = ('tc_gemm_3xtf32', 'tc_gemm_3xtf32_skinny', 'gemm_', 'att_')


def _options(case):
    return dict(dim_word=case['W'], dim=case['D'], dim_att=case['A'], n_words=case['V'], encoder='gru',
                decoder='gru_cond')


def _params(case):
    """Reference init under the case's seed with non-zero biases, sharper attention (U_att) and a livelier readout
    (ff_logit_W) and target side (Wemb): at the reference scales the attention is near uniform and the logits near 0."""
    np.random.seed(case['seed'])
    P = O.init_params(_options(case))
    rng = np.random.RandomState(case['seed'] + 1)
    for k in P:
        if P[k].ndim == 1:
            P[k] = (0.1 * rng.randn(*P[k].shape)).astype('float32')
    P['ff_logit_W'] = (P['ff_logit_W'] * 40).astype('float32')
    P['decoder_U_att'] = (P['decoder_U_att'] * 30).astype('float32')
    P['Wemb'] = (P['Wemb'] * 10).astype('float32')
    return P


def _batch(case):
    B, Tx, Ty, V = case['B'], case['Tx'], case['Ty'], case['V']
    rs = np.random.RandomState(case['seed'] + 2)
    lx = rs.randint(1, Tx + 1, size=B)          # valid positions per column, EOS included
    ly = rs.randint(1, Ty + 1, size=B)
    lx[0], ly[0] = Tx, Ty
    if B > 1:
        lx[1], ly[1] = 1, (Ty + 1) // 2
    sx = [list(rs.randint(2, V, size=L - 1)) for L in lx]
    sy = [list(rs.randint(2, V, size=L - 1)) for L in ly]
    batch = O.prepare_data(sx, sy, n_words=V)
    assert batch[0].shape == (Tx, B) and batch[2].shape == (Ty, B)
    return batch


def _relerr(g, ref):
    nr = np.linalg.norm(ref)
    if nr == 0.0:
        return 0.0 if not np.any(g) else np.inf
    return float(np.linalg.norm(np.asarray(g, 'float64') - ref) / nr)


def _tf32(x):
    """the tf32 part of an fp32 word: its upper 19 bits (what a kernel that drops the lo term multiplies with)"""
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype('float64')


class _AttCapture:
    """numpy for the oracle module, recording the per-step attention terms gru_cond_layer_bwd hands to np.einsum:
    d e [Tx, B] (into U_att) and d zp [Tx, B, A] (into D_wei), in the order of the reverse scan"""

    def __init__(self):
        self.de, self.dzp = [], []

    def __getattr__(self, name):
        return getattr(np, name)

    def einsum(self, spec, *ops):
        if spec == 'tb,tba->a':
            self.de.append(ops[0])
        elif spec == 'bt,tba->a':
            self.dzp.append(ops[1])
        return np.einsum(spec, *ops)


# ------------------------------------------------------------------------------------------------ reference
def _reference(P, batch, ctx, init, scale):
    """float64 decoder, readout, NLL and their backward on the encoder output (ctx [Tx, B, C], init [B, D]), as
    O.model_fwd / O.model_bwd compose them.  Returns the device's quantities under the same names, plus S: per
    near-cancelling tensor the sum of the magnitudes of the per-step terms its gradient sums (b_att: sum |d zp|;
    W_att: |h1|^T . sum_t |d zp|; c_att: sum |d e|; U_att: sum |d e| |z|; D_wei: sum |acc_alpha| |d zp|; Wc_att:
    |ctx|^T . sum over steps of |d zp|)."""
    x, xm, y, ym = batch
    Tx, B = x.shape
    Ty = y.shape[0]
    Wd = P['Wemb'].shape[1]
    D = P['decoder_Ux'].shape[1]
    xm64, ym64 = xm.astype('float64'), ym.astype('float64')
    embs = np.zeros((Ty, B, Wd))
    embs[1:] = P['Wemb'][y[:-1].flatten()].reshape(Ty - 1, B, Wd)               # nats_oracle.py:410-411
    (Hs, Cs, As, _, _), cd = O.gru_cond_layer_fwd(P, embs, ym64, ctx, xm64, init)
    # readout and NLL (nats_oracle.py:413-422)
    pre = (Hs @ P['ff_logit_lstm_W'] + P['ff_logit_lstm_b'] + embs @ P['ff_logit_prev_W'] + P['ff_logit_prev_b']
           + Cs @ P['ff_logit_ctx_W'] + P['ff_logit_ctx_b'])
    L = np.tanh(pre).reshape(Ty * B, Wd)
    lg = L @ P['ff_logit_W'] + P['ff_logit_b']
    mx = lg.max(1, keepdims=True)
    lse = mx[:, 0] + np.log(np.exp(lg - mx).sum(1))
    rows = np.arange(Ty * B)
    cost = ((lse - lg[rows, y.flatten()]).reshape(Ty, B) * ym64).sum(0)
    # readout backward (nats_oracle.py:444-458)
    G = O.zero_grads(P)
    dlg = np.exp(lg - lse[:, None])
    dlg[rows, y.flatten()] -= 1.
    dlg *= (ym64 * scale).reshape(Ty * B, 1)
    G['ff_logit_W'] += L.T @ dlg
    G['ff_logit_b'] += dlg.sum(0)
    dpre = (dlg @ P['ff_logit_W'].T) * (1. - L * L)
    G['ff_logit_lstm_W'] += Hs.reshape(Ty * B, D).T @ dpre
    G['ff_logit_prev_W'] += embs.reshape(Ty * B, Wd).T @ dpre
    G['ff_logit_ctx_W'] += Cs.reshape(Ty * B, 2 * D).T @ dpre
    for k in ('ff_logit_lstm_b', 'ff_logit_prev_b', 'ff_logit_ctx_b'):
        G[k] += dpre.sum(0)
    dHs = (dpre @ P['ff_logit_lstm_W'].T).reshape(Ty, B, D)
    dCs = (dpre @ P['ff_logit_ctx_W'].T).reshape(Ty, B, 2 * D)
    dembs = (dpre @ P['ff_logit_prev_W'].T).reshape(Ty, B, Wd)
    cap = _AttCapture()
    O.np = cap
    try:
        demb_d, dcc, dinit = O.gru_cond_layer_bwd(P, cd, dHs, dCs, G)
    finally:
        O.np = np
    dembs = dembs + demb_d
    np.add.at(G['Wemb'], y[:-1].flatten(), dembs[1:].reshape((Ty - 1) * B, Wd))  # nats_oracle.py:462
    # ff_state (nats_oracle.py:464-467), on the masked mean of the given ctx
    mean = (ctx * xm64[:, :, None]).sum(0) / xm64.sum(0)[:, None]
    dpre0 = dinit * (1. - init ** 2)
    G['ff_state_W'] += mean.T @ dpre0
    G['ff_state_b'] += dpre0.sum(0)
    dmean = dpre0 @ P['ff_state_W'].T
    # per-step terms, in scan order
    dzp, de, steps = cap.dzp[::-1], cap.de[::-1], cd['steps']
    adzp = sum(np.abs(z) for z in dzp)                                          # [Tx, B, A]
    C = ctx.shape[2]
    S = {'decoder_b_att': adzp.sum((0, 1)),
         'decoder_W_att': sum(np.abs(s['h1']).T @ np.abs(z).sum(0) for s, z in zip(steps, dzp)),
         'decoder_c_att': np.array([sum(np.abs(e).sum() for e in de)]),
         'decoder_U_att': sum(np.einsum('tb,tba->a', np.abs(e), np.abs(s['z'])) for s, e in zip(steps, de)),
         'decoder_D_wei': sum(np.einsum('bt,tba->a', np.abs(s['acc_alpha']), np.abs(z)) for s, z in zip(steps, dzp)),
         'decoder_Wc_att': np.abs(ctx).reshape(-1, C).T @ adzp.reshape(-1, adzp.shape[2])}
    return dict(pctx=cd['pctx'], dec_h=Hs, dec_ctx=Cs, dec_alpha=As, logits=lg, dlogits=dlg, cost=cost, G=G,
                dcc=dcc, dmean=dmean, S=S)


def _cancel_err(g, ref, S):
    """max_i |g_i - g*_i| / S_i; where S_i = 0 the gradient is an empty sum and must be exactly 0"""
    d = np.abs(np.asarray(g, 'float64').reshape(S.shape) - ref.reshape(S.shape))
    if np.any(d[S == 0] != 0):
        return np.inf
    return float((d[S > 0] / S[S > 0]).max()) if np.any(S > 0) else 0.0


def _errors(out, ref):
    """per-member errors of a run (device, or the degraded reference) against the reference"""
    e = {k: float(np.abs(out[k] - ref[k]).max()) for k in STATE_VIEWS}
    e['logits'] = _relerr(out['logits'], ref['logits'])
    for k in READOUT + PRODUCTS + ELEMENTWISE + ('ff_logit_W', 'Wemb'):
        e[k] = _relerr(out['G'][k], ref['G'][k])
    e['dcc'] = _relerr(out['dcc'], ref['dcc'])
    e['dmean'] = _relerr(out['dmean'], ref['dmean'])
    for k in CANCEL:
        e[k] = _cancel_err(out['G'][k], ref['G'][k], ref['S'][k])
    return e


def _kernel_errors(out, batch, scale):
    """nll_rows, dlogits_inplace and colsum, each on the device's own input (the saved logits / the d logits view):
    the cost (relative, per sample), d logits (max abs / scale) and the ff_logit_b gradient (relative)"""
    y, ym = batch[2], batch[3]
    lg = out['logits'].astype('float64')
    rows = np.arange(lg.shape[0])
    mx = lg.max(1, keepdims=True)
    lse = mx[:, 0] + np.log(np.exp(lg - mx).sum(1))
    ymf = ym.astype('float64').flatten()
    cost = ((lse - lg[rows, y.flatten()]) * ymf).reshape(ym.shape).sum(0)
    dlg = np.exp(lg - lse[:, None])
    dlg[rows, y.flatten()] -= 1.
    dlg *= (ymf * scale)[:, None]
    return {'cost': float((np.abs(out['cost'] - cost) / np.abs(cost)).max()),
            'dlogits': float(np.abs(out['dlogits'] - dlg).max() / scale),
            'colsum': _relerr(out['G']['ff_logit_b'], out['dlogits'].astype('float64').sum(0))}


def _family_errors(errs):
    """each family's worst error (the families whose members errs has: the emulation has no 'kernels')"""
    return {f: max(errs[k] for k in members) for f, members in FAMILIES.items() if all(k in errs for k in members)}


# ------------------------------------------------------------------------------------------------ device
def _launches(lib, eng):
    n = lib.nats_profile_num_classes()
    ms, fl, by, la = (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_int64 * n)()
    from nats_b200 import _lib
    _lib.check(lib.nats_profile_read(eng.ctx, n, ms, fl, by, la), 'nats_profile_read')
    lib.nats_profile_enable(eng.ctx, 0)
    names = [lib.nats_profile_class_name(i).decode() for i in range(n)]
    return {k: int(la[i]) for i, k in enumerate(names) if la[i] and k.startswith(COUNTED)}


def _device_run(case, P32, batch, repeat=1):
    """the case through the C ABI (nats_train_fwd, nats_train_bwd_begin); one dict per repetition on the same
    workspace with the forward views, the cost, the saved logits, d logits, dcc, dmean, the gradients and the launch
    counts"""
    import torch
    from nats_b200 import nats, _lib
    eng = nats.get_engine()
    lib = eng.lib
    tparams = nats.init_tparams(P32)
    D, A, C = case['D'], case['A'], 2 * case['D']
    x, xm, y, ym = batch
    Tx, B = x.shape
    Ty = y.shape[0]
    dims = _lib.Dims(case['V'], case['W'], D, A)
    dev = eng.device
    xd, xmd, yd, ymd = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in batch]
    nbytes = int(lib.nats_train_workspace_bytes(ctypes.byref(dims), Tx, Ty, B))
    assert nbytes > 0
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    cost = torch.zeros(B, dtype=torch.float32, device=dev)
    grads = torch.zeros(tparams.total + _lib.GRAD_TAIL, dtype=torch.float32, device=dev)
    split = int(lib.nats_grad_split(ctypes.byref(dims)))
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    st = eng.stream()

    def view(name, shape):
        ptr = lib.nats_train_ws_view(ctypes.byref(dims), Tx, Ty, B, p(ws), name.encode())
        assert ptr, name
        off = (ptr - ws.data_ptr()) // 4
        return ws.view(torch.float32)[off:off + int(np.prod(shape))].cpu().numpy().reshape(shape).copy()

    runs = []
    for _ in range(repeat):
        out = {}
        _lib.check(lib.nats_profile_enable(eng.ctx, 1), 'nats_profile_enable')
        _lib.check(lib.nats_train_fwd(eng.ctx, st, ctypes.byref(dims), p(tparams.flat), p(xd), p(xmd), p(yd), p(ymd),
                                      Tx, Ty, B, p(ws), nbytes, p(cost)), 'nats_train_fwd')
        torch.cuda.synchronize()
        out['cost'] = cost.cpu().numpy().copy()
        for name, shape in (('ctx', (Tx, B, C)), ('init_state', (B, D)), ('pctx', (Tx, B, A)), ('dec_h', (Ty, B, D)),
                            ('dec_ctx', (Ty, B, C)), ('dec_alpha', (Ty, B, Tx)), ('logits', (Ty * B, case['V']))):
            out[name] = view(name, shape)
        _lib.check(lib.nats_train_bwd_begin(eng.ctx, st, ctypes.byref(dims), p(tparams.flat), p(xd), p(xmd), p(yd),
                                            p(ymd), Tx, Ty, B, p(ws), nbytes, ctypes.c_float(1.0 / B), p(grads)),
                   'nats_train_bwd_begin')
        out['launches'] = _launches(lib, eng)
        out['dlogits'] = view('logits', (Ty * B, case['V']))
        out['dcc'] = view('dcc', (Tx, B, C))
        out['dmean'] = view('dmean', (B, C))
        out['G'] = tparams.view_of(grads)
        # what lies before the split is Wemb and the two encoders; only the target-side Wemb scatter has run
        assert tparams['ff_state_W'].offset == split
        runs.append(out)
    torch.cuda.synchronize()
    return runs


def _check_alpha(alpha, xm):
    """alpha is exactly 0 at masked source positions; every row sums to 1"""
    masked = np.broadcast_to((xm.T == 0)[None], alpha.shape)
    assert np.all(alpha[masked] == 0)
    dev = float(np.abs(alpha.astype('float64').sum(2) - 1.0).max())
    assert dev <= ALPHA_SUM, dev
    return dev


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c['id'] for c in CASES])
def test_decoder_vs_float64(case):
    P32 = _params(case)
    P = O.cast_params(P32, 'float64')
    batch = _batch(case)
    scale = 1.0 / case['B']
    out = _device_run(case, P32, batch)[0]
    ref = _reference(P, batch, out['ctx'].astype('float64'), out['init_state'].astype('float64'), scale)
    errs = _errors(out, ref)
    errs.update(_kernel_errors(out, batch, scale))
    errs['alpha_sum'] = _check_alpha(out['dec_alpha'], batch[1])
    # d logits rows of masked target steps are exactly 0
    assert np.all(out['dlogits'][batch[3].flatten() == 0] == 0)
    fam = _family_errors(errs)
    print('decoder errors', case['id'], json.dumps(fam), json.dumps(errs), 'launches', json.dumps(out['launches']))
    ts = os.environ.get('NATS_TS', '1')
    if ts == '1':
        assert out['launches'] == LAUNCHES[case['id']], out['launches']
    for f, members in FAMILIES.items():
        for k in members:
            assert errs[k] <= BOUND[f], (case['id'], f, k, errs[k])


@pytest.mark.gpu
def test_decoder_is_deterministic():
    """Every reduction of the decoder, readout and their backward has a fixed order: two runs on the same workspace give
    the same bits, except the Wemb gradient, whose scatter uses atomics."""
    case = next(c for c in CASES if c['D'] == 500)
    r1, r2 = _device_run(case, _params(case), _batch(case), repeat=2)
    for k in ('ctx', 'init_state', 'pctx', 'dec_h', 'dec_ctx', 'dec_alpha', 'logits', 'cost', 'dlogits', 'dcc',
              'dmean'):
        np.testing.assert_array_equal(r1[k], r2[k], err_msg=k)
    for k in r1['G']:
        if k != 'Wemb' and not k.startswith('encoder'):
            np.testing.assert_array_equal(r1['G'][k], r2['G'][k], err_msg=k)


@pytest.mark.gpu
def test_skinny_in_shared_memory_vs_float64():
    """NATS_TS=0 (read at context creation, hence a fresh process): the skinny products split the weights in shared
    memory instead of registers.  Two cases whose per-step products are skinny, under the same bounds."""
    env = dict(os.environ, NATS_TS='0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', '-s', '-m', 'gpu', 'tests/test_gpu_decoder.py', '-k',
                        'test_decoder_vs_float64 and (b33_d256 or b64_d500)'],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print('\n'.join(l[l.index('decoder errors'):] for l in r.stdout.splitlines() if 'decoder errors' in l))
    assert r.returncode == 0 and '2 passed' in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ emulation (no GPU)
def _degraded_errors(case):
    """-> {degradation: per-member errors} of the float64 reference with the per-step or the readout weights truncated
    to tf32, against the exact one, on the case's inputs and the oracle's own encoder output"""
    P = O.cast_params(_params(case), 'float64')
    batch = _batch(case)
    _, cache = O.model_fwd(P, *batch)
    ctx, init = cache['ctx'], cache['init_state']
    scale = 1.0 / case['B']
    ref = _reference(P, batch, ctx, init, scale)
    out = {}
    for name, keys in (('step', STEP_WEIGHTS), ('readout', READOUT_WEIGHTS)):
        Q = dict(P)
        for k in keys:
            Q[k] = _tf32(P[k])
        out[name] = _errors(_reference(Q, batch, ctx, init, scale), ref)
    return out


# The cases with a decoder step to degrade, at most 40 source positions (the degraded error hardly depends on Tx); the
# config-3 decoder at Tx = 40 and Ty = 12.
EMULATED = ([dict(c, Tx=min(c['Tx'], 40)) for c in CASES if c['Tx'] > 1 and c['D'] < 1000] +
            [dict(c, Tx=40, Ty=12) for c in CASES if c['D'] == 1000])


def test_bounds_reject_a_degraded_decoder():
    """Every bound of a family a degradation must fail (MUST_FAIL) sits at most at a quarter of the smallest error, over
    the emulated cases and the family's members, of the reference with those weights truncated to tf32; and every
    recorded device error is within its bound."""
    assert set(MEASURED) == {c['id'] for c in CASES} | {c['id'] + ' NATS_TS=0' for c in CASES
                                                         if c['id'].startswith(('b33_d256', 'b64_d500'))}
    for case, errs in MEASURED.items():
        for f, v in zip(MEASURED_COLUMNS, errs):
            assert v <= BOUND[f], (case, f, v)
    worst = {}
    for case in EMULATED:
        res = _degraded_errors(case)
        print(case['id'], json.dumps({d: _family_errors(e) for d, e in res.items()}))
        for d, fams in MUST_FAIL.items():
            for f in fams:
                low = min(res[d][k] for k in FAMILIES[f])      # every member of the family must fail, not only one
                worst[(d, f)] = min(worst.get((d, f), np.inf), low)
    print('smallest degraded error per family', worst)
    for (d, f), v in worst.items():
        assert BOUND[f] <= v / 4, (d, f, BOUND[f], v)
