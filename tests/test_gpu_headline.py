"""GPU parity AT THE HEADLINE DIMENSIONS (BASELINE configs 3 and 5: D=1000, W=A=100, V=30000, src_len 400 / 800, beam 10)
against the float64 oracle: these are the shapes on which the persistent wgmma encoder (64 + 64 CTAs per pass, 189-row
tiles x 4 K chunks forward, 125-row tiles x 8 K chunks backward), the split-K decoder products, the TMA slices of the
attention kernels and the top-k over 30 k words run.
Tolerances as everywhere (fp32 path, 3xTF32 products): per-sample cost rel <= 1e-4, every gradient ||g-g*||/||g*|| <= 1e-3,
f_next probabilities max abs <= 1e-5, identical beam tokens.  Also: every kernel-selection switch of the library is run
through the parity tests in a subprocess (the switches are read once, at context creation)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import nats_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTS = dict(dim_word=100, dim=1000, dim_att=100, n_words=30000, encoder='gru', decoder='gru_cond')


@pytest.fixture(scope='module')
def N():
    from nats_b200 import nats
    return nats


@pytest.fixture(scope='module')
def params():
    """Reference init under a fixed seed, with non-zero biases and a livelier attention / readout than the reference's
    N(0, 0.01^2) so that alpha and the output distribution are far from uniform (well-separated beam candidates)."""
    np.random.seed(2024)
    P32 = O.init_params(OPTS)
    rng = np.random.RandomState(7)
    for k in P32:
        if P32[k].ndim == 1:
            P32[k] = (0.05 * rng.randn(*P32[k].shape)).astype('float32')
    P32['ff_logit_W'] = (P32['ff_logit_W'] * 40).astype('float32')
    P32['decoder_U_att'] = (P32['decoder_U_att'] * 30).astype('float32')
    P32['Wemb'] = (P32['Wemb'] * 10).astype('float32')
    return O.cast_params(P32, 'float32')


def _relerr(a, b):
    return np.linalg.norm(a.astype('float64') - b) / max(np.linalg.norm(b), 1e-30)


def _ragged(B, lo_x, hi_x, lo_y, hi_y, seed):
    rs = np.random.RandomState(seed)
    sx = [list(rs.randint(2, 30000, size=rs.randint(lo_x, hi_x + 1))) for _ in range(B)]
    sy = [list(rs.randint(2, 30000, size=rs.randint(lo_y, hi_y + 1))) for _ in range(B)]
    sx[0] = list(rs.randint(2, 30000, size=hi_x)); sy[0] = list(rs.randint(2, 30000, size=hi_y))     # the full padded shape
    return sx, sy


def test_config3_cost_and_grads_vs_oracle(N, params):
    """Tx=400, Ty=30, B=4 ragged: per-sample cost and all 43 gradients; then the same four sentences inside a B=32
    batch (batch / padding invariance ties the B=32 execution to the oracle-checked one)."""
    P = O.cast_params(params, 'float64')
    sx, sy = _ragged(4, 200, 399, 12, 29, seed=11)
    batch = O.prepare_data(sx, sy, n_words=30000)
    assert batch[0].shape == (400, 4) and batch[2].shape == (30, 4)
    tparams = N.init_tparams(params)
    graph = N.build_model(tparams, OPTS)[-1]
    cost_ref, _ = O.model_fwd(P, *batch)
    cost = graph.f_log_probs(*batch)
    np.testing.assert_allclose(cost, cost_ref, rtol=1e-4)
    mean_ref, G, _ = O.f_grad(P, *batch)
    g = graph.mean()
    mean_cost = g.grad_step(*batch, after_grads=lambda: None)
    Gd = tparams.view_of(g.grads[:tparams.total])
    assert abs(mean_cost - mean_ref) <= 1e-4 * abs(mean_ref)
    gnorm = np.sqrt(sum(np.sum(G[k] ** 2) for k in G))
    worst = 0.0
    for k in G:
        n = np.linalg.norm(G[k])
        if n < 1e-12:
            assert np.abs(Gd[k]).max() < 1e-6, k
            continue
        rel = _relerr(Gd[k], G[k])
        worst = max(worst, rel)
        # near-total cancellations (b_att / W_att: softmax backward terms sum to ~0 over the source) are bounded against
        # the global gradient norm instead
        assert rel <= 1e-3 or np.linalg.norm(Gd[k] - G[k]) / gnorm <= 1e-6, (k, rel)
    print('config-3 dims: cost rel err %.2e, worst per-tensor gradient rel err %.2e' %
          (np.abs(cost - cost_ref).max() / np.abs(cost_ref).max(), worst))
    # B = 32: the four checked sentences + 28 others
    sx2, sy2 = _ragged(28, 150, 399, 10, 29, seed=12)
    big = O.prepare_data(sx + sx2, sy + sy2, n_words=30000)
    assert big[0].shape == (400, 32)
    cost32 = graph.f_log_probs(*big)
    np.testing.assert_allclose(cost32[:4], cost, rtol=2e-5)
    assert np.all(np.isfinite(cost32))


def test_config5_sampler_vs_oracle(N, params):
    """f_init at src_len 800 (+EOS: Tx = 801) and 5 chained f_next calls with n = 10 hypotheses."""
    P = O.cast_params(params, 'float64')
    rs = np.random.RandomState(3)
    x = np.concatenate([rs.randint(2, 30000, size=800), [0]]).astype('int64')[:, None]
    tparams = N.init_tparams(params)
    f_init, f_next = N.build_sampler(tparams, OPTS)
    s0, ctx0 = f_init(x)
    r0, rctx = O.f_init(P, x)
    np.testing.assert_allclose(np.asarray(s0), r0, rtol=1e-4, atol=2e-6)
    np.testing.assert_allclose(np.asarray(ctx0), rctx, rtol=1e-4, atol=2e-6)
    n = 10
    state = np.tile(np.asarray(s0), [n, 1]) + 0.05 * rs.randn(n, 1000).astype('float32')
    ac = np.zeros((n, 2000), 'float32'); aa = np.zeros((n, 801), 'float32')
    rstate, rac, raa = state.astype('float64'), ac.astype('float64'), aa.astype('float64')
    y = -np.ones((n,), 'int64')
    ctx_t = np.tile(ctx0, [n, 1])
    rctx_t = np.tile(rctx, [n, 1])
    for t in range(5):
        out = f_next(y, ctx_t, state, ac, aa)
        ref = O.f_next(P, y, rctx_t, rstate, rac, raa)
        assert np.abs(np.asarray(out[0]) - ref[0]).max() <= 1e-5, t
        for i in (2, 3, 4, 5, 6):
            np.testing.assert_allclose(np.asarray(out[i]), ref[i], rtol=2e-4, atol=2e-6, err_msg='step %d out %d' % (t, i))
        state, ac, aa = out[2], out[5], out[6]
        rstate, rac, raa = ref[2], ref[5], ref[6]
        y = rs.randint(2, 30000, size=n).astype('int64')


def test_config5_softmax_cluster_matches_row_kernel(N, params):
    """The beam-search f_next (no multinomial draw) normalises the |V| = 30000 rows with the 8-CTA cluster kernel, the
    sampling f_next with one CTA per row: same probabilities (nats.py:861) up to the summation order."""
    import torch
    rs = np.random.RandomState(9)
    x = np.concatenate([rs.randint(2, 30000, size=120), [0]]).astype('int64')[:, None]
    tparams = N.init_tparams(params)
    f_init, f_next = N.build_sampler(tparams, OPTS)
    s0, ctx0 = f_init(x)
    h = ctx0._nats_handle
    eng = f_next.engine
    n, Tx = 10, int(ctx0.shape[0])
    f32 = dict(dtype=torch.float32, device=eng.device)
    st = torch.from_numpy(np.tile(np.asarray(s0), [n, 1]) + 0.05 * rs.randn(n, 1000).astype('float32')).to(eng.device)
    ac, aa = torch.zeros((n, 2000), **f32), torch.zeros((n, Tx), **f32)
    y = torch.from_numpy(rs.randint(2, 30000, size=n).astype('int64')).to(eng.device)
    res = []
    for smp in (None, torch.empty((n,), dtype=torch.int64, device=eng.device)):
        outs = [torch.empty((n, 30000), **f32), smp, torch.empty((n, 1000), **f32), torch.empty((n, Tx), **f32),
                torch.empty((n, 2000), **f32), torch.empty((n, 2000), **f32), torch.empty((n, Tx), **f32)]
        f_next.next_device(y, h.ctx_dev, h.pctx_dev, st, ac, aa, Tx, n, outs)
        res.append(outs[0].cpu().numpy())
    assert np.isfinite(res[0]).all()
    np.testing.assert_allclose(res[0].sum(1), 1.0, rtol=1e-5)
    np.testing.assert_allclose(res[0], res[1], rtol=2e-6, atol=1e-12)


def test_config5_batched_f_init_vs_oracle(N, params):
    """Three sources of 400 / 250 / 31 words encoded in one masked launch of the persistent encoder kernel: init_state and
    the valid rows of ctx equal the float64 oracle's single-sentence f_init."""
    P = O.cast_params(params, 'float64')
    rs = np.random.RandomState(21)
    xs = [np.concatenate([rs.randint(2, 30000, size=L), [0]]).astype('int64') for L in (400, 250, 31)]
    tparams = N.init_tparams(params)
    f_init, f_next = N.build_sampler(tparams, OPTS)
    f_init.prefetch(xs)
    for x in xs:
        s0, ctx, pctx = f_init.device(x)
        r0, rctx = O.f_init(P, x[:, None])
        np.testing.assert_allclose(s0.cpu().numpy(), r0[0], rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(ctx.cpu().numpy(), rctx[:, 0], rtol=1e-4, atol=2e-6)
        assert tuple(pctx.shape) == (len(x), 100)


def test_config5_beam_vs_oracle(N, params):
    """10 beam steps, k = 10, all three distraction factors on, src_len 400: identical tokens, scores and penalty
    vectors (nats.py:981-999) as the literal restatement driven by the float64 oracle's f_init / f_next."""
    P = O.cast_params(params, 'float64')
    rs = np.random.RandomState(5)
    x = np.concatenate([rs.randint(2, 30000, size=400), [0]]).astype('int64')[:, None]
    tparams = N.init_tparams(params)
    f_init, f_next = N.build_sampler(tparams, OPTS)
    tr = []
    got_s, got_sc, _ = N.gen_sample(tparams, f_init, f_next, x, OPTS, k=10, maxlen=10, stochastic=False, use_unk=True,
                                    kl_factor=1.0, ctx_factor=1.0, state_factor=1.0, _trace=tr)
    fi = lambda x_: O.f_init(P, x_)
    fn = lambda y_, c_, s_, ac_, aa_: O.f_next(P, y_, c_, s_, ac_, aa_)
    rtr = []
    ref_s, ref_sc, _ = O.gen_sample(fi, fn, x, k=10, maxlen=10, stochastic=False, use_unk=True, kl_factor=1.0,
                                    ctx_factor=1.0, state_factor=1.0, trace=rtr)
    assert [list(map(int, s)) for s in got_s] == [list(map(int, s)) for s in ref_s]
    np.testing.assert_allclose(np.array(got_sc, 'float64'), np.array(ref_sc, 'float64'), rtol=2e-4)
    ref_pen = [r['pen'] for r in rtr if r['pen'] is not None]
    assert len(tr) == len(ref_pen) and len(tr) >= 8
    for a, b in zip(tr, ref_pen):
        np.testing.assert_allclose(a['pen'], b, rtol=5e-4, atol=5e-6)


SWITCHES = [
    {'NATS_ENC_TC': '0'},                 # per-step encoder path instead of the persistent tensor-core kernel
    {'NATS_ENC_TC': '2'},                 # persistent forward + per-step backward
    {'NATS_ENC_TC': '3'},                 # per-step forward + persistent backward
    {'NATS_TS': '0'},                     # skinny products split in shared memory instead of registers
    {'NATS_PDL': '0'},                    # no programmatic dependent launch
    # beam-search kernels: one CTA per row / per (row, slice) and library GEMMs instead of the 8-CTA cluster kernels
    {'NATS_TOPK_SIMPLE': '1', 'NATS_SOFTMAX_SIMPLE': '1', 'NATS_ATT_BCAST': '0', 'NATS_NARROW_PROJ': '0'},
    {'NATS_DEVICE_BEAM': '0'},            # beam bookkeeping on the host (the reference's loop) instead of on the device
]


@pytest.mark.parametrize('env', SWITCHES, ids=lambda e: ','.join('%s=%s' % kv for kv in e.items()))
def test_kernel_switches_keep_parity(env):
    """Every non-default kernel selection goes through the oracle parity tests (toy shapes + LCSTS-shaped dims, where the
    persistent encoder is eligible) in a fresh process."""
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', '-m', 'gpu', 'tests/test_gpu_parity.py', '-k',
                        'cost_and_grads or real_dims or sampler_matches or sampler_batched or beam_search or topk'], cwd=ROOT, env=e, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
