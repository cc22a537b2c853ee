"""GPU parity: the CUDA path (through the C ABI, via nats_b200.nats) against the float64 oracle on the same
seeded inputs, and against the committed golden fixtures.  Tolerances (fp32 FFMA path, stated per output):
  per-sample cost   rel <= 1e-4        gradients  ||g-g*|| / ||g*|| <= 1e-3 per tensor (measured ~1e-6)
  f_next probs      max abs <= 1e-5    beam search: identical token sequences
"""
import os

import numpy as np
import pytest

from oracle import nats_oracle as O
from tests.helpers import toy_options, toy_params, ragged_batch, full_batch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def N():
    from nats_b200 import nats
    return nats


def _setup(N, opts, P64):
    tparams = N.init_tparams(O.cast_params(P64, 'float32'))
    graph = N.build_model(tparams, opts)[-1]
    return tparams, graph


def _grads_of(N, tparams, graph, batch, decay_c=0., clip_c=-1.):
    g = graph.mean()
    g.decay_c, g.clip_c = decay_c, clip_c
    cost = g.grad_step(*batch, after_grads=lambda: None)
    return cost, tparams.view_of(g.grads[:tparams.total]), g


def _relerr(a, b):
    return np.linalg.norm(a.astype('float64') - b) / max(np.linalg.norm(b), 1e-30)


CASES = [
    dict(D=8, W=6, A=5, V=50, B=3, max_x=8, max_y=5),          # golden dims (bulk-copy path, C % 4 == 0)
    dict(D=7, W=5, A=3, V=40, B=2, max_x=9, max_y=4),          # odd sizes: scalar / non-bulk fallbacks
    dict(D=64, W=20, A=12, V=300, B=5, max_x=37, max_y=11),    # toy-config dims (BASELINE config 1)
    dict(D=40, W=16, A=33, V=200, B=35, max_x=21, max_y=9),    # batch > 32: second row tile of the step GEMMs
]


@pytest.mark.parametrize('case', CASES)
def test_cost_and_grads_match_oracle(N, case):
    opts = toy_options(D=case['D'], W=case['W'], A=case['A'], V=case['V'])
    P = toy_params(opts)
    batch = ragged_batch(case['V'], B=case['B'], max_x=case['max_x'], max_y=case['max_y'], seed=11)
    tparams, graph = _setup(N, opts, P)
    cost_ref, cache = O.model_fwd(P, *batch)
    cost = graph.f_log_probs(*batch)
    np.testing.assert_allclose(cost, cost_ref, rtol=1e-4)
    mean_ref, G, _ = O.f_grad(P, *batch)
    mean_cost, Gd, _ = _grads_of(N, tparams, graph, batch)
    assert abs(mean_cost - mean_ref) <= 1e-4 * abs(mean_ref)
    for k in G:
        if np.linalg.norm(G[k]) < 1e-12:
            assert np.abs(Gd[k]).max() < 1e-6, k        # decoder_c_att: exact gradient is 0
        else:
            assert _relerr(Gd[k], G[k]) <= 1e-3, (k, _relerr(Gd[k], G[k]))
    # second and third call exercise the CUDA-graph capture + replay of the same shape
    for _ in range(3):
        c2, Gd2, _ = _grads_of(N, tparams, graph, batch)
        assert abs(c2 - mean_ref) <= 1e-4 * abs(mean_ref)
    for k in G:
        if np.linalg.norm(G[k]) >= 1e-12:
            assert _relerr(Gd2[k], G[k]) <= 1e-3, k


def test_golden_train_fixture(N):
    z = np.load(os.path.join(GOLD, 'train_toy.npz'))
    V, W, D, A = [int(v) for v in z['opt_dims']]
    opts = toy_options(D=D, W=W, A=A, V=V)
    names = list(O.init_params(opts).keys())
    P = O.OrderedDict((k, z['p_' + k]) for k in names)
    tparams, graph = _setup(N, opts, P)
    batch = (z['x'], z['x_mask'], z['y'], z['y_mask'])
    np.testing.assert_allclose(graph.f_log_probs(*batch), z['cost'], rtol=1e-4)
    _, Gd, _ = _grads_of(N, tparams, graph, batch)
    for k in names:
        g = z['g_' + k]
        if np.linalg.norm(g) >= 1e-12:
            assert _relerr(Gd[k], g) <= 1e-3, k
    # one Adadelta step with clipping (nats.py:1145-1173, 1344-1353)
    tparams2, graph2 = _setup(N, opts, P)
    gm = graph2.mean()
    gm.clip_c = 1.0
    f_grad_shared, f_update = N.adadelta('lr', tparams2, gm, None, gm)
    f_grad_shared(*batch)
    f_update(0.01)
    za = np.load(os.path.join(GOLD, 'adadelta_toy.npz'))
    new = N.unzip(tparams2)
    for k in names:
        np.testing.assert_allclose(new[k], za['p_' + k], rtol=2e-4, atol=2e-6, err_msg=k)


def test_workspace_views_match_oracle(N):
    import ctypes
    import torch
    from nats_b200 import _lib
    opts = toy_options(D=16, W=10, A=9, V=80)
    P = toy_params(opts)
    batch = ragged_batch(80, B=4, max_x=13, max_y=7, seed=3)
    tparams, graph = _setup(N, opts, P)
    _, cache = O.model_fwd(P, *batch)
    graph.f_log_probs(*batch)
    Tx, Ty, B = batch[0].shape[0], batch[2].shape[0], batch[0].shape[1]
    p = graph.plan(Tx, Ty, B)
    PTx, PTy, _ = p.shape                         # the plan's (bucketed) shape: rows beyond Tx / Ty are masked padding
    lib = _lib.load()
    D, C = 16, 32

    def view(name, shape):
        pshape = {'ctx': (PTx, B, C), 'init_state': (B, D), 'dec_h': (PTy, B, D), 'dec_ctx': (PTy, B, C),
                  'dec_alpha': (PTy, B, PTx)}[name]
        ptr = lib.nats_train_ws_view(ctypes.byref(graph.dims), PTx, PTy, B, ctypes.c_void_p(p.ws.data_ptr()),
                                     name.encode())
        assert ptr
        off = (ptr - p.ws.data_ptr()) // 4
        n = int(np.prod(pshape))
        a = p.ws.view(torch.float32)[off:off + n].cpu().numpy().reshape(pshape)
        return a[tuple(slice(0, d) for d in shape)]

    np.testing.assert_allclose(view('ctx', (Tx, B, C)), cache['ctx'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(view('init_state', (B, D)), cache['init_state'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(view('dec_h', (Ty, B, D)), cache['Hs'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(view('dec_ctx', (Ty, B, C)), cache['Cs'], rtol=1e-4, atol=1e-6)
    al = view('dec_alpha', (Ty, B, Tx))
    np.testing.assert_allclose(al, cache['As'], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(al.sum(2), 1.0, rtol=1e-5)                     # rows sum to one (nats.py:540)
    assert np.all(al * (1 - batch[1].T[None]) == 0)                           # zero on padding (nats.py:538-539)


@pytest.mark.parametrize('opt', ['adadelta', 'adam', 'rmsprop'])
def test_optimizers_three_steps(N, opt):
    opts = toy_options(D=12, W=8, A=6, V=60)
    P = toy_params(opts)
    batch = ragged_batch(60, B=4, max_x=10, max_y=6, seed=5)
    tparams, graph = _setup(N, opts, P)
    g = graph.mean()
    g.clip_c, g.decay_c = 5.0, 1e-3
    f_grad_shared, f_update = getattr(N, opt)('lr', tparams, g, None, g)
    Pr = O.cast_params(P, 'float64')
    ref = {'adadelta': O.Adadelta, 'adam': O.Adam, 'rmsprop': O.RMSprop}[opt](Pr)
    for _ in range(3):
        cost = f_grad_shared(*batch)
        f_update(0.01)
        cr, Gr, _ = O.f_grad(Pr, *batch, decay_c=1e-3, clip_c=5.0)
        assert abs(cost - cr) <= 2e-4 * abs(cr)
        ref.grad_shared(Gr)
        ref.update(Pr)
    new = N.unzip(tparams)
    for k in Pr:
        np.testing.assert_allclose(new[k], Pr[k], rtol=5e-3, atol=2e-5, err_msg=k)


def test_sampler_matches_oracle_and_golden(N):
    z = np.load(os.path.join(GOLD, 'sampler_toy.npz'))
    zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
    V, W, D, A = [int(v) for v in zt['opt_dims']]
    opts = toy_options(D=D, W=W, A=A, V=V)
    names = list(O.init_params(opts).keys())
    P = O.OrderedDict((k, zt['p_' + k]) for k in names)
    tparams = N.init_tparams(O.cast_params(P, 'float32'))
    f_init, f_next = N.build_sampler(tparams, opts)
    init_state, ctx = f_init(z['x'])
    np.testing.assert_allclose(init_state, z['init_state'], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(np.asarray(ctx), z['ctx'], rtol=1e-4, atol=1e-6)
    state = init_state
    ac = np.zeros((1, ctx.shape[2]), 'float32'); aa = np.zeros((1, ctx.shape[0]), 'float32')
    for t in range(5):
        # alternate between the device-resident context handle and a plain ndarray (re-upload + pctx recompute)
        c_in = ctx if t % 2 == 0 else np.array(ctx)
        probs, smp, state, alT, c, ac, aa = f_next(z['yprev%d' % t], c_in, state, ac, aa)
        assert np.abs(probs - z['probs%d' % t]).max() <= 1e-5
        np.testing.assert_allclose(state, z['state%d' % t], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(alT, z['alpha%d' % t], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(c, z['ctxs%d' % t], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(ac, z['acc_ctx%d' % t], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(aa, z['acc_alpha%d' % t], rtol=1e-4, atol=1e-7)
        assert 0 <= int(smp[0]) < V


def test_sampler_batched_hypotheses(N):
    """n > 1 hypotheses sharing one source (tile of nats.py:958) == the oracle on the materialised tile."""
    opts = toy_options(D=16, W=10, A=9, V=80)
    P = toy_params(opts)
    P32 = O.cast_params(P, 'float32')
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    x = np.array([5, 9, 33, 7, 12, 41, 3, 8, 0], 'int64')[:, None]
    s0, ctx0 = f_init(x)
    n = 4
    rng = np.random.RandomState(0)
    y = np.array([4, -1, 7, 19], 'int64')
    state = np.tile(s0, [n, 1]) + 0.1 * rng.randn(n, 16).astype('float32')
    ac = 0.2 * rng.randn(n, 32).astype('float32')
    aa = np.abs(0.3 * rng.randn(n, x.shape[0])).astype('float32')
    ctx_t = np.tile(ctx0, [n, 1])
    out = f_next(y, ctx_t, state, ac, aa)
    ref = O.f_next(P, y, np.asarray(ctx_t, 'float64'), state.astype('float64'), ac.astype('float64'),
                   aa.astype('float64'))
    for i in (0, 2, 3, 4, 5, 6):
        np.testing.assert_allclose(out[i], ref[i], rtol=2e-4, atol=2e-6)


def test_distraction_scores_match_scipy(N):
    import scipy.spatial.distance
    import scipy.stats
    eng = N.get_engine()
    k, L, Tx, C, D = 3, 6, 37, 24, 12
    rng = np.random.RandomState(2)
    sc = N.DistractionScorer(eng, k, L, Tx, C, D)
    hist = []
    for s in range(4):
        a = rng.rand(k, Tx).astype('float32'); a /= a.sum(1, keepdims=True)
        c = rng.randn(k, C).astype('float32'); h = rng.randn(k, D).astype('float32')
        hist.append((a, c, h))
        sc.advance(a, c, h, [0, 1, 2])
    a = rng.rand(k, Tx).astype('float32'); a /= a.sum(1, keepdims=True)
    c = rng.randn(k, C).astype('float32'); h = rng.randn(k, D).astype('float32')
    pen = sc.penalties(a, c, h, k, 1.5, 0.7, 2.0)
    for i in range(k):
        kl = min(scipy.stats.entropy(hh[0][i], a[i]) for hh in hist)
        cc = max(scipy.spatial.distance.cosine(hh[1][i], c[i]) for hh in hist)
        ss = max(scipy.spatial.distance.cosine(hh[2][i], h[i]) for hh in hist)
        np.testing.assert_allclose(pen[:, i], [-1.5 * kl, 0.7 * cc, 2.0 * ss], rtol=2e-4, atol=2e-6)
    # reorder: new hypothesis 0 descends from old 2, new 1 from old 0
    sc.advance(a, c, h, [2, 0])
    pen2 = sc.penalties(a[[2, 0]], c[[2, 0]], h[[2, 0]], 2, 1.0, 1.0, 1.0)
    # the newest history entry equals the current vectors: min KL = 0; the cosine maxima come from older entries
    np.testing.assert_allclose(pen2[0], 0.0, atol=1e-5)
    for j, i in enumerate((2, 0)):
        cc = max(scipy.spatial.distance.cosine(hh[1][i], c[i]) for hh in hist)
        ss = max(scipy.spatial.distance.cosine(hh[2][i], h[i]) for hh in hist)
        np.testing.assert_allclose(pen2[1:, j], [cc, ss], rtol=2e-4, atol=2e-6)


def test_beam_search_matches_oracle_and_golden(N):
    z = np.load(os.path.join(GOLD, 'beam_toy.npz'))
    zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
    V, W, D, A = [int(v) for v in zt['opt_dims']]
    opts = toy_options(D=D, W=W, A=A, V=V)
    names = list(O.init_params(opts).keys())
    P32 = O.cast_params(O.OrderedDict((k, zt['p_' + k]) for k in names), 'float32')
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    samples, scores, alphas = N.gen_sample(tparams, f_init, f_next, z['x'], opts, k=3, maxlen=7, stochastic=False,
                                           use_unk=True, kl_factor=1.5, ctx_factor=1.5, state_factor=1.5)
    assert len(samples) == int(z['n_samples'])
    for i, s in enumerate(samples):
        assert list(map(int, s)) == list(map(int, z['sample%d' % i])), (i, s)
    np.testing.assert_allclose(np.array(scores, 'float32'), z['scores'], rtol=2e-4)
    assert all(len(a) == len(s) for a, s in zip(alphas, samples))
    # no distraction: plain beam search equals the oracle's
    fi = lambda x_: O.f_init(P32, x_)
    fn = lambda y_, c_, s_, ac_, aa_: O.f_next(P32, y_, c_, s_.astype('float32'), ac_.astype('float32'),
                                               aa_.astype('float32'))
    ref_s, ref_sc, _ = O.gen_sample(fi, fn, z['x'], k=4, maxlen=6, stochastic=False, use_unk=False)
    got_s, got_sc, _ = N.gen_sample(tparams, f_init, f_next, z['x'], opts, k=4, maxlen=6, stochastic=False,
                                    use_unk=False)
    assert [list(map(int, s)) for s in got_s] == [list(map(int, s)) for s in ref_s]
    np.testing.assert_allclose(np.array(got_sc), np.array(ref_sc), rtol=2e-4)
    # stochastic argmax decoding
    s1, _, _ = N.gen_sample(tparams, f_init, f_next, z['x'], opts, k=1, maxlen=6, stochastic=True, argmax=True)
    s2, _, _ = O.gen_sample(fi, fn, z['x'], k=1, maxlen=6, stochastic=True, argmax=True)
    assert list(map(int, s1)) == list(map(int, s2))


@pytest.mark.parametrize('k', [12, 20, 32])
@pytest.mark.parametrize('model', ['golden', 'w8'])
def test_beam_search_wide_beams(N, k, model):
    """Beams of 12 / 20 / 32 rows: 12 still runs the few-row cluster kernels (<= 16 rows), 20 and 32 take the general
    attention / library-GEMM paths under the same device-resident bookkeeping (beam <= 32); distraction on, early EOS
    retirements included.  'w8' has dim_word = 8 (a multiple of 4: the fused readout projection is eligible), 'golden' has
    dim_word = 6 (it is not).  Same tokens and scores as the oracle's literal restatement of nats.py:951-1066."""
    if model == 'golden':
        z = np.load(os.path.join(GOLD, 'beam_toy.npz'))
        zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
        V, W, D, A = [int(v) for v in zt['opt_dims']]
        opts = toy_options(D=D, W=W, A=A, V=V)
        names = list(O.init_params(opts).keys())
        P32 = O.cast_params(O.OrderedDict((kk, zt['p_' + kk]) for kk in names), 'float32')
        x = z['x']
    else:
        opts = toy_options(D=32, W=8, A=12, V=120)
        P32 = O.cast_params(toy_params(opts), 'float32')
        x = np.concatenate([np.random.RandomState(7).randint(2, 120, size=23), [0]]).astype('int64')[:, None]
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    fi = lambda x_: O.f_init(P32, x_)
    fn = lambda y_, c_, s_, ac_, aa_: O.f_next(P32, y_, c_, s_.astype('float32'), ac_.astype('float32'),
                                               aa_.astype('float32'))
    kw = dict(k=k, maxlen=8, stochastic=False, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    ref_s, ref_sc, _ = O.gen_sample(fi, fn, x, **kw)
    got_s, got_sc, got_al = N.gen_sample(tparams, f_init, f_next, x, opts, **kw)
    assert [list(map(int, s)) for s in got_s] == [list(map(int, s)) for s in ref_s]
    np.testing.assert_allclose(np.array(got_sc, 'float64'), np.array(ref_sc, 'float64'), rtol=5e-4)
    assert all(len(a) == len(s) for a, s in zip(got_al, got_s))


def test_f_init_prefetch_encodes_several_sentences_at_once(N):
    """f_init.prefetch: ragged sentences in ONE masked encoder launch (nats_sampler_init with x_mask) give every sentence
    the init_state / ctx / pctx of its own f_init (nats.py:789-817), and the beam search that consumes the parked result
    returns what it returns without prefetch."""
    opts = toy_options(D=32, W=8, A=12, V=120)
    P32 = O.cast_params(toy_params(opts), 'float32')
    tparams = N.init_tparams(P32)
    rs = np.random.RandomState(17)
    xs = [np.concatenate([rs.randint(2, 120, size=L), [0]]).astype('int64') for L in (5, 9, 3, 9, 14, 1)]
    f_init, f_next = N.build_sampler(tparams, opts)
    single = [tuple(t.clone() for t in f_init.device(x)) for x in xs]
    f_init.prefetch(xs, max_batch=4)                       # two launches: 4 + 2 sentences
    for x, ref in zip(xs, single):
        got = f_init.device(x)
        assert got[1].shape == ref[1].shape == (len(x), 64) and got[2].shape == (len(x), 12)
        for g, r in zip(got, ref):
            np.testing.assert_allclose(g.cpu().numpy(), r.cpu().numpy(), rtol=2e-4, atol=2e-6)
        r0, rc = O.f_init(P32, x[:, None])
        np.testing.assert_allclose(got[0].cpu().numpy(), r0[0], rtol=2e-4, atol=2e-6)
        np.testing.assert_allclose(got[1].cpu().numpy(), rc[:, 0], rtol=2e-4, atol=2e-6)
    kw = dict(k=5, maxlen=7, stochastic=False, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    plain = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, **kw) for x in xs]
    f_init.prefetch(xs)
    for x, (ps, psc, _) in zip(xs, plain):
        gs, gsc, _ = N.gen_sample(tparams, f_init, f_next, x[:, None], opts, **kw)
        assert [list(map(int, s)) for s in gs] == [list(map(int, s)) for s in ps]
        np.testing.assert_allclose(np.array(gsc, 'float64'), np.array(psc, 'float64'), rtol=2e-4)


@pytest.mark.parametrize('concurrency', [1, 3])
def test_gen_sample_many_equals_sentence_by_sentence(N, concurrency):
    """gen_sample_many: searches interleaved on separate CUDA streams (own workspace each), encoders batched -- every
    sentence gets exactly the hypotheses, scores and attention histories of its own gen_sample call (nats.py:879-1076)."""
    opts = toy_options(D=32, W=8, A=12, V=120)
    P32 = O.cast_params(toy_params(opts), 'float32')
    tparams = N.init_tparams(P32)
    rs = np.random.RandomState(23)
    xs = [np.concatenate([rs.randint(2, 120, size=L), [0]]).astype('int64') for L in (6, 11, 3, 11, 17, 2, 9, 9)]
    f_init, f_next = N.build_sampler(tparams, opts)
    kw = dict(k=6, maxlen=9, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    one = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=concurrency, chunk=5, **kw)
    assert len(many) == len(xs)
    for (s1, c1, a1), (s2, c2, a2) in zip(one, many):
        assert [list(map(int, s)) for s in s2] == [list(map(int, s)) for s in s1]
        np.testing.assert_allclose(np.array(c2, 'float64'), np.array(c1, 'float64'), rtol=2e-4)
        for h1, h2 in zip(a1, a2):
            np.testing.assert_allclose(np.array(h2), np.array(h1), rtol=2e-4, atol=1e-6)


def test_beam_topk_matches_numpy(N):
    """nats_beam_topk: per row the k largest probabilities, descending, ties by ascending index, entry 1 -> 1e-20
    when use_unk is off (nats.py:975) -- the selection that replaces the host argsort of nats.py:997-999."""
    import ctypes
    import torch
    from nats_b200 import _lib
    eng = N.get_engine()
    rng = np.random.RandomState(5)
    # (…, 32768, …) is the largest row of the 8-CTA cluster kernel (one read of the row, candidates merged through
    # distributed shared memory); 32769 columns or K = 33 take the one-CTA-per-row kernel
    for (n, V, K) in [(7, 1000, 5), (3, 30011, 10), (2, 6, 6), (1, 3, 5), (10, 30000, 10), (2, 32768, 32), (2, 32769, 7),
                      (3, 5000, 33), (4, 9, 10)]:
        p = rng.rand(n, V).astype('float32')
        p[:, 1] = 2.0                                   # the unk entry is the largest unless masked
        if V > 40:
            p[0, 17] = p[0, 33] = 1.5                   # a tie: lower index first
        if V >= 5000:
            p[1, :] = 0.25                              # a whole row of ties: indices 0, 1, 2, ... in order
            p[1, V - 3] = 0.5
            p[n - 1, 4000:4100] = 0.0                   # zeros are candidates like any other value
            p[n - 1, V - 1] = 3.0                       # the last column (last CTA of the cluster) wins
        pd = torch.from_numpy(p).to(eng.device)
        for mask in (0, 1):
            op = torch.empty((n, K), dtype=torch.float32, device=eng.device)
            oi = torch.empty((n, K), dtype=torch.int32, device=eng.device)
            _lib.check(eng.lib.nats_beam_topk(eng.ctx, eng.stream(), ctypes.c_void_p(pd.data_ptr()), n, V, K, mask,
                                              ctypes.c_void_p(op.data_ptr()), ctypes.c_void_p(oi.data_ptr())), 'topk')
            gp, gi = op.cpu().numpy(), oi.cpu().numpy()
            q = p.copy()
            if mask:
                q[:, 1] = 1e-20
            for r in range(n):
                order = np.lexsort((np.arange(V), -q[r]))[:K]        # value descending, index ascending
                kk = min(K, V)
                assert list(gi[r, :kk]) == list(order[:kk]), (n, V, K, mask, r)
                np.testing.assert_array_equal(gp[r, :kk], q[r, order[:kk]])
                assert all(gi[r, kk:] == -1)


def test_sampler_outputs_are_lazy_device_arrays(N):
    """f_next returns the seven outputs of nats.py:869-870 as DeviceArray: NumPy sees ordinary arrays, row selection
    stays on the device and can be fed back to f_next unchanged."""
    zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
    V, W, D, A = [int(v) for v in zt['opt_dims']]
    opts = toy_options(D=D, W=W, A=A, V=V)
    names = list(O.init_params(opts).keys())
    P32 = O.cast_params(O.OrderedDict((k, zt['p_' + k]) for k in names), 'float32')
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    x = np.array([[3], [5], [7], [0]], dtype='int64')
    st, ctx = f_init(x)
    k = 3
    y = -np.ones((1,), 'int64')
    out = f_next(y, ctx, st, np.zeros((1, 2 * D), 'float32'), np.zeros((1, 4), 'float32'))
    assert all(isinstance(o, N.DeviceArray) for o in out)
    assert out[0].shape == (1, V) and out[0].dtype == np.float32 and out[1].dtype == np.int64
    p_host = np.asarray(out[0])
    np.testing.assert_allclose(p_host.sum(1), 1.0, rtol=1e-5)
    # grow to k hypotheses by device-side row selection, then compare with the same call on host copies
    par = [0] * k
    y2 = np.array([4, 5, 6], 'int64')
    dev_in = (out[2][par].copy(), out[5][par].copy(), out[6][par].copy())
    assert all(isinstance(a, N.DeviceArray) for a in dev_in)
    host_in = tuple(np.asarray(o)[par].copy() for o in (out[2], out[5], out[6]))
    ctx_k = np.tile(ctx, [k, 1])
    a = f_next(y2, ctx_k, *dev_in)
    b = f_next(y2, ctx_k, *host_in)
    for i, (u, v) in enumerate(zip(a, b)):
        if i != 1:                      # the multinomial draw advances its counter at every call
            np.testing.assert_array_equal(np.asarray(u), np.asarray(v))
    # writes go to the host copy and are honoured when the array is passed back
    s_mod = out[2][par].copy()
    s_mod[:, 0] = 0.25
    hm = host_in[0].copy()
    hm[:, 0] = 0.25
    c = f_next(y2, ctx_k, s_mod, dev_in[1], dev_in[2])
    d = f_next(y2, ctx_k, hm, host_in[1], host_in[2])
    np.testing.assert_array_equal(np.asarray(c[0]), np.asarray(d[0]))


def test_full_size_properties(N):
    """BASELINE config 2 shape (Tx=120, Ty=20, D=500, V=4000, B=64 -> here B=16 to keep the oracle out): size-
    independent properties only: alpha rows sum to 1, acc_alpha row sums = #valid steps, padding invariance of the
    cost, cost finite and ~ Ty*log(V) at init."""
    opts = dict(dim_word=100, dim=500, dim_att=100, n_words=4000, encoder='gru', decoder='gru_cond')
    np.random.seed(1234)
    P = N.init_params(opts)
    tparams = N.init_tparams(P)
    graph = N.build_model(tparams, opts)[-1]
    x, xm, y, ym = full_batch(4000, B=16, Tx=120, Ty=20)
    cost = graph.f_log_probs(x, xm, y, ym)
    assert np.all(np.isfinite(cost))
    np.testing.assert_allclose(cost, 20 * np.log(4000.), rtol=0.02)
    pad = lambda a, n: np.concatenate([a, np.zeros((n,) + a.shape[1:], a.dtype)], 0)
    cost2 = graph.f_log_probs(pad(x, 5), pad(xm, 5), pad(y, 3), pad(ym, 3))
    np.testing.assert_allclose(cost2, cost, rtol=1e-5)
    g = graph.mean()
    c1 = g.grad_step(x, xm, y, ym, after_grads=lambda: None)
    assert np.isfinite(c1) and abs(c1 - cost.mean()) < 1e-3 * cost.mean()
    gn = float(g.grads[:tparams.total].double().pow(2).sum().sqrt().item())
    assert np.isfinite(gn) and gn > 0


def test_real_dims_vs_oracle(N):
    """LCSTS-shaped dims (BASELINE config 2: D=500, W=A=100, V=4000, Tx=120, Ty=20) with a reduced batch so that the
    float64 oracle finishes in seconds: the wgmma 3xTF32 path through 120 recurrent encoder steps and 20 decoder
    steps must stay within the fp32 tolerances (cost 1e-4, gradients 1e-3 per tensor)."""
    opts = dict(dim_word=100, dim=500, dim_att=100, n_words=4000, encoder='gru', decoder='gru_cond')
    np.random.seed(4321)
    P32 = N.init_params(opts)
    rng = np.random.RandomState(5)
    for k in P32:                                   # non-zero biases / livelier attention than the reference init
        if P32[k].ndim == 1:
            P32[k] = (0.05 * rng.randn(*P32[k].shape)).astype('float32')
    P = O.cast_params(P32, 'float64')
    rs = np.random.RandomState(9)
    sx = [list(rs.randint(2, 4000, size=rs.randint(60, 120))) for _ in range(4)]
    sy = [list(rs.randint(2, 4000, size=rs.randint(8, 20))) for _ in range(4)]
    batch = O.prepare_data(sx, sy, n_words=4000)
    tparams, graph = _setup(N, opts, P)
    cost_ref, _ = O.model_fwd(P, *batch)
    cost = graph.f_log_probs(*batch)
    rel_cost = np.abs(cost - cost_ref).max() / np.abs(cost_ref).max()
    mean_ref, G, _ = O.f_grad(P, *batch)
    _, Gd, _ = _grads_of(N, tparams, graph, batch)
    gnorm = np.sqrt(sum(np.sum(G[k] ** 2) for k in G))
    rows = sorted(((_relerr(Gd[k], G[k]), np.linalg.norm(Gd[k] - G[k]) / gnorm, np.linalg.norm(G[k]) / gnorm, k)
                   for k in G if np.linalg.norm(G[k]) > 1e-12), reverse=True)
    print('real-dims parity: cost rel err %.2e; global grad rel err %.2e' %
          (rel_cost, np.sqrt(sum(np.sum((Gd[k] - G[k]) ** 2) for k in G)) / gnorm))
    for r in rows[:8]:
        print('   rel %.2e  err/|g_all| %.2e  |g_k|/|g_all| %.2e  %s' % r)
    assert rel_cost <= 1e-4
    # per tensor: 1e-3 relative, except tensors whose gradient is a near-total cancellation (b_att, W_att: the softmax
    # backward terms sum to ~0 over the source positions) -- those are bounded against the global gradient norm
    for rel, err_g, share, k in rows:
        assert rel <= 1e-3 or err_g <= 1e-6, (k, rel, err_g)
    assert np.sqrt(sum(np.sum((Gd[k] - G[k]) ** 2) for k in G)) / gnorm <= 1e-4
