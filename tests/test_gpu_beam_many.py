"""Beam search over a GROUP of source sentences (nats_beam_step_many through gen_sample_many): one device step advances the
beams of every sentence of the group, and every sentence must get what its own gen_sample returns (identical tokens,
scores and attention histories within rtol 2e-4, the tolerances of test_gen_sample_many_equals_sentence_by_sentence) and
what the float64 oracle's literal restatement of nats.py:879-1076 returns (identical tokens, scores within rtol 5e-4)."""
import ctypes
import os

import numpy as np
import pytest

from oracle import nats_oracle as O
from tests.helpers import toy_options, toy_params

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# ten ragged sources (EOS included): lengths 1, 6, 10, 10, 4, 15, 3, 21, 8, 12 -- a source of one word and two equal lengths
WORDS = (0, 5, 9, 9, 3, 14, 2, 20, 7, 11)


@pytest.fixture(scope='module')
def N():
    from nats_b200 import nats
    return nats


def _sources(V, seed=31, words=WORDS):
    rs = np.random.RandomState(seed)
    return [np.concatenate([rs.randint(2, V, size=L), [0]]).astype('int64') for L in words]


def _same(one, many, xs, rtol=2e-4):
    """sentence by sentence: tokens identical, scores and attention histories close, alpha rows of the source's length"""
    assert len(many) == len(one) == len(xs)
    for i, ((s1, c1, a1), (s2, c2, a2), x) in enumerate(zip(one, many, xs)):
        assert [list(map(int, s)) for s in s2] == [list(map(int, s)) for s in s1], i
        np.testing.assert_allclose(np.array(c2, 'float64'), np.array(c1, 'float64'), rtol=rtol)
        assert len(a2) == len(s2)
        for h1, h2, s in zip(a1, a2, s2):
            assert len(h2) == len(s) and all(len(row) == len(x) for row in h2), i
            np.testing.assert_allclose(np.array(h2), np.array(h1), rtol=rtol, atol=1e-6)


_TOY = {}


def _toy(N):
    if 'model' not in _TOY:
        opts = toy_options(D=32, W=8, A=12, V=120)
        P32 = O.cast_params(toy_params(opts), 'float32')
        tparams = N.init_tparams(P32)
        _TOY['model'] = (opts, P32, tparams) + tuple(N.build_sampler(tparams, opts))
    return _TOY['model']


@pytest.mark.parametrize('concurrency', [1, 2])
@pytest.mark.parametrize('chunk', [1, 3, 16])
@pytest.mark.parametrize('use_unk', [True, False])
@pytest.mark.parametrize('lam', [0.0, 0.5])
@pytest.mark.parametrize('k', [1, 6, 17, 32])
def test_group_equals_sentence_by_sentence(N, k, lam, use_unk, chunk, concurrency):
    """k = 17 takes the column-slice context kernel (more than 16 rows per source), 32 is the cap; chunk = 1 is a group of
    one (the single-sentence search), 16 puts all ten sentences in one group."""
    opts, P32, tparams, f_init, f_next = _toy(N)
    xs = _sources(120)
    kw = dict(k=k, maxlen=9, use_unk=use_unk, kl_factor=lam, ctx_factor=lam, state_factor=lam)
    key = (k, lam, use_unk)
    if key not in _TOY:                                  # each sentence's own search, shared by the chunk / concurrency cases
        _TOY[key] = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=concurrency, chunk=chunk, **kw)
    _same(_TOY[key], many, xs)


def _eos_bias(P32, delta):
    P = O.OrderedDict((kk, v.copy()) for kk, v in P32.items())
    P['ff_logit_b'][0] += delta
    return P


def test_uneven_retirement_within_a_group(N):
    """With the end-of-sentence logit raised by 1, some sentences of the group retire every hypothesis within a few steps
    while others still have live rows at maxlen: the finished ones stay untouched while the group goes on."""
    opts = toy_options(D=32, W=8, A=12, V=120)
    P32 = _eos_bias(O.cast_params(toy_params(opts), 'float32'), 1.0)
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    xs = _sources(120)
    k, maxlen = 3, 10
    kw = dict(k=k, maxlen=maxlen, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1, chunk=len(xs), **kw)
    early = [i for i, (s, _, _) in enumerate(many)
             if len(s) == k and all(q[-1] == 0 for q in s) and max(len(q) for q in s) < maxlen]
    at_max = [i for i, (s, _, _) in enumerate(many) if any(len(q) == maxlen and q[-1] != 0 for q in s)]
    assert early and at_max, (early, at_max)
    one = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
    _same(one, many, xs)


@pytest.mark.parametrize('model', ['golden', 'w8'])
def test_group_vs_oracle(N, model):
    """Each sentence of one group against the oracle's gen_sample (nats.py:879-1076) driven by the float64 f_init / f_next.
    'golden' has dim_word = 6 (the narrow readout projection is not eligible), 'w8' dim_word = 8."""
    if model == 'golden':
        zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
        V, W, D, A = [int(v) for v in zt['opt_dims']]
        opts = toy_options(D=D, W=W, A=A, V=V)
        names = list(O.init_params(opts).keys())
        P32 = O.cast_params(O.OrderedDict((kk, zt['p_' + kk]) for kk in names), 'float32')
    else:
        opts = toy_options(D=32, W=8, A=12, V=120)
        P32 = O.cast_params(toy_params(opts), 'float32')
    V = opts['n_words']
    tparams = N.init_tparams(P32)
    f_init, f_next = N.build_sampler(tparams, opts)
    xs = _sources(V, seed=11)
    fi = lambda x_: O.f_init(P32, x_)
    fn = lambda y_, c_, s_, ac_, aa_: O.f_next(P32, y_, c_, s_.astype('float32'), ac_.astype('float32'),
                                               aa_.astype('float32'))
    kw = dict(k=5, maxlen=8, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1, chunk=len(xs), **kw)
    for x, (gs, gsc, _) in zip(xs, many):
        rs_, rsc, _ = O.gen_sample(fi, fn, x[:, None], stochastic=False, **kw)
        assert [list(map(int, s)) for s in gs] == [list(map(int, s)) for s in rs_]
        np.testing.assert_allclose(np.array(gsc, 'float64'), np.array(rsc, 'float64'), rtol=5e-4)


def test_group_at_headline_dims(N):
    """D = 1000, W = A = 100, V = 30000 (the parameter recipe of test_gpu_headline.py): sources of 800, 433, 120 and 17
    words in one group, k = 10, 8 steps, all three penalties at 1 -- each sentence as its own device gen_sample."""
    opts = dict(dim_word=100, dim=1000, dim_att=100, n_words=30000, encoder='gru', decoder='gru_cond')
    np.random.seed(2024)
    P32 = O.init_params(opts)
    rng = np.random.RandomState(7)
    for kk in P32:
        if P32[kk].ndim == 1:
            P32[kk] = (0.05 * rng.randn(*P32[kk].shape)).astype('float32')
    P32['ff_logit_W'] = (P32['ff_logit_W'] * 40).astype('float32')
    P32['decoder_U_att'] = (P32['decoder_U_att'] * 30).astype('float32')
    P32['Wemb'] = (P32['Wemb'] * 10).astype('float32')
    tparams = N.init_tparams(O.cast_params(P32, 'float32'))
    f_init, f_next = N.build_sampler(tparams, opts)
    xs = _sources(30000, seed=3, words=(799, 432, 119, 16))
    kw = dict(k=10, maxlen=8, use_unk=True, kl_factor=1.0, ctx_factor=1.0, state_factor=1.0)
    one = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1, chunk=4, **kw)
    _same(one, many, xs)


def test_step_many_rejects_bad_shapes(N):
    """Host-side checks: a beam wider than 32 and an empty group are errors, before anything is launched."""
    import torch
    from nats_b200 import _lib
    opts, P32, tparams, f_init, f_next = _toy(N)
    eng = f_next.engine
    src_len = torch.ones(1, dtype=torch.int32, device=eng.device)
    dims = _lib.Dims(opts['n_words'], opts['dim_word'], opts['dim'], opts['dim_att'])
    for k, n_src in ((33, 1), (5, 0)):
        m = _lib.BeamStepMany()
        m.n_src, m.src_len = n_src, src_len.data_ptr()
        m.beam.Tx, m.beam.k, m.beam.maxlen = 4, k, 6
        rc = eng.lib.nats_beam_step_many(eng.ctx, eng.stream(), ctypes.byref(dims), ctypes.byref(m), 0)
        with pytest.raises(_lib.NatsB200Error):
            _lib.check(rc, 'nats_beam_step_many')
    torch.cuda.synchronize()
