"""Beam-search output constraints on the device (no_repeat_ngram, min_len; additions beyond the reference): the grouped
device search (gen_sample_many -> nats_beam_step_many -> beam_constrain_kernel) must return, sentence by sentence, what the
host loop (NATS_DEVICE_BEAM=0: full-vocabulary branch, bans computed on the host) returns -- identical tokens, scores and
attention histories within the tolerances of test_gpu_beam_many.py -- and what the float64 oracle returns (identical
tokens, scores within rtol 5e-4).  Every case keeps >= k admissible words in every live row, and asserts it."""
import ctypes
import os
import pickle

import numpy as np
import pytest

from oracle import nats_oracle as O
from tests import constrained_beam_oracle as CO
from tests.helpers import toy_options, toy_params
from tests.test_gpu_beam_many import _same, _sources

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@pytest.fixture(scope='module')
def N():
    from nats_b200 import nats
    return nats


def _ngrams(seq, n):
    return [tuple(seq[i:i + n]) for i in range(len(seq) - n + 1)]


def _check_output(res, N_, L, k, maxlen):
    """no hypothesis repeats an N-gram, every retired one has >= L words before EOS, no +inf cost was selected"""
    for samples, scores, _ in res:
        assert 1 <= len(samples) <= k
        assert np.all(np.isfinite(np.array(scores, 'float64'))), scores
        for s in samples:
            s = [int(w) for w in s]
            body = s[:-1] if s[-1] == 0 else s
            assert 0 not in body and len(s) <= maxlen
            if N_ >= 1:
                assert len(_ngrams(body, N_)) == len(set(_ngrams(body, N_))), (s, N_)
            if s[-1] == 0:
                assert len(s) >= L + 1, (s, L)


def _admissible(V, k, maxlen):
    """a live row bans at most its maxlen - 1 history words and EOS; UNK (1e-20 when use_unk=False) is not counted"""
    assert V - 2 - (maxlen - 1) - 1 >= k, (V, k, maxlen)


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
@pytest.mark.parametrize('L', [0, 5])
@pytest.mark.parametrize('N_', [2, 3])
@pytest.mark.parametrize('k', [1, 6, 17, 32])
def test_group_equals_host_loop(N, monkeypatch, k, N_, L, lam, use_unk, chunk, concurrency):
    """the ten ragged sources of test_gpu_beam_many.py; k = 17 takes the column-slice context kernel, 32 is the cap,
    chunk = 1 is a group of one, 16 puts all ten sentences in one group"""
    opts, P32, tparams, f_init, f_next = _toy(N)
    xs = _sources(120)
    maxlen = 9
    _admissible(120, k, maxlen)
    kw = dict(k=k, maxlen=maxlen, use_unk=use_unk, kl_factor=lam, ctx_factor=lam, state_factor=lam, no_repeat_ngram=N_,
              min_len=L)
    key = (k, N_, L, lam, use_unk)
    if key not in _TOY:                       # the host loop, once per key, shared by the chunk / concurrency cases
        with monkeypatch.context() as mp:
            mp.setenv('NATS_DEVICE_BEAM', '0')
            _TOY[key] = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
        _check_output(_TOY[key], N_, L, k, maxlen)
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=concurrency, chunk=chunk, **kw)
    _same(_TOY[key], many, xs)


@pytest.mark.parametrize('model', ['golden', 'w8'])
def test_group_vs_oracle(N, model):
    """each sentence of one group against the float64 oracle's constrained search ('golden': dim_word 6, V 50; 'w8':
    dim_word 8, V 120)"""
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
    k, maxlen = 5, 8
    _admissible(V, k, maxlen)
    for N_, L in ((2, 4), (3, 0), (0, 6)):
        kw = dict(k=k, maxlen=maxlen, use_unk=True, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5, no_repeat_ngram=N_,
                  min_len=L)
        many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1, chunk=len(xs), **kw)
        _check_output(many, N_, L, k, maxlen)
        for x, (gs, gsc, _) in zip(xs, many):
            rs_, rsc, _ = CO.gen_sample(fi, fn, x[:, None], **kw)
            assert [list(map(int, s)) for s in gs] == [list(map(int, s)) for s in rs_]
            np.testing.assert_allclose(np.array(gsc, 'float64'), np.array(rsc, 'float64'), rtol=5e-4)


def test_group_at_headline_dims(N):
    """D = 1000, W = A = 100, V = 30000 (the parameter recipe of test_group_at_headline_dims in test_gpu_beam_many.py):
    sources of 800, 433, 120 and 17 words in one group, k = 10, all three penalties at 1, N = 3, min_len = 6 -- each
    sentence as its own device gen_sample"""
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
    k, maxlen = 10, 10
    _admissible(30000, k, maxlen)
    kw = dict(k=k, maxlen=maxlen, use_unk=True, kl_factor=1.0, ctx_factor=1.0, state_factor=1.0, no_repeat_ngram=3, min_len=6)
    one = [N.gen_sample(tparams, f_init, f_next, x[:, None], opts, stochastic=False, **kw) for x in xs]
    many = N.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1, chunk=4, **kw)
    _same(one, many, xs)
    _check_output(many, 3, 6, k, maxlen)


def test_errors(N):
    """negative constraints are refused by nats_beam_step_many before anything is launched; the host rejects constraints
    on stochastic sampling and on the five-call step trace"""
    import torch
    from nats_b200 import _lib
    opts, P32, tparams, f_init, f_next = _toy(N)
    eng = f_next.engine
    src_len = torch.ones(1, dtype=torch.int32, device=eng.device)
    dims = _lib.Dims(opts['n_words'], opts['dim_word'], opts['dim'], opts['dim_att'])
    for nr, ml in ((-1, 0), (0, -1), (-3, 4)):
        m = _lib.BeamStepMany()
        m.n_src, m.src_len = 1, src_len.data_ptr()
        m.no_repeat_ngram, m.min_len = nr, ml
        m.beam.Tx, m.beam.k, m.beam.maxlen = 4, 5, 6
        rc = eng.lib.nats_beam_step_many(eng.ctx, eng.stream(), ctypes.byref(dims), ctypes.byref(m), 0)
        with pytest.raises(_lib.NatsB200Error, match='no_repeat_ngram and min_len'):
            _lib.check(rc, 'nats_beam_step_many')
    torch.cuda.synchronize()
    x = _sources(120)[5][:, None]
    for kw in (dict(no_repeat_ngram=2), dict(min_len=3)):
        with pytest.raises(ValueError):
            N.gen_sample(tparams, f_init, f_next, x, opts, k=1, stochastic=True, **kw)
        with pytest.raises(ValueError):
            N.gen_sample(tparams, f_init, f_next, x, opts, k=3, stochastic=False, _trace=[], **kw)
    with pytest.raises(ValueError):
        N.gen_sample_many(tparams, f_init, f_next, [x[:, 0]], opts, k=3, no_repeat_ngram=-1)
    # the five-call trace still runs when both are 0
    tr = []
    N.gen_sample(tparams, f_init, f_next, x, opts, k=3, maxlen=4, stochastic=False, kl_factor=0.5, _trace=tr,
                 no_repeat_ngram=0, min_len=0)
    assert tr


def _toy_checkpoint(tmp_path, V=40, seed=5):
    """a random model (no training) in the reference's checkpoint layout, a dictionary of V - 2 distinct words and a
    source file of twelve lines"""
    opts = dict(dim_word=8, dim=16, dim_att=6, n_words=V, encoder='gru', decoder='gru_cond')
    P = toy_params(opts, seed=seed, dtype='float32')
    model = str(tmp_path / 'toy.npz')
    np.savez(model, **P)
    with open(model + '.pkl', 'wb') as f:
        pickle.dump(opts, f, protocol=2)
    words = ['w%02d' % i for i in range(2, V)]
    dic = str(tmp_path / 'dict.pkl')
    with open(dic, 'wb') as f:
        pickle.dump(dict([('eos', 0), ('UNK', 1)] + [(w, i + 2) for i, w in enumerate(words)]), f, protocol=2)
    rng = np.random.RandomState(seed)
    src = str(tmp_path / 'src.txt')
    with open(src, 'w') as f:
        for _ in range(12):
            f.write(' '.join(rng.choice(words, size=rng.randint(3, 20))) + '\n')
    return model, dic, src


def test_gen_twin_end_to_end(N, tmp_path):
    """nats_b200.gen with --no-repeat-ngram 3 --min-len 4, in-process (-p 1) and in two worker processes (-p 2): every
    line is free of repeated trigrams and, when it ended in EOS (fewer than gen's maxlen = 100 words), has >= 4 words"""
    from nats_b200 import gen
    model, dic, src = _toy_checkpoint(tmp_path)
    outs = []
    for p in (1, 2):
        out = str(tmp_path / ('gen_p%d.txt' % p))
        gen.main(model, dic, src, out, k=5, normalize=True, n_process=p, no_repeat_ngram=3, min_len=4)
        lines = open(out).read().split('\n')[:12]
        assert len(lines) == 12
        for line in lines:
            toks = line.split()
            words = toks[0::2]
            assert all(w.startswith('w') or w == 'UNK' for w in words) and all(q.startswith('[') for q in toks[1::2])
            assert len(_ngrams(words, 3)) == len(set(_ngrams(words, 3))), line
            assert len(words) <= 100 and (len(words) == 100 or len(words) >= 4), line
        outs.append(open(out).read())
    assert outs[0] == outs[1]
    with pytest.raises(ValueError):
        gen.main(model, dic, src, str(tmp_path / 'bad.txt'), k=5, n_process=1, min_len=-1)
