"""Filtered sampling on the device (nats.sample_many -> nats_sample_step_many -> sample_filter_kernel; an addition beyond
the reference) against the float64 rule of tests/sample_oracle.py, teacher-forced along the device's own words.

A draw is DECIDABLE when every boundary it depends on -- the top-k gap, the top-p cut mass and its neighbours' weights,
u*Z against the cumulative sums -- is more than MARGIN away (relative to the largest weight or to the kept total): then a
float32 evaluation whose probabilities are within MARGIN / 10 of float64 must pick the oracle's word (where two weights at
a cut are closer than the margin, every set the device could keep must give the same word).  MARGIN = 2e-5, and
BIG_MARGIN = 4e-5 for the V = 40000 model, whose sharper logits lose more to float32 (up to 2.9e-6 measured on an H100,
against 1.5e-7 for the toy models and 3e-7 at the headline size): test_margin_covers_f_next_error measures the device's
first-step probabilities of every model used here against float64 and requires max |p - p64| / p_max < margin / 10.
(The margin cannot be much larger: the share of undecidable draws grows with margin x the number of kept words,
2 x 2e-5 x 120 ~ 0.5 % for an unfiltered toy row.)  Every decidable draw must equal the oracle's, at least 99 % must be
decidable, costs match float64 within rtol 1e-5 (plus 1e-6 per word, for costs near 0) and attention rows within the
beam tests' tolerance.  Edge cases have tests of their own: float32 underflow of the weights at small T, exact ties at
the cuts across CTA slices, and a row forced to end because every word is banned."""
import ctypes
import itertools
import pickle

import numpy as np
import pytest

from oracle import nats_oracle as O
from tests import sample_oracle as SO
from tests.helpers import toy_options, toy_params
from tests.test_gpu_beam_many import _sources

pytestmark = pytest.mark.gpu

MARGIN = 2e-5
BIG_MARGIN = 4e-5

_M = {}


def _model(name):
    """'toy': D 32, W 8, A 12, V 120 (the beam tests' model); 'odd': V 121; 'big': V 40000, above the 32768 words a
    register-resident row would hold, with sharper logits so that the top-p cuts fall where the weights are distinct"""
    if name not in _M:
        from nats_b200 import nats
        V = dict(toy=120, odd=121, big=40000)[name]
        opts = toy_options(D=32, W=8, A=12, V=V)
        P32 = O.cast_params(toy_params(opts), 'float32')
        if name == 'big':
            P32['ff_logit_W'] = (P32['ff_logit_W'] * 20).astype('float32')
        tparams = nats.init_tparams(P32)
        f_init, f_next = nats.build_sampler(tparams, opts)
        _M[name] = (opts, P32, O.cast_params(P32, 'float64'), tparams, f_init, f_next)
    return _M[name]


def _check(res, xs, P64, kw, ids=None, margin=MARGIN):
    """every source's samples against the teacher-forced oracle -> (draws, decidable draws); ids: the sources' indices in
    the list sample_many drew them from (default 0, 1, ...), which fix their rows' ids"""
    R = kw['n_samples']
    n = ok = 0
    fk = dict((k_, kw[k_]) for k_ in ('temperature', 'top_k', 'top_p', 'use_unk', 'no_repeat_ngram', 'min_len', 'seed')
              if k_ in kw)
    for i, (x, (samples, costs, alphas)) in enumerate(zip(xs, res)):
        assert len(samples) == len(costs) == len(alphas) == R
        for s in samples:
            assert 1 <= len(s) <= kw['maxlen'] and 0 not in s[:-1]
        ref = SO.teacher_forced(P64, x, samples, kw['maxlen'], row_base=(i if ids is None else ids[i]) * R, margin=margin,
                                **fk)
        for j in range(R):
            for (ii, dev, word, dec) in ref['draws'][j]:
                n += 1
                if dec:
                    ok += 1
                    assert dev == word, (i, j, ii, dev, word, kw)
            np.testing.assert_allclose(float(costs[j]), ref['cost'][j], rtol=1e-5, atol=1e-6 * len(samples[j]))
            assert len(alphas[j]) == len(samples[j]) and all(len(a) == len(x) for a in alphas[j])
            np.testing.assert_allclose(np.array(alphas[j]), ref['alphas'][j], rtol=2e-4, atol=1e-6)
    return n, ok


# R, chunk and concurrency cycle through all their combinations along the filter grid
_LAYOUT = list(itertools.product([1, 7, 32], [1, 3, 16], [1, 2]))
_GRID = list(itertools.product([1., 0.7, 1.5], [0, 1, 5], [1., 0.9, 0.5]))


@pytest.mark.parametrize('model', ['toy', 'odd'])
@pytest.mark.parametrize('T,K,P', _GRID)
def test_exact_vs_float64(model, T, K, P):
    """the ten ragged sources of test_gpu_beam_many.py, maxlen 9, use_unk both ways, constraints off and (N 2, L 5)"""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model(model)
    xs = _sources(opts['n_words'])
    n = ok = 0
    for c, (use_unk, (N_, L)) in enumerate(itertools.product([True, False], [(0, 0), (2, 5)])):
        R, chunk, conc = _LAYOUT[(_GRID.index((T, K, P)) * 4 + c) % len(_LAYOUT)]
        kw = dict(n_samples=R, maxlen=9, temperature=T, top_k=K, top_p=P, use_unk=use_unk, no_repeat_ngram=N_, min_len=L,
                  seed=77)
        res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=chunk, concurrency=conc, **kw)
        dn, dok = _check(res, xs, P64, kw)
        n, ok = n + dn, ok + dok
    print('%s T=%g K=%d P=%g: %d of %d draws decidable' % (model, T, K, P, ok, n))
    assert ok >= 0.99 * n, (ok, n)


def test_exact_vs_float64_above_32768_words():
    """V = 40000: four sources, R = 7, two groups on two streams, constraints on; six filter settings, 99 % over all"""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model('big')
    xs = _sources(opts['n_words'], seed=5)[:4]
    n = ok = 0
    for T, K, P in [(0.7, 0, 1.), (0.7, 5, 0.9), (1.5, 1, 1.), (1., 0, 0.5), (0.7, 0, 0.9), (1.5, 5, 0.5)]:
        kw = dict(n_samples=7, maxlen=6, temperature=T, top_k=K, top_p=P, use_unk=False, no_repeat_ngram=2, min_len=3, seed=3)
        res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=2, concurrency=2, **kw)
        dn, dok = _check(res, xs, P64, kw, margin=BIG_MARGIN)
        print('big T=%g K=%d P=%g: %d of %d draws decidable' % (T, K, P, dok, dn))
        n, ok = n + dn, ok + dok
    assert ok >= 0.99 * n, (ok, n)


def test_margin_covers_f_next_error():
    """the device f_next's first-step probabilities of every model here, against float64: within margin / 10 of p_max"""
    import torch
    for name in ('toy', 'odd', 'big', 'head'):
        opts, P32, P64, tparams, f_init, f_next = _model(name) if name != 'head' else _headline()
        margin = BIG_MARGIN if name == 'big' else MARGIN
        for x in (_sources(opts['n_words'])[:4] if name != 'head' else _headline_sources()[:2]):
            s0, c0 = f_init(x[:, None])
            out = f_next(-np.ones((1,), 'int64'), c0, s0, np.zeros((1, 2 * opts['dim']), 'float32'),
                         np.zeros((1, len(x)), 'float32'))
            r0, rc = O.f_init(P64, x[:, None])
            ref = O.f_next(P64, -np.ones((1,), 'int64'), rc, r0, np.zeros((1, 2 * opts['dim'])), np.zeros((1, len(x))))[0]
            err = np.abs(np.asarray(out[0], dtype='float64') - ref).max() / ref.max()
            print('%s: max |p - p64| / p_max = %.2e' % (name, err))
            assert err < margin / 10, (name, err)
    torch.cuda.synchronize()


def test_greedy():
    """K = 1: all R samples of a source are identical and equal the oracle's argmax decoding where the top-2 gap is clear"""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model('toy')
    xs = _sources(120)
    kw = dict(n_samples=6, maxlen=9, temperature=0.7, top_k=1, top_p=1., use_unk=True, seed=5)
    res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=4, concurrency=2, **kw)
    for samples, costs, _ in res:
        assert all(s == samples[0] for s in samples) and len(set(float(c) for c in costs)) == 1
    n, ok = _check(res, xs, P64, kw)
    assert ok >= 0.99 * n, (ok, n)


def _filtered_first_word(P64, x, T, K, P):
    r0, rc = O.f_init(P64, x[:, None])
    p = O.f_next(P64, -np.ones((1,), 'int64'), rc, r0, np.zeros((1, rc.shape[2])), np.zeros((1, len(x))))[0][0]
    w = SO.weights(p, T)
    keep = SO.kept(w, K, P)
    q = np.zeros_like(w)
    q[keep] = w[keep]
    return q / q.sum()


@pytest.mark.parametrize('T,K,P', [(1., 0, 1.), (0.5, 20, 0.8)])
def test_first_word_distribution(T, K, P):
    """one source, R = 8192, maxlen = 1: a chi-square test of the first word against the filtered float64 distribution
    (bins of expected count < 5 pooled) gives p > 1e-3 at the fixed seed, and no draw falls outside the support"""
    from scipy import stats
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model('toy')
    x = _sources(120)[5]
    R = 8192
    res = nats.sample_many(tparams, f_init, f_next, [x], opts, n_samples=R, maxlen=1, temperature=T, top_k=K, top_p=P,
                           seed=2024, chunk=1)
    words = np.array([s[0] for s in res[0][0]])
    q = _filtered_first_word(P64, x, T, K, P)
    assert np.all(q[words] > 0), sorted(set(words[q[words] == 0]))
    counts = np.bincount(words, minlength=len(q)).astype('float64')
    exp = q * R
    big = exp >= 5
    obs_b, exp_b = list(counts[big]), list(exp[big])
    if (~big & (q > 0)).any():
        obs_b.append(counts[~big].sum())
        exp_b.append(exp[~big].sum())
    chi = stats.chisquare(obs_b, exp_b)
    print('T=%g K=%d P=%g: support %d, chi2 %.1f, p = %.3g' % (T, K, P, int((q > 0).sum()), chi.statistic, chi.pvalue))
    assert chi.pvalue > 1e-3


def test_determinism_and_independence():
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model('toy')
    xs = _sources(120)
    kw = dict(n_samples=7, maxlen=9, temperature=0.7, top_k=5, top_p=0.9, no_repeat_ngram=2, min_len=2, seed=9)
    a = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=3, concurrency=2, **kw)
    b = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=3, concurrency=2, **kw)
    for (s1, c1, a1), (s2, c2, a2) in zip(a, b):               # the same call twice: the same bits
        assert s1 == s2
        assert np.array_equal(np.array(c1), np.array(c2))
        assert all(np.array_equal(np.array(h1), np.array(h2)) for h1, h2 in zip(a1, a2))
    for chunk, conc in ((1, 1), (16, 1), (4, 3)):               # tokens do not depend on the grouping
        c = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=chunk, concurrency=conc, **kw)
        assert [r[0] for r in c] == [r[0] for r in a], (chunk, conc)
    # a source's samples do not depend on its neighbours: sources 4..6 alone, with index_base = 4, and among others
    alone = nats.sample_many(tparams, f_init, f_next, xs[4:7], opts, index_base=4, chunk=16, **kw)
    assert [r[0] for r in alone] == [r[0] for r in a[4:7]]
    other = _sources(120, seed=99)
    mixed = nats.sample_many(tparams, f_init, f_next, other[:4] + xs[4:7] + other[4:], opts, chunk=16, **kw)
    assert [r[0] for r in mixed[4:7]] == [r[0] for r in a[4:7]]
    d = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=3, concurrency=2, **dict(kw, seed=10))
    assert [r[0] for r in d] != [r[0] for r in a]


def _ngrams(seq, n):
    return [tuple(seq[i:i + n]) for i in range(len(seq) - n + 1)]


def test_bans():
    """no repeated N-gram, no EOS before L words, no UNK with use_unk=False -- on a model that prefers all three"""
    from nats_b200 import nats
    opts = toy_options(D=32, W=8, A=12, V=30)
    P32 = O.cast_params(toy_params(opts), 'float32')
    P32['ff_logit_b'][0] += 2.
    P32['ff_logit_b'][1] += 2.
    tparams = nats.init_tparams(P32)
    f_init, f_next = nats.build_sampler(tparams, opts)
    xs = _sources(30)
    for N_, L in ((1, 6), (2, 4), (3, 0)):
        res = nats.sample_many(tparams, f_init, f_next, xs, opts, n_samples=16, maxlen=12, use_unk=False, no_repeat_ngram=N_,
                               min_len=L, temperature=1.5, seed=N_)
        for samples, costs, _ in res:
            assert np.all(np.isfinite(np.array(costs, 'float64')))
            for s in samples:
                body = s[:-1] if s[-1] == 0 else s
                assert 1 not in s and 0 not in body
                assert len(_ngrams(body, N_)) == len(set(_ngrams(body, N_))), (s, N_)
                if s[-1] == 0:
                    assert len(s) >= L + 1, (s, L)
    free = nats.sample_many(tparams, f_init, f_next, xs, opts, n_samples=16, maxlen=12, temperature=1.5, seed=1)
    assert any(s[-1] == 0 and len(s) < 5 for samples, _, _ in free for s in samples)   # the bans changed something
    assert any(1 in s for samples, _, _ in free for s in samples)


def _headline():
    """D 1000, W = A = 100, V 30000 (the recipe of test_gpu_beam_many.py's headline test)"""
    if 'head' in _M:
        return _M['head']
    from nats_b200 import nats
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
    P32 = O.cast_params(P32, 'float32')
    tparams = nats.init_tparams(P32)
    f_init, f_next = nats.build_sampler(tparams, opts)
    _M['head'] = (opts, P32, O.cast_params(P32, 'float64'), tparams, f_init, f_next)
    return _M['head']


def _headline_sources():
    rs = np.random.RandomState(12)
    return [np.concatenate([rs.randint(2, 30000, size=L), [0]]).astype('int64') for L in rs.randint(100, 400, size=16)]


def test_headline_size():
    """16 sources of 100-400 words, R 10, 10 steps, T 0.8, K 50, P 0.95 at the headline size (_headline); the
    teacher-forced oracle covers two sources and all their rows"""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _headline()
    xs = _headline_sources()
    kw = dict(n_samples=10, maxlen=10, temperature=0.8, top_k=50, top_p=0.95, seed=4)
    res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=16, concurrency=1, **kw)
    assert len(res) == 16
    pick = [0, 9]
    n, ok = _check([res[i] for i in pick], [xs[i] for i in pick], P64, kw, ids=pick)
    print('headline: %d of %d draws decidable' % (ok, n))
    assert ok >= 0.99 * n, (ok, n)


def test_errors():
    """each invalid input is refused by nats_sample_step_many (non-zero, with a message) and by sample_many (ValueError)"""
    import torch
    from nats_b200 import _lib, nats
    opts, P32, P64, tparams, f_init, f_next = _model('toy')
    eng = f_next.engine
    dims = _lib.Dims(opts['n_words'], opts['dim_word'], opts['dim'], opts['dim_att'])
    good = dict(n_src=1, n_samples=3, Tx=4, maxlen=6, temperature=1., top_k=0, top_p=1.)
    bad = [(dict(temperature=0.), 'temperature'), (dict(temperature=-1.), 'temperature'),
           (dict(temperature=float('nan')), 'temperature'), (dict(top_k=-1), 'top_k'), (dict(top_p=0.), 'top_p'),
           (dict(top_p=1.5), 'top_p'), (dict(top_p=float('nan')), 'top_p'), (dict(n_samples=0), 'n_samples'),
           (dict(n_src=300, n_samples=300), 'group size'), (dict(no_repeat_ngram=-1), 'no_repeat_ngram'),
           (dict(min_len=-1), 'no_repeat_ngram'), (dict(min_len=2, maxlen=12289), 'maxlen <= 12288')]
    for change, msg in bad:
        m = _lib.SampleStepMany()
        for k_, v in dict(good, **change).items():
            setattr(m, k_, v)
        rc = eng.lib.nats_sample_step_many(eng.ctx, eng.stream(), ctypes.byref(dims), ctypes.byref(m), 0)
        assert rc != 0, change
        with pytest.raises(_lib.NatsB200Error, match=msg):
            _lib.check(rc, 'nats_sample_step_many')
        kw = dict(n_samples=change.get('n_samples', 3), temperature=change.get('temperature', 1.), top_k=change.get('top_k', 0),
                  top_p=change.get('top_p', 1.), no_repeat_ngram=change.get('no_repeat_ngram', 0),
                  min_len=change.get('min_len', 0), maxlen=change.get('maxlen', 6), chunk=change.get('n_src', 1))
        with pytest.raises(ValueError):
            nats.sample_many(tparams, f_init, f_next, _sources(120)[:1], opts, **kw)
    torch.cuda.synchronize()


def _toy_checkpoint(tmp_path, V=40, seed=5):
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
        for _ in range(40):
            f.write(' '.join(rng.choice(words, size=rng.randint(3, 20))) + '\n')
    return model, dic, src


def test_gen_twin_end_to_end(tmp_path):
    """gen --sample 5 --top-p 0.9 (-n) writes the same file in-process (-p 1) and in two worker processes (-p 2): 40 lines,
    three chunks, the draws keyed by each line's position"""
    from nats_b200 import gen
    model, dic, src = _toy_checkpoint(tmp_path)
    outs = []
    for p in (1, 2):
        out = str(tmp_path / ('gen_p%d.txt' % p))
        gen.main(model, dic, src, out, normalize=True, n_process=p, sample=5, top_p=0.9, no_repeat_ngram=3, min_len=2)
        lines = open(out).read().split('\n')[:40]
        assert len(lines) == 40
        for line in lines:
            toks = line.split()
            assert all(w.startswith('w') or w == 'UNK' for w in toks[0::2]) and all(q.startswith('[') for q in toks[1::2])
        outs.append(open(out).read())
    assert outs[0] == outs[1]
    other = str(tmp_path / 'gen_seed.txt')
    gen.main(model, dic, src, other, normalize=True, n_process=1, sample=5, top_p=0.9, seed=99, no_repeat_ngram=3, min_len=2)
    assert open(other).read() != outs[0]


@pytest.mark.parametrize('T,K,P', [(0.05, 50, 1.), (0.05, 50, 0.9), (0.1, 5000, 1.)])
def test_small_temperature_underflow(T, K, P):
    """At small T the float32 power (p / p_max)^(1/T) underflows to 0 for all but a few words of the peaked V = 40000
    model, so fewer words carry weight than top_k asks for: every word of positive weight is then kept.  The rows must
    really reach that case (checked on the float32 weights of the first step), and the draws match the oracle, whose
    float64 weights of the underflowed words are too small to change a decidable draw."""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next = _model('big')
    xs = _sources(opts['n_words'], seed=5)[:4]
    short = 0
    for x in xs:
        r0, rc = O.f_init(P64, x[:, None])
        p = O.f_next(P64, -np.ones((1,), 'int64'), rc, r0, np.zeros((1, rc.shape[2])), np.zeros((1, len(x))))[0][0]
        w32 = np.power((p / p.max()).astype('float32'), np.float32(1. / T))
        short += int(np.count_nonzero(w32) < K)
    assert short >= 1, 'no row has fewer than top_k words of positive float32 weight'
    kw = dict(n_samples=7, maxlen=6, temperature=T, top_k=K, top_p=P, seed=21)
    res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=2, concurrency=2, **kw)
    n, ok = _check(res, xs, P64, kw, margin=BIG_MARGIN)
    print('big T=%g K=%d P=%g: %d rows of %d short of K, %d of %d draws decidable' % (T, K, P, short, len(xs), ok, n))
    assert ok >= 0.99 * n, (ok, n)


def _tied_model():
    """V = 40000 whose logit columns repeat with period 64 (column j = column j % 64, likewise the bias), so every
    probability occurs 625 times, EXACTLY: the 8 CTA slices of 5000 words each hold copies of all 64 values, and the copies
    of one value cut by top-k or top-p straddle slice boundaries"""
    if 'tied' not in _M:
        from nats_b200 import nats
        opts = toy_options(D=32, W=8, A=12, V=40000)
        P32 = O.cast_params(toy_params(opts), 'float32')
        cls = np.arange(40000) % 64
        P32['ff_logit_W'] = np.ascontiguousarray((P32['ff_logit_W'][:, :64] * 6)[:, cls]).astype('float32')
        P32['ff_logit_b'] = np.ascontiguousarray(P32['ff_logit_b'][:64][cls]).astype('float32')
        tparams = nats.init_tparams(P32)
        f_init, f_next = nats.build_sampler(tparams, opts)
        _M['tied'] = (opts, P32, O.cast_params(P32, 'float64'), tparams, f_init, f_next, cls)
    return _M['tied']


@pytest.mark.parametrize('T,K,P', [(1., 100, 1.), (0.7, 1000, 1.), (1., 0, 0.3), (1., 0, 0.7), (0.7, 3000, 0.5)])
def test_exact_ties_across_slices(T, K, P):
    """Ties at the cut are kept in index order: K = 100 takes the first 100 copies of the top value (words c + 64 t,
    t < 100: up to index 6400, across the first slice boundary), K = 1000 / 3000 cut inside later values, and top-p cuts
    inside a class.  The first word of R = 64 rows per source is checked against the rule applied to the device's own
    float32 probabilities of that step (f_next on the same R rows, exactly tied within a class), so float64 rounding of
    the weights is the only slack: margin 1e-6, ties resolved by index on both sides."""
    from nats_b200 import nats
    opts, P32, P64, tparams, f_init, f_next, cls = _tied_model()
    xs = _sources(opts['n_words'], seed=8)[:3]
    R, seed = 64, 13
    res = nats.sample_many(tparams, f_init, f_next, xs, opts, n_samples=R, maxlen=1, temperature=T, top_k=K, top_p=P,
                           seed=seed, chunk=3)
    n = ok = 0
    for i, (x, (samples, _, _)) in enumerate(zip(xs, res)):
        s0, c0 = f_init(x[:, None])
        pd = np.asarray(f_next(-np.ones((R,), 'int64'), np.tile(c0, [R, 1]), np.tile(s0, [R, 1]),
                               np.zeros((R, 2 * opts['dim']), 'float32'), np.zeros((R, len(x)), 'float32'))[0])[0]
        assert np.array_equal(pd, pd[cls]), 'probabilities of one class differ on the device'
        u = SO.uniform01(seed, 0, np.arange(R, dtype=np.uint64) + np.uint64(i * R))
        for j in range(R):
            word, dec = SO.decide(pd.astype('float64'), T, K, P, [], u[j], 1e-6, exact_ties=True)
            n += 1
            if dec:
                ok += 1
                assert samples[j] == [word], (i, j, samples[j], word)
    words = [s[0] for _, (samples, _, _) in zip(xs, res) for s in samples]
    print('ties T=%g K=%d P=%g: %d of %d draws decidable, first words up to %d' % (T, K, P, ok, n, max(words)))
    assert ok >= 0.99 * n, (ok, n)


def test_forced_end_pays_the_unfiltered_eos_probability():
    """V = 4 (EOS, UNK and two words), use_unk=False, no_repeat_ngram = 1, min_len = 5: after both words every word is
    banned, EOS included, so the row ends with word 0 at step 2, and its cost term is -log of the f_next probability of
    EOS, finite, as the oracle's"""
    from nats_b200 import nats
    opts = toy_options(D=16, W=8, A=6, V=4)
    P32 = O.cast_params(toy_params(opts), 'float32')
    tparams = nats.init_tparams(P32)
    f_init, f_next = nats.build_sampler(tparams, opts)
    xs = _sources(4, seed=2)[:3]
    kw = dict(n_samples=5, maxlen=6, use_unk=False, no_repeat_ngram=1, min_len=5, seed=6)
    res = nats.sample_many(tparams, f_init, f_next, xs, opts, chunk=2, **kw)
    for samples, costs, _ in res:
        assert all(sorted(s[:2]) == [2, 3] and s[2:] == [0] for s in samples), samples
        assert np.all(np.isfinite(np.array(costs, 'float64')))
    n, ok = _check(res, xs, O.cast_params(P32, 'float64'), kw)
    assert ok == n
