"""CPU tests of the beam-search output constraints (no_repeat_ngram, min_len; additions beyond the reference) on the float64
oracle: the banned-word rule against brute force, the properties every returned hypothesis must have, that the
constraints change what an unconstrained search returns, and that the host loop of nats_b200.nats.gen_sample (driven by
oracle callables) applies them exactly as the oracle does."""
import itertools
import os

import numpy as np
import pytest

from nats_b200 import nats as N
from oracle import nats_oracle as O
from tests import constrained_beam_oracle as CO
from tests.helpers import toy_options, toy_params

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _callables(P):
    dt = P['Wemb'].dtype
    fi = lambda x: O.f_init(P, x)
    fn = lambda y, ctx, s, ac, aa: O.f_next(P, y, np.asarray(ctx), s.astype(dt), ac.astype(dt), aa.astype(dt))
    return fi, fn


def _golden():
    zt = np.load(os.path.join(GOLD, 'train_toy.npz'))
    V, W, D, A = [int(v) for v in zt['opt_dims']]
    opts = toy_options(D=D, W=W, A=A, V=V)
    names = list(O.init_params(opts).keys())
    return opts, O.OrderedDict((kk, zt['p_' + kk].astype('float64')) for kk in names)


def _ngrams(seq, n):
    return [tuple(seq[i:i + n]) for i in range(len(seq) - n + 1)]


def _brute_banned(hyp, N_, L):
    """every word w such that hyp + [w] would contain some N-gram twice (EOS aside), and EOS while len(hyp) < L"""
    out = set()
    if len(hyp) < L:
        out.add(0)
    if N_ >= 1:
        for w in set(hyp):
            grams = _ngrams(list(hyp) + [w], N_)
            if len(grams) != len(set(grams)):
                out.add(w)
    return out


def test_banned_words_match_brute_force():
    """random histories over a small alphabet (many repeats), lengths 0..12 (including shorter than N - 1), N = 1..4; the
    host loop's rule (nats._banned_words) and the oracle's are the same set"""
    rng = np.random.RandomState(5)
    n_cases = 0
    for _ in range(400):
        ii = rng.randint(0, 13)
        hyp = [int(w) for w in rng.randint(2, 6, size=ii)]
        for N_, L in itertools.product((0, 1, 2, 3, 4), (0, 3, 7)):
            # a history that itself repeats no N-gram (as every live hypothesis of a constrained search) keeps the
            # brute-force reading exact; longer repeats are still compared between the two implementations
            want = CO.banned_words(hyp, N_, L)
            assert set(N._banned_words(hyp, N_, L)) == want, (hyp, N_, L)
            if N_ == 0 or len(_ngrams(hyp, N_)) == len(set(_ngrams(hyp, N_))):
                assert want == _brute_banned(hyp, N_, L), (hyp, N_, L)
                n_cases += 1
    assert n_cases > 2000
    assert CO.banned_words([5, 6, 5], 2, 0) == {6}
    assert CO.banned_words([5, 6, 5, 6], 3, 0) == {5}
    assert CO.banned_words([7, 8, 7], 1, 0) == {7, 8}
    assert CO.banned_words([4], 3, 2) == {0}                # shorter than N - 1: only the length rule


def _check_output(samples, scores, N_, L, k, maxlen):
    assert 1 <= len(samples) <= k and len(scores) == len(samples)
    assert np.all(np.isfinite(np.array(scores, 'float64'))), scores      # no +inf candidate was ever selected
    for s in samples:
        s = [int(w) for w in s]
        body = s[:-1] if s[-1] == 0 else s
        assert 0 not in body and len(s) <= maxlen
        if N_ >= 1:
            grams = _ngrams(body, N_)
            assert len(grams) == len(set(grams)), (s, N_)
        if s[-1] == 0:
            assert len(s) >= L + 1, (s, L)


@pytest.mark.parametrize('N_', [1, 2, 3])
@pytest.mark.parametrize('L', [0, 4])
@pytest.mark.parametrize('k', [1, 3, 5])
def test_constrained_search_properties(N_, L, k):
    opts = toy_options(D=8, W=6, A=5, V=30)
    P = toy_params(opts)
    fi, fn = _callables(P)
    maxlen = 12
    # every live row keeps >= k admissible words: at most maxlen - 1 words of its history plus EOS are banned
    assert opts['n_words'] - 2 - (maxlen - 1) - 1 >= k
    for x in (np.array([3, 7, 9, 4, 11, 5, 21, 0], 'int64'), np.array([4, 4, 4, 4, 4, 4, 0], 'int64')):
        s, sc, al = CO.gen_sample(fi, fn, x[:, None], k=k, maxlen=maxlen, use_unk=True, kl_factor=0.5, ctx_factor=0.5,
                                  state_factor=0.5, no_repeat_ngram=N_, min_len=L)
        _check_output(s, sc, N_, L, k, maxlen)
        assert [len(a) for a in al] == [len(q) for q in s]


def _eos_bias(P, delta):
    P = O.OrderedDict((kk, v.copy()) for kk, v in P.items())
    P['ff_logit_b'][0] += delta
    return P


def test_constraints_bite():
    """An EOS logit raised by 2 makes the unconstrained search retire hypotheses within a few words, and a source of one
    repeated word makes it repeat a trigram; with min_len = 6 and no_repeat_ngram = 3 neither happens."""
    opts = toy_options(D=8, W=6, A=5, V=30)
    P = toy_params(opts)
    x = np.array([4] * 12 + [0], 'int64')[:, None]
    k, maxlen = 3, 14
    fi, fn = _callables(_eos_bias(P, 2.0))
    s0, _, _ = CO.gen_sample(fi, fn, x, k=k, maxlen=maxlen, use_unk=True)
    assert any(q[-1] == 0 and len(q) < 6 + 1 for q in s0), s0
    s1, sc1, _ = CO.gen_sample(fi, fn, x, k=k, maxlen=maxlen, use_unk=True, min_len=6)
    _check_output(s1, sc1, 0, 6, k, maxlen)
    fi, fn = _callables(P)
    s0, _, _ = CO.gen_sample(fi, fn, x, k=k, maxlen=maxlen, use_unk=True)
    assert any(len(_ngrams(list(q), 3)) != len(set(_ngrams(list(q), 3))) for q in s0), s0
    s1, sc1, _ = CO.gen_sample(fi, fn, x, k=k, maxlen=maxlen, use_unk=True, no_repeat_ngram=3)
    _check_output(s1, sc1, 3, 0, k, maxlen)


@pytest.mark.parametrize('model', ['toy', 'golden'])
def test_off_equals_the_oracle(model):
    """both constraints at 0: the oracle's search, hypothesis for hypothesis"""
    if model == 'toy':
        opts = toy_options(D=8, W=6, A=5, V=30)
        P = toy_params(opts)
    else:
        opts, P = _golden()
    fi, fn = _callables(P)
    x = np.array([3, 7, 9, 4, 11, 5, 21, 0], 'int64')[:, None] % opts['n_words']
    for k, use_unk, lam in ((1, True, 0.), (3, False, 0.5), (5, True, 1.5)):
        kw = dict(k=k, maxlen=9, use_unk=use_unk, kl_factor=lam, ctx_factor=lam, state_factor=lam)
        ref = O.gen_sample(fi, fn, x, stochastic=False, **kw)
        got = CO.gen_sample(fi, fn, x, no_repeat_ngram=0, min_len=0, **kw)
        assert [list(map(int, s)) for s in got[0]] == [list(map(int, s)) for s in ref[0]]
        np.testing.assert_array_equal(np.array(got[1]), np.array(ref[1]))
        for ga, ra in zip(got[2], ref[2]):
            np.testing.assert_array_equal(np.array(ga), np.array(ra))


@pytest.mark.parametrize('use_unk', [True, False])
@pytest.mark.parametrize('N_,L', [(1, 0), (2, 4), (3, 6), (0, 5)])
def test_host_loop_equals_oracle(N_, L, use_unk):
    """nats.gen_sample's host loop (foreign f_init / f_next: the full-vocabulary branch) against the oracle"""
    opts = toy_options(D=8, W=6, A=5, V=30)
    P = toy_params(opts, dtype='float32')
    fi, fn = _callables(P)
    x = np.array([4, 4, 9, 4, 4, 9, 4, 4, 0], 'int64')[:, None]
    for k in (1, 3, 5):
        kw = dict(k=k, maxlen=11, use_unk=use_unk, kl_factor=0., ctx_factor=0., state_factor=0., no_repeat_ngram=N_,
                  min_len=L)
        ref = CO.gen_sample(fi, fn, x, **kw)
        got = N.gen_sample(None, fi, fn, x, opts, stochastic=False, **kw)
        assert [list(map(int, s)) for s in got[0]] == [list(map(int, s)) for s in ref[0]]
        np.testing.assert_allclose(np.array(got[1], 'float64'), np.array(ref[1], 'float64'), rtol=1e-6)
        _check_output(got[0], got[1], N_, L, k, 11)


def test_invalid_arguments():
    opts = toy_options(D=8, W=6, A=5, V=30)
    P = toy_params(opts, dtype='float32')
    fi, fn = _callables(P)
    x = np.array([3, 7, 0], 'int64')[:, None]
    for kw in (dict(no_repeat_ngram=-1), dict(min_len=-2)):
        with pytest.raises(ValueError):
            N.gen_sample(None, fi, fn, x, opts, k=2, stochastic=False, **kw)
        with pytest.raises(ValueError):
            CO.gen_sample(fi, fn, x, k=2, **kw)
    for kw in (dict(no_repeat_ngram=3), dict(min_len=2)):
        with pytest.raises(ValueError):
            N.gen_sample(None, fi, fn, x, opts, k=1, stochastic=True, **kw)
