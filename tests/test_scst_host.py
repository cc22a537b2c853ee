"""Self-critical training, the parts a CPU can check: the integer restatement of the device ROUGE (tests/rouge_oracle.py)
against nats_b200.evaluate, the float64 truth of the weighted step, scst_batch's columns, and the argument checks of
train(), scst_step's options and rouge_f."""
import numpy as np
import pytest

from nats_b200 import _lib, evaluate
from oracle import nats_oracle as O
from tests import rouge_oracle as RO
from tests.helpers import toy_options, toy_params, ragged_batch

# evaluate.py cuts P, R and F to 5 decimals: two roundings of P and R (dF/dP + dF/dR <= 2) plus that of F
TOL = 1.5e-5


def _line(ws, side):
    """space-joined ids; each UNK renamed to a string of its own, so it matches nothing, as in the kernel"""
    return ' '.join('unk_%s%d' % (side, i) if w == RO.UNK else str(w) for i, w in enumerate(ws))


def _evaluate(cand, ref):
    a, b = _line(ref, 'r'), _line(cand, 'c')
    return np.array([evaluate.rouge_n(a, b, 1)[2], evaluate.rouge_n(a, b, 2)[2], evaluate.rouge_l(a, b)[2]])


CASES = [
    ([], []), ([5], []), ([], [5]), ([5], [5]), ([5], [6]),                       # empty, and lengths below N = 2
    ([5, 5, 5, 7], [5, 7, 5, 5, 5, 5]), ([3, 4, 3, 4, 3, 4], [4, 3, 4, 3]),       # repeated n-grams on both sides
    ([1, 1, 1], [1, 1, 1]), ([1, 5, 1, 6], [5, 1, 6, 1]),                       # UNK never matches, UNK included
    ([9, 8, 0, 7, 6], [9, 8, 7, 6]), ([0, 3], [3]),                             # EOS in mid-row
    ([2, 3, 4, 5, 6, 7], [7, 6, 5, 4, 3, 2]),
]


@pytest.mark.parametrize('cand,ref', CASES)
def test_restatement_matches_evaluate(cand, ref):
    got = RO.rouge_rows([cand], [ref])[:, 0]
    want = _evaluate(RO.words(cand), RO.words(ref))
    assert np.abs(got - want).max() <= TOL, (got, want)


def test_restatement_matches_evaluate_random():
    rng = np.random.RandomState(5)
    worst = 0.
    for _ in range(300):
        V = rng.choice([4, 8, 40])
        ref = list(rng.randint(1, V, size=rng.randint(0, 40)))
        cand = list(rng.randint(1, V, size=rng.randint(0, 40)))
        if rng.rand() < 0.3:                                          # rows with an EOS in them, or never ending
            cand.insert(rng.randint(0, len(cand) + 1), 0)
        got = RO.rouge_rows([cand], [ref])[:, 0]
        want = _evaluate(RO.words(cand), RO.words(ref))
        worst = max(worst, float(np.abs(got - want).max()))
    assert worst <= TOL, worst


def test_restatement_clamps_lengths():
    assert RO.words([4, 5, 6], length=-3, cap=3) == []
    assert RO.words([4, 5, 6], length=99, cap=3) == [4, 5, 6]
    assert RO.words([4, 0, 6], length=3, cap=3) == [4]
    assert RO.words([4, 5, 6], length=2, cap=3) == [4, 5]


def test_weighted_oracle_is_the_sum_of_single_sample_gradients():
    """O.model_bwd with dcost = scale * w equals sum_b of the gradient of column b alone, weights of both signs and zero
    included: the truth of nats_train_bwd_weighted"""
    opts = toy_options(D=8, W=6, A=5, V=37)
    P = toy_params(opts)
    x, xm, y, ym = ragged_batch(37, B=5, max_x=7, max_y=5, seed=11)
    w = np.array([0.5, -1.25, 0., 2., -0.125])
    scale = 1. / 3
    _, cache = O.model_fwd(P, x, xm, y, ym)
    G = O.model_bwd(P, cache, scale * w)
    acc = O.zero_grads(P)
    for b in range(x.shape[1]):
        _, cb = O.model_fwd(P, x[:, b:b + 1], xm[:, b:b + 1], y[:, b:b + 1], ym[:, b:b + 1])
        Gb = O.model_bwd(P, cb, np.array([scale * w[b]]))
        for k in acc:
            acc[k] += Gb[k]
    for k in G:
        np.testing.assert_allclose(G[k], acc[k], rtol=1e-10, atol=1e-14, err_msg=k)


# ------------------------------------------------------------------------------------------------ scst_batch
def test_scst_batch_columns_weights_masks():
    from nats_b200 import nats as N
    sx = [[5, 6, 7], [8, 9]]
    sy = [[3, 4], [2]]
    samples = [[4, 4, 0], [7, 8, 9],          # source 0: ended with EOS, cut at maxlen
               [0], [5, 6]]                   # source 1: EOS first, cut
    rewards = np.array([0.5, 0.25, 0., 1.], dtype=np.float32)
    base = np.array([0.25, 0.5], dtype=np.float32)
    x, xm, y, ym, w = N.scst_batch(sx, sy, samples, rewards, base, 0.75)
    assert x.shape[1] == 6 and w.dtype == np.float32
    # ground truth first, then (source, sample) in order
    cols_x = [sx[0], sx[1], sx[0], sx[0], sx[1], sx[1]]
    cols_y = [sy[0], sy[1], [4, 4], [7, 8, 9], [], [5, 6]]
    for c in range(6):
        L = len(cols_x[c])
        assert list(x[:L, c]) == cols_x[c] and np.all(x[L:, c] == 0) and xm[:L + 1, c].sum() == L + 1
        Ly = len(cols_y[c])
        assert list(y[:Ly, c]) == cols_y[c] and np.all(y[Ly:, c] == 0)
        assert np.all(ym[:Ly, c] == 1) and np.all(ym[Ly + 1:, c] == 0)
    # the implicit EOS row: mask 1 for the ground truth and the samples that ended, 0 for the cut ones
    assert [ym[len(cols_y[c]), c] for c in range(6)] == [1, 1, 1, 0, 1, 0]
    np.testing.assert_array_equal(w, np.float32([0.25, 0.25, 0.75 * 0.25 / 2, 0.75 * 0. / 2, 0.75 * -0.5 / 2,
                                                 0.75 * 0.5 / 2]))


def test_scst_batch_gamma_one_drops_ground_truth():
    from nats_b200 import nats as N
    x, xm, y, ym, w = N.scst_batch([[5, 6]], [[3]], [[3, 0], [4, 4]], [1., 0.], [0.5], 1.)
    assert x.shape[1] == 2 and list(w) == [0.25, -0.25]
    assert list(y[:, 0]) == [3, 0, 0] and list(ym[:, 0]) == [1, 1, 0]
    assert list(y[:, 1]) == [4, 4, 0] and list(ym[:, 1]) == [1, 1, 0]


@pytest.mark.parametrize('kw', [dict(gamma=1.5), dict(gamma=-0.1), dict(base=[0.]), dict(samples=[[3], [4], [5]]),
                                dict(rewards=[1.])])
def test_scst_batch_rejects(kw):
    from nats_b200 import nats as N
    a = dict(seqs_x=[[5], [6]], seqs_y=[[3], [4]], samples=[[3], [4]], rewards=[0., 1.], base=[0., 0.], gamma=0.5)
    a.update(kw)
    with pytest.raises(ValueError):
        N.scst_batch(a['seqs_x'], a['seqs_y'], a['samples'], a['rewards'], a['base'], a['gamma'])


# ------------------------------------------------------------------------------------------------ argument errors
@pytest.mark.parametrize('kw', [dict(rl_weight=1.5), dict(rl_weight=-0.5), dict(rl_weight=float('nan')),
                                dict(rl_weight=0.5, rl_samples=0), dict(rl_weight=0.5, rl_samples=1.5),
                                dict(rl_weight=0.5, rl_maxlen=50, maxlen=50), dict(rl_weight=0.5, rl_maxlen=0),
                                dict(rl_weight=0.5, rl_seed=-1)])
def test_train_rejects_bad_rl_options(kw, tmp_path):
    """before anything is read or built: the dictionary does not even exist"""
    from nats_b200 import nats as N
    with pytest.raises(ValueError):
        N.train(dictionary=str(tmp_path / 'missing.pkl'), **kw)


def test_train_default_rl_options_are_accepted():
    """with rl_weight = 0 the sampling options are not checked: train()'s defaults (maxlen 100, rl_maxlen 100) hold"""
    from nats_b200 import nats as N
    assert N._check_scst(0., 4, 100, 100)[0] == 0.
    assert N._check_scst(1., 4, 99, 100) == (1., 4, 99)


@pytest.mark.parametrize('args', [
    (([[3]], [[3]]), dict(rows_per_ref=0)),
    (([[3]], [[3]]), dict(rows_per_ref=1.5)),
    (([[3], [4], [5]], [[3]]), dict(rows_per_ref=2)),
    (([], []), {}),
    (([[3.5]], [[3]]), {}),
    (([[2 ** 31]], [[3]]), {}),
    (([[[3]]], [[3]]), {}),
    (('abc', [[3]]), {}),
    (([[3] * 3000], [[3] * 1097]), {}),
])
def test_rouge_f_rejects(args):
    from nats_b200 import nats as N
    (c, r), kw = args
    with pytest.raises(ValueError):
        N.rouge_f(c, r, **kw)


def test_version_and_cap():
    lib = _lib.load()
    assert lib.nats_version() == 104
    src = open(_lib.HEADER_PATH).read()
    assert '#define NATS_ROUGE_MAX_CAP %d ' % _lib.ROUGE_MAX_CAP in src
