"""CPU tests of the host-side mirror of the reference interface (nats_b200/nats.py): parameter inventory and init,
batch layout, beam-search bookkeeping (driven by oracle callables -- the product's own callables need a GPU),
the data iterator and the npz / pkl checkpoint layout (nats.py:81-89, 1427-1435)."""
import os
import pickle

import numpy as np
import pytest

from nats_b200 import nats as N
from nats_b200.data_iterator import TextIterator
from oracle import nats_oracle as O
from tests.helpers import toy_options, toy_params


def test_init_params_matches_reference_inventory_and_rng_stream():
    opts = toy_options(D=8, W=6, A=5, V=50)
    np.random.seed(1234)
    a = N.init_params(opts)
    np.random.seed(1234)
    b = O.init_params(opts)
    assert list(a.keys()) == list(b.keys()) and len(a) == 43
    for k in a:
        assert a[k].dtype == np.float32
        np.testing.assert_array_equal(a[k], b[k])
    # square matrices are orthogonal (nats.py:138-139), incl. decoder_W_1 [2D,2D] and ff_logit_prev is NOT (ortho=False)
    np.testing.assert_allclose(a['decoder_W_1'].T @ a['decoder_W_1'], np.eye(16), atol=1e-5)
    assert np.abs(a['ff_logit_prev_W']).max() < 0.1


def test_prepare_data_contract():
    sx = [[5, 6, 7], [8], [9, 10, 11, 12, 13, 14]]
    sy = [[3, 4], [5, 6, 7, 8], [9]]
    for maxlen in (None, 4, 100):
        a = N.prepare_data(sx, sy, maxlen=maxlen, n_words=50)
        b = O.prepare_data(sx, sy, maxlen=maxlen, n_words=50)
        for u, v in zip(a, b):
            np.testing.assert_array_equal(u, v)
            assert u.dtype == v.dtype
    x, xm, y, ym = N.prepare_data(sx, sy, maxlen=4)
    assert x.shape == (4, 3) and xm[:, 2].tolist() == [1, 1, 1, 1] and xm[:, 1].tolist() == [1, 1, 0, 0]
    assert x.dtype == np.int64 and xm.dtype == np.float32
    assert N.prepare_data([], [], maxlen=4) == (None, None, None, None)


class HostScorer(object):
    """test double for DistractionScorer: same interface, SciPy-semantics arithmetic from the oracle"""

    def __init__(self, k, maxlen, Tx, C, D):
        self.h = [[], [], []]          # per live hypothesis: lists of past alpha / ctx / state vectors

    def penalties(self, a, c, s, live_k, kl, cf, sf):
        return O.distraction_scores(self.h[0][:live_k], self.h[1][:live_k], self.h[2][:live_k], a, c, s, kl, cf, sf)

    def advance(self, a, c, s, parents):
        if not self.h[0]:
            self.h = [[[] for _ in range(1)] for _ in range(3)]
        new = [[], [], []]
        for p in parents:
            for i, cur in enumerate((a, c, s)):
                new[i].append(self.h[i][p] + [np.array(cur[p])] if p < len(self.h[i]) else [np.array(cur[p])])
        self.h = new


@pytest.mark.parametrize('lam', [(0., 0., 0.), (1.5, 1.5, 1.5), (0., 2.0, 0.)])
def test_gen_sample_bookkeeping_equals_reference_restatement(lam):
    opts = toy_options(D=8, W=6, A=5, V=30)
    P = toy_params(opts, dtype='float32')
    fi = lambda x: O.f_init(P, x)
    fn = lambda y, ctx, s, ac, aa: O.f_next(P, y, np.asarray(ctx), s.astype('float32'), ac.astype('float32'),
                                            aa.astype('float32'))
    x = np.array([3, 7, 9, 4, 11, 5, 21, 0], 'int64')[:, None]
    for k in (1, 3, 5):
        ref = O.gen_sample(fi, fn, x, k=k, maxlen=9, stochastic=False, use_unk=(k != 3), kl_factor=lam[0],
                           ctx_factor=lam[1], state_factor=lam[2])
        got = N.gen_sample(None, fi, fn, x, opts, k=k, maxlen=9, stochastic=False, use_unk=(k != 3), kl_factor=lam[0],
                           ctx_factor=lam[1], state_factor=lam[2], _scorer_factory=HostScorer)
        assert [list(map(int, s)) for s in got[0]] == [list(map(int, s)) for s in ref[0]]
        np.testing.assert_allclose(np.array(got[1], 'float64'), np.array(ref[1], 'float64'), rtol=1e-6)
        assert len(got[2]) == len(ref[2])
        for ga, ra in zip(got[2], ref[2]):
            assert len(ga) == len(ra)
            for u, v in zip(ga, ra):
                np.testing.assert_allclose(u, v, rtol=1e-6)
    s1, sc1, _ = N.gen_sample(None, fi, fn, x, opts, k=1, maxlen=9, stochastic=True, argmax=True)
    s2, sc2, _ = O.gen_sample(fi, fn, x, k=1, maxlen=9, stochastic=True, argmax=True)
    assert list(map(int, s1)) == list(map(int, s2)) and np.isclose(sc1, sc2)
    with pytest.raises(AssertionError):
        N.gen_sample(None, fi, fn, x, opts, k=2, stochastic=True)


def test_device_backed_array_survives_tile_and_detects_foreign_arrays():
    host = np.arange(5 * 1 * 4, dtype='float32').reshape(5, 1, 4)
    h = N._CtxHandle('ctx_dev', 'pctx_dev', host)
    arr = N.DeviceBackedArray(host, h)
    tiled = np.tile(arr, [3, 1])                      # what the reference's gen_sample does (nats.py:958)
    assert tiled.shape == (5, 3, 4) and getattr(tiled, '_nats_handle', None) is h and h.matches(tiled)
    view = N._tile_ctx(arr, 3)
    assert view.shape == (5, 3, 4) and h.matches(view) and view.strides[1] == 0
    assert not h.matches(tiled * 2.0)                 # derived data must not be mistaken for the device copy
    assert not h.matches(np.tile(arr, [1, 1])[:4])


def test_text_iterator_and_checkpoint_layout(tmp_path):
    src = tmp_path / 'src.txt'; tgt = tmp_path / 'tgt.txt'; dic = tmp_path / 'dict.pkl'
    src.write_text('a b c\nb c d e\nzz a\n'); tgt.write_text('a\nb c\nd\n')
    with open(dic, 'wb') as f:
        pickle.dump({'eos': 0, 'UNK': 1, 'a': 2, 'b': 3, 'c': 4, 'd': 5, 'e': 6}, f, protocol=2)
    it = TextIterator(str(src), str(tgt), str(dic), batch_size=2, n_words=6)
    batches = list(it)
    assert batches[0] == ([[2, 3, 4], [3, 4, 5, 1]], [[2], [3, 4]])      # 'e' (id 6 >= n_words) -> UNK
    assert batches[1] == ([[1, 2]], [[5]])                               # 'zz' unknown -> UNK
    assert list(it) == batches                                           # automatic rewind (data_iterator.py:33-36)
    # checkpoint layout: npz keys = the 43 names + history_errs; load_params fills / warns (nats.py:81-89)
    opts = toy_options(D=8, W=6, A=5, V=50)
    np.random.seed(0)
    P = N.init_params(opts)
    path = str(tmp_path / 'model.npz')
    np.savez(path, history_errs=[1.5], **P)
    with open(path + '.pkl', 'wb') as f:
        pickle.dump(opts, f, protocol=2)
    np.random.seed(1)
    Q = N.load_params(path, N.init_params(opts))
    for k in P:
        np.testing.assert_array_equal(P[k], Q[k])
    partial = dict(P); partial.pop('decoder_D_wei')
    np.savez(str(tmp_path / 'partial.npz'), **partial)
    with pytest.warns(UserWarning):
        N.load_params(str(tmp_path / 'partial.npz'), N.init_params(opts))
    assert N._load_pickle(path + '.pkl') == opts


def test_toy_corpus_runs_through_the_data_path(tmp_path):
    """BASELINE config 1 plumbing: build a dictionary like data/build_dictionary.py:9-35 does and iterate the committed
    cut of the reference's toy corpus (tests/data/toy: the first 128 training pairs)."""
    base = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'data', 'toy')
    from collections import OrderedDict
    freqs = OrderedDict()
    with open(os.path.join(base, 'train_input.txt')) as f:
        for line in f:
            for w in line.strip().split(' '):
                freqs[w] = freqs.get(w, 0) + 1
    words = list(freqs.keys())
    order = np.argsort(list(freqs.values()))[::-1]
    worddict = OrderedDict([('eos', 0), ('UNK', 1)])
    for i, idx in enumerate(order):
        worddict[words[idx]] = i + 2
    dic = tmp_path / 'toy.pkl'
    with open(dic, 'wb') as f:
        pickle.dump(worddict, f, protocol=2)
    it = TextIterator(os.path.join(base, 'train_input.txt'), os.path.join(base, 'train_output.txt'), str(dic),
                      batch_size=4, n_words=200)
    sx, sy = next(it)
    x, xm, y, ym = N.prepare_data(sx, sy, maxlen=500, n_words=200)
    assert x.shape[1] == 4 and x.max() < 200 and xm.sum(0).min() >= 2 and y.shape[0] == ym.shape[0]
    assert sum(len(b[0]) for b in [(sx, sy)] + list(it)) == 128


def test_device_array_behaves_like_the_host_array_f_next_used_to_return():
    """DeviceArray (what f_next returns): NumPy sees an ordinary array, index lists select rows without leaving the
    tensor's device, writes go to the host copy and are pushed back on the next .tensor() (here on a CPU tensor)."""
    import torch
    base = np.arange(12, dtype='float32').reshape(4, 3)
    a = N.DeviceArray(torch.from_numpy(base.copy()))
    assert a.shape == (4, 3) and a.ndim == 2 and len(a) == 4 and a.dtype == np.float32 and a.size == 12
    np.testing.assert_array_equal(np.asarray(a), base)
    np.testing.assert_array_equal(np.log(a + 1.0), np.log(base + 1.0))
    np.testing.assert_array_equal(a[1], base[1])                      # scalar index -> host row
    assert a[0, 2] == base[0, 2] and a[0].argmax() == 2
    sel = a[[2, 0, 2]]                                                # index list -> stays a DeviceArray
    assert isinstance(sel, N.DeviceArray)
    c = sel.copy()                                                    # before any host access: a device-side clone
    assert isinstance(c, N.DeviceArray)
    np.testing.assert_array_equal(np.asarray(sel), base[[2, 0, 2]])
    assert isinstance(sel.copy(), np.ndarray)                         # once on the host, copies are host arrays
    c[:, 1] = -5.0                                                    # write: host copy, marked dirty
    assert np.asarray(sel)[0, 1] == base[2, 1]                        # the source of the copy is untouched
    np.testing.assert_array_equal(c.tensor().numpy()[:, 1], [-5.0, -5.0, -5.0])     # pushed back to the tensor
    b = N.DeviceArray(torch.tensor([3, 1, 2], dtype=torch.int64))
    assert b.dtype == np.int64 and int(b[0]) == 3
    hyp = np.zeros(4, 'float32')
    np.testing.assert_array_equal(hyp[:, None] - np.log(a + 1.0), -np.log(base + 1.0))


def test_text_iterator_bucketing_keeps_the_epoch_and_cuts_padding(tmp_path):
    """bucket_batches (ours, default off): every pair is still seen exactly once per epoch, the iterator rewinds like
    the reference's, and the padded source area shrinks."""
    from collections import OrderedDict
    rng = np.random.RandomState(0)
    words = ['w%d' % i for i in range(12)]
    wd = OrderedDict([('eos', 0), ('UNK', 1)] + [(w, i + 2) for i, w in enumerate(words)])
    with open(tmp_path / 'd.pkl', 'wb') as f:
        pickle.dump(wd, f, protocol=2)
    lens = rng.randint(2, 40, size=37)
    with open(tmp_path / 's.txt', 'w') as fs, open(tmp_path / 't.txt', 'w') as ft:
        for i, n in enumerate(lens):
            fs.write(' '.join(rng.choice(words, size=n)) + '\n')
            ft.write(' '.join(rng.choice(words, size=1 + i % 5)) + '\n')

    def epoch(it):
        batches = list(it)
        pairs = sorted((tuple(s), tuple(t)) for sx, sy in batches for s, t in zip(sx, sy))
        area = sum(max(len(s) for s in sx) * len(sx) for sx, _ in batches)
        return batches, pairs, area

    plain = TextIterator(str(tmp_path / 's.txt'), str(tmp_path / 't.txt'), str(tmp_path / 'd.pkl'), batch_size=4)
    buck = TextIterator(str(tmp_path / 's.txt'), str(tmp_path / 't.txt'), str(tmp_path / 'd.pkl'), batch_size=4,
                        bucket_batches=5)
    b0, p0, a0 = epoch(plain)
    b1, p1, a1 = epoch(buck)
    assert p0 == p1 and len(p1) == 37                       # same multiset of pairs
    assert sum(len(sx) for sx, _ in b1) == 37 and max(len(sx) for sx, _ in b1) <= 4
    assert a1 < 0.8 * a0                                    # much less padding
    _, p2, _ = epoch(buck)                                  # automatic rewind: a second epoch yields the same pairs
    assert p2 == p1
