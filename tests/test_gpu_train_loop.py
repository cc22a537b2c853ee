"""End to end through the reference's driver surface on an H100: train() on a tiny synthetic corpus (validation,
checkpoint, sampling and reload branches of nats.py:1380-1539), then the gen.py path: load_params -> build_sampler ->
gen_sample with a beam and all three distraction penalties."""
import os
import pickle
from collections import OrderedDict

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _corpus(tmp_path, n_train=24, n_valid=8, vocab=30, seed=7):
    rng = np.random.RandomState(seed)
    words = ['w%02d' % i for i in range(vocab)]
    worddict = OrderedDict([('eos', 0), ('UNK', 1)])
    for i, w in enumerate(words):
        worddict[w] = i + 2
    dic = tmp_path / 'dict.pkl'
    with open(dic, 'wb') as f:
        pickle.dump(worddict, f, protocol=2)          # the reference's dictionaries are python-2 pickles

    def write(name, n, lo, hi):
        path = tmp_path / name
        with open(path, 'w') as f:
            for _ in range(n):
                f.write(' '.join(rng.choice(words, size=rng.randint(lo, hi))) + '\n')
        return str(path)

    tr = [write('train.src', n_train, 5, 13), write('train.tgt', n_train, 3, 7)]
    va = [write('valid.src', n_valid, 5, 13), write('valid.tgt', n_valid, 3, 7)]
    return tr, va, str(dic), worddict


def test_train_then_generate(tmp_path):
    from nats_b200 import nats as N
    tr, va, dic, worddict = _corpus(tmp_path)
    saveto = str(tmp_path / 'model.npz')
    kw = dict(dim_word=8, dim=16, dim_att=6, n_words=32, batch_size=4, valid_batch_size=4, maxlen=50, max_epochs=3,
              dispFreq=1, validFreq=3, saveFreq=4, sampleFreq=5, clip_c=10., decay_c=0., optimizer='adadelta',
              datasets=tr, valid_datasets=va, dictionary=dic, saveto=saveto, patience=10)
    err = N.train(finish_after=9, **kw)
    assert np.isfinite(err) and err > 0
    z = np.load(saveto, allow_pickle=True)
    opts = pickle.load(open(saveto + '.pkl', 'rb'))
    assert opts['dim'] == 16 and opts['n_words'] == 32
    names = list(N.init_params(opts).keys())
    assert len(names) == 43 and all(k in z.files for k in names)
    assert 'history_errs' in z.files and 'zipped_params' in z.files and len(z['history_errs']) >= 3
    assert z['Wemb'].shape == (32, 8) and z['decoder_W_att'].shape == (16, 6)
    n_hist = len(z['history_errs'])
    z.close()                                          # the file is rewritten by the next call

    # reload (nats.py:1268-1276, 1290-1292, 1372-1375): continues from the checkpoint and its validation history
    err2 = N.train(finish_after=3, reload_=True, **kw)
    assert np.isfinite(err2)
    z2 = np.load(saveto, allow_pickle=True)
    assert len(z2['history_errs']) >= n_hist
    z2.close()

    # gen.py:78-100: parameters from the checkpoint, sampler, beam search with distraction
    params = N.load_params(saveto, N.init_params(opts))
    tparams = N.init_tparams(params)
    f_init, f_next = N.build_sampler(tparams, opts, None)
    src = [worddict[w] for w in open(va[0]).readline().split()] + [0]
    x = np.array(src, dtype='int64').reshape(-1, 1)
    samples, scores, alphas = N.gen_sample(tparams, f_init, f_next, x, opts, trng=None, k=3, maxlen=8, stochastic=False,
                                           argmax=False, use_unk=False, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    assert 1 <= len(samples) <= 3 and len(scores) == len(samples) and len(alphas) == len(samples)
    assert all(np.isfinite(s) for s in scores) and all(1 <= len(s) <= 8 for s in samples)
    assert all(0 <= int(w) < 32 and int(w) != 1 for s in samples for w in s)        # use_unk=False never emits UNK
    best = samples[int(np.argmin(np.array(scores) / np.array([len(s) for s in samples])))]   # gen.py:45-47
    assert len(best) >= 1
    assert all(np.asarray(a).shape == (x.shape[0],) for al in alphas for a in al)
    # validation cost of the reloaded parameters through f_log_probs equals what train() reported at the end
    from nats_b200.data_iterator import TextIterator
    graph = N.build_model(tparams, opts)[-1]
    vit = TextIterator(va[0], va[1], dic, n_words=32, batch_size=4)
    v = N.pred_probs(graph.f_log_probs, N.prepare_data, opts, vit, verbose=False).mean()
    np.testing.assert_allclose(v, err2, rtol=1e-5)


def test_py3_drivers(tmp_path):
    """nats_b200.train_nats.main(job_id, params) and nats_b200.gen.main(...) -- the python-3 twins of the reference's
    train_nats.py / gen.py -- on the synthetic corpus: same parameter dictionary, same output format."""
    from nats_b200 import gen, train_nats
    tr, va, dic, worddict = _corpus(tmp_path)
    model = str(tmp_path / 'm.npz')
    base = lambda p: os.path.basename(p)
    params = {'data-dir': [str(tmp_path)], 'model': [model], 'train': [base(tr[0]), base(tr[1])],
              'valid': [base(va[0]), base(va[1])], 'dictionary': [base(dic)], 'dim_word': [8], 'dim': [16],
              'dim_att': [6], 'n-words': [32], 'patience': [1], 'optimizer': ['adadelta'], 'decay-c': [0.],
              'clip-c': [100.], 'use-dropout': [False], 'learning-rate': [0.0001], 'reload': [False],
              'batch-size': [4], 'finish-after': [11]}
    err = train_nats.main(0, params)
    assert np.isfinite(err) and os.path.exists(model) and os.path.exists(model + '.pkl')
    out = str(tmp_path / 'gen.txt')
    gen.main(model, dic, va[0], out, k=3, normalize=True, n_process=1, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    lines = open(out).read().split('\n')
    assert len([l for l in lines if l is not None]) >= 8
    n_src = [len(l.split()) + 1 for l in open(va[0])]
    for l, ns in zip(lines[:8], n_src):
        toks = l.split()
        assert len(toks) % 2 == 0
        for w, p in zip(toks[0::2], toks[1::2]):
            assert (w in worddict or w == 'UNK') and p.startswith('[') and 0 <= int(p[1:-1]) < ns
    # -p 2: two spawned worker processes (model replicas) fed with chunks of sentences -- same file, line for line
    out2 = str(tmp_path / 'gen_p2.txt')
    gen.main(model, dic, va[0], out2, k=3, normalize=True, n_process=2, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    assert open(out2).read() == open(out).read()
    # one search at a time on the current stream (NATS_GEN_STREAMS=1) gives the same file as 12 in flight
    os.environ['NATS_GEN_STREAMS'] = '1'
    try:
        out3 = str(tmp_path / 'gen_s1.txt')
        gen.main(model, dic, va[0], out3, k=3, normalize=True, n_process=1, kl_factor=0.5, ctx_factor=0.5, state_factor=0.5)
    finally:
        del os.environ['NATS_GEN_STREAMS']
    assert open(out3).read() == open(out).read()
