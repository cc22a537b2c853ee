"""GPU tests of the training pipeline around the kernels: shape-bucketed plans on ragged batches, optimizer-state
save / reload, the data-parallel step (2 GPUs, skipped on a 1-GPU box), and the config-1 plumbing run of BASELINE.json:
train on the toy corpus -> generate -> replace_unk -> ROUGE (scripts/test.sh:18-26) with the loss curve recorded."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from oracle import nats_oracle as O
from tests.helpers import toy_options, toy_params

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOY = os.path.join(ROOT, 'tests', 'data', 'toy')


def test_ragged_batches_hit_bucketed_graphs():
    """Batches whose padded lengths differ but fall into the same (Tx, Ty) bucket share ONE plan and replay its captured
    CUDA graph; cost and update are those of the oracle on the unpadded batch (padding invariance, nats.py:354,518,770)."""
    from nats_b200 import nats as N
    opts = toy_options(D=32, W=12, A=10, V=120)
    P = toy_params(opts)
    tparams = N.init_tparams(O.cast_params(P, 'float32'))
    graph = N.build_model(tparams, opts)[-1].mean()
    assert graph.bucket_tx == 8 and graph.bucket_ty == 5
    rng = np.random.RandomState(1)
    seen = []
    for i in range(6):
        mx, my = int(rng.randint(57, 63)), int(rng.randint(11, 14))             # Tx = mx+1 in 58..63 -> bucket 64, Ty = my+1 in 12..14 -> 15
        sx = [list(rng.randint(2, 120, size=rng.randint(5, mx + 1))) for _ in range(4)]
        sy = [list(rng.randint(2, 120, size=rng.randint(2, my + 1))) for _ in range(4)]
        sx[0] = list(rng.randint(2, 120, size=mx)); sy[0] = list(rng.randint(2, 120, size=my))
        batch = O.prepare_data(sx, sy, n_words=120)
        c = graph.grad_step(*batch, after_grads=lambda: None)
        cr, G, _ = O.f_grad(P, *batch)
        assert abs(float(c) - cr) <= 1e-4 * abs(cr), i
        Gd = tparams.view_of(graph.grads[:tparams.total])
        for k in ('Wemb', 'encoder_U', 'decoder_Wc_att', 'ff_logit_W'):
            assert np.linalg.norm(Gd[k] - G[k]) / np.linalg.norm(G[k]) <= 1e-3, (i, k)
        seen.append(batch[0].shape[0])
    assert len(set(seen)) > 1                       # really ragged
    assert len(graph._plans) == 1                   # ... but one bucket
    plan = list(graph._plans.values())[0]
    assert plan.shape == (64, 15, 4) and plan.graph_step is not None and plan.uses == 6


def _toy_kwargs(tmp_path, **kw):
    base = dict(dim_word=32, dim=64, dim_att=24, n_words=200, batch_size=4, valid_batch_size=4, maxlen=150, max_epochs=50,
                dispFreq=10, validFreq=40, saveFreq=40, sampleFreq=1000, clip_c=10., decay_c=0., optimizer='adadelta',
                datasets=[os.path.join(TOY, 'train_input.txt'), os.path.join(TOY, 'train_output.txt')],
                valid_datasets=[os.path.join(TOY, 'validation_input.txt'), os.path.join(TOY, 'validation_output.txt')],
                dictionary=os.path.join(TOY, 'train_input.txt.pkl'), saveto=str(tmp_path / 'toy.npz'), patience=50)
    base.update(kw)
    return base


def test_optimizer_state_save_and_reload(tmp_path):
    from nats_b200 import nats as N
    kw = _toy_kwargs(tmp_path, saveFreq=5, validFreq=1000)
    N.train(finish_after=5, save_optimizer_state=True, **kw)
    opt = str(tmp_path / 'toy.npz') + '.opt.npz'
    with np.load(opt) as zf:                                      # read now: the file is rewritten by the next train()
        z = {k: zf[k].copy() for k in zf.files}
    assert set(z) == {'running_up2', 'running_grads2'}
    assert float(np.abs(z['running_grads2']).sum()) > 0 and float(np.abs(z['running_up2']).sum()) > 0
    ref_names = list(N.init_params(pickle.load(open(str(tmp_path / 'toy.npz') + '.pkl', 'rb'))).keys())
    with np.load(str(tmp_path / 'toy.npz'), allow_pickle=True) as mz:
        assert sorted(set(mz.files) - {'history_errs', 'zipped_params'}) == sorted(ref_names)      # the model file keeps the reference keys
    # reload path: accumulators restored into the new optimiser
    graph_state = {}
    orig = N.load_optimizer_state

    def spy(path, f):
        orig(path, f)
        graph_state.update({k: v.detach().cpu().numpy().copy() for k, v in f.state.items()})
    N.load_optimizer_state = spy
    try:
        N.train(finish_after=1, reload_=True, save_optimizer_state=True, **kw)
    finally:
        N.load_optimizer_state = orig
    np.testing.assert_array_equal(graph_state['running_grads2'], z['running_grads2'])
    np.testing.assert_array_equal(graph_state['running_up2'], z['running_up2'])


def test_toy_corpus_train_generate_rouge(tmp_path):
    """BASELINE.json configs[0] plumbing (dim=64, |V|=200, batch=4) on the committed cut of the reference's toy corpus:
    3000 updates, then gen (beam 5, normalised) -> replace_unk -> ROUGE-1/2/L.  Regression values: the training cost must
    fall well below its initial value and the summaries must share unigrams with the references."""
    from nats_b200 import nats as N, gen, evaluate
    import logging
    records = []

    class H(logging.Handler):
        def emit(self, rec):
            m = rec.getMessage()
            if m.startswith('Epoch'):
                t = m.split()
                records.append((int(t[3]), float(t[5])))
    h = H()
    lg = logging.getLogger('nats_b200.nats')
    old_level = lg.level
    lg.setLevel(logging.DEBUG)                  # pytest owns the root logger: train()'s basicConfig(level=DEBUG) is a no-op here
    lg.addHandler(h)
    try:
        err = N.train(finish_after=3000, **_toy_kwargs(tmp_path, dispFreq=100, validFreq=1000, saveFreq=1000, n_words=1000))
    finally:
        lg.removeHandler(h)
        lg.setLevel(old_level)
    assert np.isfinite(err)
    assert len(records) >= 15
    first, last = np.mean([c for _, c in records[:3]]), np.mean([c for _, c in records[-3:]])
    assert last < 0.9 * first, (first, last, records)
    model = str(tmp_path / 'toy.npz')
    scores = {}
    for split in ('test', 'train'):                 # unseen articles, and the first 16 training articles (memorisation)
        src = os.path.join(TOY, '%s_input.txt' % split)
        ref = os.path.join(TOY, '%s_output.txt' % split)
        if split == 'train':
            src16, ref16 = str(tmp_path / 'tr_in.txt'), str(tmp_path / 'tr_out.txt')
            open(src16, 'w').writelines(open(src).readlines()[:16]); open(ref16, 'w').writelines(open(ref).readlines()[:16])
            src, ref = src16, ref16
        out = str(tmp_path / ('temp_%s.txt' % split)); final = str(tmp_path / ('final_%s.txt' % split))
        gen.main(model, os.path.join(TOY, 'train_input.txt.pkl'), src, out, k=5, normalize=True, n_process=1, kl_factor=0.,
                 ctx_factor=0., state_factor=0.)
        evaluate.replace_unk(src, out, final)
        assert len(open(final).read().split('\n')) >= 16
        for k, (n, m) in {'rouge1': (1, 'N'), 'rouge2': (2, 'N'), 'rougeL': (1, 'L')}.items():
            scores['%s_%s' % (split, k)] = evaluate.rouge_file(n, m, ref, final)
            assert all(0.0 <= v <= 1.0 for v in scores['%s_%s' % (split, k)])
    print('TOY_SCORES', scores, first, last)
    assert scores['train_rouge1'][2] > 0.0 or scores['test_rouge1'][2] > 0.0, scores     # the chain produces words of the references
    rec = {'config': 'toy corpus cut (128 pairs), dim=64, dim_word=32, dim_att=24, n_words=1000, batch=4, adadelta, 3000 updates',
           'loss_curve': records, 'valid_err': float(err), 'rouge': {k: list(v) for k, v in scores.items()}}
    print('TOY_PIPELINE ' + json.dumps(rec))


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize('overlap', ['1', '0'])
def test_dp2_step_equals_single_gpu_step(tmp_path, overlap):
    """Two ranks, each on its shard of a 7-pair global batch (4 + 3), two updates with clipping: the parameters equal the
    single-GPU run on the whole batch (same mean cost, same gradient after the all-reduce), with the all-reduce overlapped
    with the encoder backward (two slices) and as one flat call."""
    if _gpus() < 2:
        pytest.skip('needs 2 GPUs')
    env = dict(os.environ, NATS_OVERLAP_ALLREDUCE=overlap)
    worker = os.path.join(ROOT, 'tests', 'dp_worker.py')
    single, multi = str(tmp_path / 'single.npz'), str(tmp_path / 'multi.npz')
    r = subprocess.run([sys.executable, worker, single], env=dict(env, CUDA_VISIBLE_DEVICES='0'), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
                        '127.0.0.1', '--master-port', '29531', worker, multi], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    a, b = np.load(single), np.load(multi)
    np.testing.assert_allclose(b['costs'], a['costs'], rtol=2e-5)
    for k in a.files:
        if k != 'costs':
            np.testing.assert_allclose(b[k], a[k], rtol=2e-4, atol=2e-6, err_msg=k)
