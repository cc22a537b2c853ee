"""One self-critical update at config-3 dimensions, phase by phase: D = 1000, W = 100, A = 100, V = 30000 (random init),
32 sources of 399 words + EOS, 30-word references, R = 4 samples of at most --maxlen words.  Phases, each timed on the host
around work that ends in a device synchronise, `--reps` times after a warm-up:
  * sampling: sample_many (R = 4, unfiltered) and the greedy baseline (sample_many, top_k = 1);
  * reward: nats.rouge_f on the 160 (sample or greedy, reference) pairs (host staging, one copy, the kernel, the read back;
    the kernel alone from the profiler), against evaluate.rouge_n(1) + rouge_n(2) + rouge_l on the same pairs;
  * the weighted step at 160 columns (32 ground-truth + 128 sampled columns, a replayed CUDA graph);
  * the ML step at 32 columns, for comparison.
Prints JSON lines, the first with the card and its power limit.

    python tools/scst_bench.py [--reps 5] [--maxlen 100]
"""
import argparse
import contextlib
import ctypes
import io
import json
import subprocess
import sys
import time

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nats_b200 import evaluate, nats  # noqa: E402


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                       text=True, timeout=60, check=True)
    return r.stdout.strip()


def timed(f, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.time()
        f()
        torch.cuda.synchronize()
        out.append(round(1e3 * (time.time() - t0), 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--maxlen', type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('scst_bench measures the GPU: no CUDA device')
    V, R, B = 30000, 4, 32
    opts = dict(dim_word=100, dim=1000, dim_att=100, n_words=V, encoder='gru', decoder='gru_cond')
    np.random.seed(1234)
    with contextlib.redirect_stdout(io.StringIO()):
        tparams = nats.init_tparams(nats.init_params(opts))
    graph = nats.build_model(tparams, opts)[-1].mean()
    f_grad_shared, _ = nats.adadelta('lr', tparams, graph, None, graph)
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    rng = np.random.RandomState(7)
    sx = [list(rng.randint(2, V, size=399)) for _ in range(B)]
    sy = [list(rng.randint(2, V, size=30)) for _ in range(B)]
    xs = [np.array(s + [0], dtype='int64') for s in sx]
    print(json.dumps({'card': card(), 'sources': B, 'samples': R, 'maxlen': args.maxlen, 'Tx': 400, 'ref_words': 30}),
          flush=True)

    res = {}

    def sample():
        res['s'] = nats.sample_many(tparams, f_init, f_next, xs, opts, n_samples=R, maxlen=args.maxlen, index_base=0)
        res['g'] = nats.sample_many(tparams, f_init, f_next, xs, opts, n_samples=1, maxlen=args.maxlen, top_k=1,
                                    index_base=0)
    sample()
    t_sample = timed(sample, args.reps)
    samples = [s for b in range(B) for s in res['s'][b][0]]
    cands = [c for b in range(B) for c in res['s'][b][0] + res['g'][b][0]]
    lens = [len(c) for c in cands]

    def reward():
        res['r'] = nats.rouge_f(cands, sy, rows_per_ref=R + 1)
    reward()
    t_rouge = timed(reward, args.reps)
    eng = nats.get_engine()
    eng.lib.nats_profile_enable(eng.ctx, 1)
    reward()
    n = eng.lib.nats_profile_num_classes()
    ms, fl, by, la = (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_int64 * n)()
    eng.lib.nats_profile_read(eng.ctx, n, ms, fl, by, la)
    eng.lib.nats_profile_enable(eng.ctx, 0)
    k_rouge = [ms[i] for i in range(n) if eng.lib.nats_profile_class_name(i) == b'rouge'][0]
    lines = []                                  # the same pairs as text: words up to EOS, each UNK a word of its own
    for q, c in enumerate(cands):
        words = []
        for t in c:
            if t == 0:
                break
            words.append('unk_%d' % len(words) if t == 1 else str(t))
        lines.append((' '.join(str(t) for t in sy[q // (R + 1)]), ' '.join(words)))
    t0 = time.time()
    for a, b in lines:
        evaluate.rouge_n(a, b, 1)
        evaluate.rouge_n(a, b, 2)
        evaluate.rouge_l(a, b)
    t_eval = round(1e3 * (time.time() - t0), 3)

    rl = res['r'][2].reshape(B, R + 1)
    x, xm, y, ym, w = nats.scst_batch(sx, sy, samples, rl[:, :R].reshape(-1), rl[:, R], 0.9)
    for _ in range(3):
        f_grad_shared(x, xm, y, ym, global_batch=B, weights=w)
    t_w = timed(lambda: float(f_grad_shared(x, xm, y, ym, global_batch=B, weights=w)), args.reps)
    bx, bxm, by_, bym = nats.prepare_data(sx, sy)
    for _ in range(3):
        f_grad_shared(bx, bxm, by_, bym)
    t_ml = timed(lambda: float(f_grad_shared(bx, bxm, by_, bym)), args.reps)
    print(json.dumps({'sample_and_greedy_ms': t_sample, 'rouge_f_ms': t_rouge, 'rouge_kernel_ms': round(k_rouge, 4),
                      'evaluate_py_ms': t_eval, 'pairs': len(cands), 'mean_candidate_len': float(np.mean(lens)),
                      'weighted_step_160_ms': t_w, 'weighted_step_shape': [int(x.shape[0]), int(y.shape[0]), int(x.shape[1])],
                      'ml_step_32_ms': t_ml, 'mean_sample_rouge_l': float(rl[:, :R].mean()),
                      'mean_greedy_rouge_l': float(rl[:, R].mean())}), flush=True)


if __name__ == '__main__':
    main()
