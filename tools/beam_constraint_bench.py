"""Cost of the beam-search output constraints on the grouped device search.  Workload: bench.py's gen_throughput at config 5
(random init, ff_logit_b[0] = -1e9 so that no hypothesis retires), 32 sources of 695..800 words, beam 10, 25 steps,
kl = ctx = state = 1, gen_sample_many(chunk=16, concurrency=12).  Constraints off and no_repeat_ngram = 3 / min_len = 10
run alternately in one process, `--reps` times each; wall clock includes f_init and the result copies.  A separate
torch.profiler run of one constrained group of 16 reports beam_constrain_kernel's share of the GPU's busy time.  Prints JSON
lines, the first with the card and its power limit.

    python tools/beam_constraint_bench.py [--reps 3] [--steps 25]
"""
import argparse
import contextlib
import io
import json
import subprocess
import sys
import time

sys.path.insert(0, '.')
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from nats_b200 import nats  # noqa: E402


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                       text=True, timeout=60, check=True)
    return r.stdout.strip()


def _ngram_repeats(s, n):
    g = [tuple(s[i:i + n]) for i in range(len(s) - n + 1)]
    return len(g) - len(set(g))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--steps', type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('beam_constraint_bench measures the GPU: no CUDA device')
    w = bench.WORKLOADS['c5']
    opts = bench.options_of(w)
    np.random.seed(1234)
    with contextlib.redirect_stdout(io.StringIO()):
        tparams = nats.init_tparams(nats.init_params(opts))
    b = tparams['ff_logit_b'].get_value()
    b[0] = -1e9
    tparams['ff_logit_b'].set_value(b)
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    rng = np.random.RandomState(99)
    xs = [np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1 - 7 * (i % 16),)).tolist() + [0], dtype='int64')
          for i in range(32)]
    print(json.dumps({'card': card(), 'beam': 10, 'steps': args.steps, 'sources': len(xs), 'chunk': 16, 'concurrency': 12}),
          flush=True)
    base = dict(k=10, maxlen=args.steps, use_unk=True, kl_factor=1.0, ctx_factor=1.0, state_factor=1.0)
    modes = {'off': dict(base), 'ngram3_min10': dict(base, no_repeat_ngram=3, min_len=10)}

    def run(mode):
        return nats.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=12, chunk=16, **modes[mode])

    for _ in range(2):                                        # warm: kernels, workspaces, streams, allocator
        res = {m: run(m) for m in modes}
    rates = {m: [] for m in modes}
    for _ in range(args.reps):
        for m in modes:
            torch.cuda.synchronize()
            t0 = time.time()
            res[m] = run(m)
            torch.cuda.synchronize()
            rates[m].append(round(len(xs) / (time.time() - t0), 1))
    rep = {m: sum(_ngram_repeats([int(t) for t in s], 3) for samples, _, _ in res[m] for s in samples) for m in modes}
    differ = sum(1 for a, c in zip(res['off'], res['ngram3_min10']) if [list(map(int, s)) for s in a[0]] !=
                 [list(map(int, s)) for s in c[0]])
    print(json.dumps({'sentences_per_s': rates, 'repeated_trigrams_in_hypotheses': rep,
                      'sentences_whose_hypotheses_differ': differ}), flush=True)
    grp = xs[:16]
    rows = bench.kernel_table(torch, lambda: nats.gen_sample_many(tparams, f_init, f_next, grp, opts, concurrency=1,
                                                                  chunk=len(grp), **modes['ngram3_min10']), steps=1)
    busy = sum(v[0] for v in rows.values())
    mine = [(k_, v) for k_, v in rows.items() if 'beam_constrain_kernel' in k_]
    if not mine:
        raise SystemExit('beam_constrain_kernel does not appear in the profile')
    excl = sum(v[0] for _, v in mine)
    print(json.dumps({'profile': 'one group of 16 sources, %d steps, no_repeat_ngram=3, min_len=10' % args.steps,
                      'busy_us': round(busy, 1), 'beam_constrain_kernel_us': round(excl, 1),
                      'launches': sum(v[2] for _, v in mine), 'share': round(excl / busy, 5)}), flush=True)


if __name__ == '__main__':
    main()
