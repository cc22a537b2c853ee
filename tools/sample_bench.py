"""Filtered sampling on the device (nats.sample_many) against beam search at equal rows.  Workload: bench.py's
gen_throughput at config 5 (random init), 32 sources of 695..800 words, 25 steps forced with min_len = 25, chunk 16,
concurrency 12.  Beam search k = 10 (gen_sample_many, no distraction factors), sample_many R = 10 unfiltered and at
T = 0.8, K = 50, P = 0.95 run alternately in one process, `--reps` times each; wall clock includes f_init and the result
copies.  A torch.profiler run of one group of 16 per mode gives the kernel table: the share of the sampling kernels
(sample_filter_kernel, sample_advance_kernel, the ban kernel) in the GPU's busy time, and the busy time per step next to
beam search's.  Prints JSON lines, the first with the card and its power limit.

    python tools/sample_bench.py [--reps 3] [--steps 25]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--steps', type=int, default=25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('sample_bench measures the GPU: no CUDA device')
    w = bench.WORKLOADS['c5']
    opts = bench.options_of(w)
    np.random.seed(1234)
    with contextlib.redirect_stdout(io.StringIO()):
        tparams = nats.init_tparams(nats.init_params(opts))
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    rng = np.random.RandomState(99)
    xs = [np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1 - 7 * (i % 16),)).tolist() + [0], dtype='int64')
          for i in range(32)]
    print(json.dumps({'card': card(), 'rows_per_source': 10, 'steps': args.steps, 'sources': len(xs), 'chunk': 16,
                      'concurrency': 12}), flush=True)
    L = args.steps
    modes = {
        'beam_k10': lambda grp, conc: nats.gen_sample_many(tparams, f_init, f_next, grp, opts, k=10, maxlen=L, use_unk=True,
                                                           min_len=L, concurrency=conc, chunk=16),
        'sample_r10': lambda grp, conc: nats.sample_many(tparams, f_init, f_next, grp, opts, n_samples=10, maxlen=L,
                                                         min_len=L, concurrency=conc, chunk=16),
        'sample_r10_t0.8_k50_p0.95': lambda grp, conc: nats.sample_many(tparams, f_init, f_next, grp, opts, n_samples=10,
                                                                        maxlen=L, min_len=L, temperature=0.8, top_k=50,
                                                                        top_p=0.95, concurrency=conc, chunk=16),
    }
    for _ in range(2):                                        # warm: kernels, workspaces, streams, allocator
        res = {m: f(xs, 12) for m, f in modes.items()}
    for m in modes:                                           # every row ran all the steps (EOS banned before L)
        assert all(len(s) == L for samples, _, _ in res[m] for s in samples), m
    rates = {m: [] for m in modes}
    for _ in range(args.reps):
        for m, f in modes.items():
            torch.cuda.synchronize()
            t0 = time.time()
            f(xs, 12)
            torch.cuda.synchronize()
            rates[m].append(round(len(xs) / (time.time() - t0), 1))
    print(json.dumps({'sentences_per_s': rates}), flush=True)
    grp = xs[:16]
    mine = ('sample_filter_kernel', 'sample_advance_kernel', 'beam_constrain_kernel')
    for m, f in modes.items():
        rows = bench.kernel_table(torch, lambda: f(grp, 1), steps=1)
        busy = sum(v[0] for v in rows.values())
        top = sorted(rows.items(), key=lambda kv: -kv[1][0])[:8]
        own = dict((k_, round(v[0], 1)) for k_, v in rows.items() if any(t in k_ for t in mine))
        print(json.dumps({'profile': '%s: one group of 16 sources, %d steps' % (m, L), 'busy_us': round(busy, 1),
                          'busy_us_per_step': round(busy / L, 1), 'sampling_kernels_us': own,
                          'sampling_share': round(sum(own.values()) / busy, 5),
                          'top_kernels_us': [(k_[:60], round(v[0], 1), v[2]) for k_, v in top]}), flush=True)


if __name__ == '__main__':
    main()
