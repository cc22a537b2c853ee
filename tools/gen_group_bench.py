"""sentences/s and peak device memory of gen_sample_many against the group size (`chunk`: sentences per device step) and the
number of groups in flight (`concurrency`).  Config-5 model (random init, ff_logit_b[0] = -1e9 so that no hypothesis
retires), beam 10, 25 steps, kl = ctx = state = 1, two sets of 32 sources: bench.py's gen_throughput lengths (695..800
words) and short ones (100..400).  Wall clock includes f_init and the result copies; chunk = 1 is the single-sentence
search.  Prints one JSON line per point, the card and its power limit, and the CUPTI kernel table of one grouped search.

    python tools/gen_group_bench.py [--steps 25] [--table-chunk 16]
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


def power_limit():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=25)
    ap.add_argument('--table-chunk', type=int, default=16)
    args = ap.parse_args()
    w = bench.WORKLOADS['c5']
    opts = bench.options_of(w)
    np.random.seed(1234)
    with contextlib.redirect_stdout(io.StringIO()):
        tparams = nats.init_tparams(nats.init_params(opts))
    b = tparams['ff_logit_b'].get_value()
    b[0] = -1e9
    tparams['ff_logit_b'].set_value(b)
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    eng = f_next.engine
    rng = np.random.RandomState(99)
    sets = {
        'long_695_800': [np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1 - 7 * (i % 16),)).tolist() + [0], dtype='int64')
                         for i in range(32)],
        'short_100_400': [np.array(rng.randint(2, w['n_words'], size=(100 + 300 * i // 31,)).tolist() + [0], dtype='int64')
                          for i in range(32)],
    }
    print(json.dumps({'card': torch.cuda.get_device_name(0), 'power_limit': power_limit(), 'beam': 10, 'steps': args.steps}))
    kw = dict(k=10, maxlen=args.steps, use_unk=True, kl_factor=1.0, ctx_factor=1.0, state_factor=1.0)
    for name, xs in sets.items():
        for chunk in (1, 4, 8, 16, 32):
            for conc in (1, 2, 4, 12):
                eng._ws.clear()                               # workspaces of the previous point do not count towards this one
                torch.cuda.empty_cache()
                nats.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=conc, chunk=chunk, **kw)    # warm
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.time()
                nats.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=conc, chunk=chunk, **kw)
                torch.cuda.synchronize()
                dt = time.time() - t0
                print(json.dumps({'set': name, 'chunk': chunk, 'concurrency': conc, 'sentences_per_s': round(len(xs) / dt, 1),
                                  'peak_gb': round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}), flush=True)
    xs = sets['long_695_800'][:args.table_chunk]
    rows = bench.kernel_table(torch, lambda: nats.gen_sample_many(tparams, f_init, f_next, xs, opts, concurrency=1,
                                                                  chunk=len(xs), **kw), steps=1)
    busy = sum(v[0] for v in rows.values())
    top = sorted(rows.items(), key=lambda kv: -kv[1][0])[:14]
    print(json.dumps({'kernel_table': 'one group of %d long sources, %d steps' % (len(xs), args.steps), 'busy_us': round(busy, 1),
                      'top': [{'kernel': k_.replace('(anonymous namespace)::', '').replace('nats::', '').split('(')[0][:50],
                               'excl_us': round(v[0], 1), 'share': round(v[0] / busy, 3), 'launches': v[2]} for k_, v in top]}))


if __name__ == '__main__':
    main()
