#!/usr/bin/env python
"""bench.py -- decoder tokens/sec of the nats hot path (BASELINE.json metric) on N H100s of one node.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--workload c3|c2|c5] [--ragged]
                    [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

Workloads (BASELINE.json configs):
  c3 (default)  CNN/DM-shaped synthetic: src_len=400, tgt_len=30, dim=1000, |V|=30000, batch=32 per GPU
  c2            LCSTS-shaped synthetic:  src_len=120, tgt_len=20, dim=500,  |V|=4000,  batch=64 per GPU
  c5            gen_sample beam search: beam=10, src_len=800, dim=1000, |V|=30000, all three distraction factors on (1 GPU)

c2 / c3: a "step" is one full training step on one synthetic batch -- region R2 of SURVEY 8(d), the reference's `UD`
bracket (nats.py:1400-1411):
    f_grad_shared(x, x_mask, y, y_mask)  = bi-GRU encoder, attention+distraction decoder scan, readout+softmax/NLL,
                                           hand-written backward, (N>1: NCCL all-reduce of the flat gradient, its larger
                                           slice overlapped with the encoder backward), clip, Adadelta accumulators
    f_update(lrate)                      = Adadelta parameter update
tokens = sum(y_mask) (= B*Ty per GPU), weak scaling.
  value : device-resident inputs, K steps replayed as CUDA graphs, CUDA-event timed, max over ranks.
  e2e   : the same K steps through the reference-facing API with HOST numpy inputs: every step copies its batch through
          pinned memory to the device and reads the step's cost back (the read of step i completes while step i+1 is
          already queued: `graph.lazy_cost`); --ragged draws the lengths uniformly in [T/2, T] (shape-bucketed plans).
  r1    : region R1 = decoder forward (gru_cond_layer scan + readout + NLL on a precomputed context, nats.py:737-770),
          the HBM-bound region SURVEY 8(d) states the 158.2 MB/step roofline for -- first-class, with its own roofline and
          CPU baseline.
  roofline / kernels : per-kernel durations taken from the REPLAYED graph step with the CUPTI activity tracer
          (torch.profiler): they add up to <= ms_per_step by construction.
c5: a "step" is one beam step (f_next on 10 live hypotheses + distraction re-ranking + bookkeeping); value = hypothesis
tokens/s, plus full-sentence latency.

cpu_baseline / --impl reference: the float32 NumPy/OpenBLAS restatement of scripts/nats.py (oracle/) on the host cores, on
the FULL batch of the workload (Python 2 + Theano cannot be installed here), BLAS thread count chosen by calibration.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WORKLOADS = {
    'c3': dict(Tx=400, Ty=30, dim=1000, dim_word=100, dim_att=100, n_words=30000, B=32,
               name='CNN/DM-shaped synthetic: src_len=400, tgt_len=30, dim=1000, |V|=30000, batch=32/GPU'),
    'c2': dict(Tx=120, Ty=20, dim=500, dim_word=100, dim_att=100, n_words=4000, B=64,
               name='LCSTS-shaped synthetic: src_len=120, tgt_len=20, dim=500, |V|=4000, batch=64/GPU'),
    'c5': dict(Tx=801, Ty=100, dim=1000, dim_word=100, dim_att=100, n_words=30000, B=10,
               name='gen_sample beam search: beam=10, src_len=800, dim=1000, |V|=30000, kl=ctx=state factor 1.0'),
}
METRIC = 'decoder tokens/sec (dim=1000, src=400, |V|=30k) @1/2/4/8 H100 vs Theano CPU'


DUMP_SAMPLE = 1 << 20          # elements kept of an output larger than this (fixed seeded positions)


def dump_outputs(d, arrays):
    """Write what the timed path returned in its last step as DIR/<name>.npy (float32, or float64 for tokens and scores).
    Outputs above DUMP_SAMPLE elements are sampled at positions drawn from a fixed seed (also written, as <name>_index),
    so two builds can be compared output for output; the whole dump stays far below 64 MB."""
    os.makedirs(d, exist_ok=True)
    for name, a in arrays.items():
        a = np.asarray(a)
        a = a.astype('float64') if a.dtype.kind in 'iuf' and a.dtype.itemsize == 8 else a.astype('float32')
        if a.size > DUMP_SAMPLE:
            idx = np.sort(np.random.RandomState(0).choice(a.size, DUMP_SAMPLE, replace=False))
            np.save(os.path.join(d, name + '_index.npy'), idx.astype('float64'))
            a = a.reshape(-1)[idx]
        np.save(os.path.join(d, name + '.npy'), a)


def make_batches(w, n, seed, B=None, ragged=False):
    """BASELINE.md synthetic inputs: ids uniform in [2,V); fixed lengths -> padded shapes exactly [Tx,B],[Ty,B];
    ragged: lengths uniform in [T/2, T] (one sentence per batch keeps the full length)."""
    from nats_b200.nats import prepare_data
    B = B or w['B']
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        if ragged:
            lx = rng.randint(w['Tx'] // 2, w['Tx'], size=B); ly = rng.randint(w['Ty'] // 2, w['Ty'], size=B)
        else:
            lx = np.full(B, w['Tx'] - 1); ly = np.full(B, w['Ty'] - 1)
        sx = [list(rng.randint(2, w['n_words'], size=int(l))) for l in lx]
        sy = [list(rng.randint(2, w['n_words'], size=int(l))) for l in ly]
        out.append(prepare_data(sx, sy, n_words=w['n_words']))
    return out


def options_of(w):
    return dict(dim_word=w['dim_word'], dim=w['dim'], dim_att=w['dim_att'], n_words=w['n_words'], encoder='gru',
                decoder='gru_cond')


def load_peaks():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return d.get('hbm_gbs', 6650.0), d.get('bf16_tflops_sustained', 1400.0), 'measured (MEASURED_PEAKS.json)'
    return 3350.0, 495.0, 'NVIDIA H100 SXM data sheet (HBM3 3.35 TB/s, dense TF32 495 TFLOP/s), not measured'


class ClockSampler(object):
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ('clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,'
         'clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap')

    def __init__(self, index):
        self.rows = []
        self.proc = None
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(index), '--query-gpu=' + self.Q,
                                          '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if self.proc is None:
            return None
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], 0, set()
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        rows = [r for (t, r) in self.rows if t0 - 0.05 <= t <= t1 + 0.15] or [r for (_, r) in self.rows]
        for r in rows:
            f = [c.strip() for c in r.split(',')]
            try:
                sm.append(float(f[0])); mx = max(mx, float(f[1]))
            except Exception:
                continue
            for nme, val in zip(names, f[2:6]):
                if val.lower().startswith('active'):
                    reasons.add(nme)
        if not sm:
            return None
        return {'sm_mhz': float(np.median(sm)), 'sm_max_mhz': mx, 'reasons': sorted(reasons), 'samples': len(sm)}


# ----------------------------------------------------------------------------------------------- CPU arm (oracle/)
_BLAS_CHOICE = {}


def best_blas_threads(w=None):
    """OpenBLAS with every host thread is pathologically slow on the skinny products of the
    recurrence; pick the thread count that is fastest on a SHORT real piece of the workload (a forward + backward pass of
    the restatement at the workload's dim / |V| / batch with src_len 40, tgt_len 6) so that the CPU baseline is a fair one."""
    try:
        from threadpoolctl import threadpool_limits
    except Exception:
        return None, os.cpu_count()
    ncpu = os.cpu_count() or 1
    key = None if w is None else (w['dim'], w['n_words'], w['B'])
    if key in _BLAS_CHOICE:
        return threadpool_limits, _BLAS_CHOICE[key]
    w = w or WORKLOADS['c3']
    from oracle import nats_oracle as O
    np.random.seed(7)
    P = O.init_params(options_of(w))
    small = dict(w, Tx=40, Ty=6)
    x, xm, y, ym = make_batches(small, 1, seed=3, B=min(w['B'], 32))[0]
    best = (None, 1e30)
    for t in sorted(set([8, 16, 32, 64, ncpu])):
        if t > ncpu:
            continue
        with threadpool_limits(limits=t):
            O.f_grad(P, x, xm, y, ym, clip_c=100.)
            t0 = time.perf_counter()
            O.f_grad(P, x, xm, y, ym, clip_c=100.)
            dt = time.perf_counter() - t0
        if dt < best[1]:
            best = (t, dt)
    _BLAS_CHOICE[key] = best[0]
    return threadpool_limits, best[0]


def _with_threads(fn, w=None):
    limiter, nthreads = best_blas_threads(w)
    if limiter is not None:
        with limiter(limits=nthreads):
            r = fn()
    else:
        r = fn()
    r['cores'] = nthreads
    r['sample'] += '; BLAS threads chosen by timing a short pass of the same model, out of %d host threads' % (os.cpu_count() or 1)
    return r


def cpu_train_step(w, steps, warmup, budget_s=None):
    """R2 on the host: float32 restatement, FULL batch of the workload, adadelta + clip as the GPU arm."""
    def run():
        from oracle import nats_oracle as O
        opts = options_of(w)
        np.random.seed(1234)
        P = O.init_params(opts)
        opt = O.Adadelta(P)
        times, cost, t_begin = [], 0.0, time.perf_counter()
        batches = make_batches(w, warmup + steps, seed=1234)
        for i, (x, xm, y, ym) in enumerate(batches):
            t0 = time.perf_counter()
            cost, G, _ = O.f_grad(P, x, xm, y, ym, clip_c=100.)
            opt.grad_shared(G)
            opt.update(P)
            dt = time.perf_counter() - t0
            if i >= warmup:
                times.append(dt)
            if budget_s is not None and i >= warmup and time.perf_counter() - t_begin > budget_s:
                break
        tokens = float(batches[0][3].sum())
        total = float(np.sum(times))
        return dict(value=tokens * len(times) / total, ms_per_step=1e3 * total / len(times), steps_timed=len(times),
                    sample='full batch: all %d sentences (Tx=%d, Ty=%d), %d timed train steps after %d warm-up'
                           % (w['B'], w['Tx'], w['Ty'], len(times), warmup), cost=float(cost))
    return _with_threads(run, w)


def cpu_decoder_forward(w, reps=2):
    """R1 on the host: decoder scan + readout + NLL on a precomputed context (nats.py:737-770), float32, full batch."""
    def run():
        from oracle import nats_oracle as O
        opts = options_of(w)
        np.random.seed(1234)
        P = O.init_params(opts)
        x, xm, y, ym = make_batches(w, 1, seed=1234)[0]
        _, cache = O.model_fwd(P, x, xm, y, ym)
        ctx, init_state, embs = cache['ctx'], cache['init_state'], cache['embs']
        Ty, B = y.shape
        ts = []
        for _ in range(reps + 1):
            t0 = time.perf_counter()
            (Hs, Cs, As, _, _), _ = O.gru_cond_layer_fwd(P, embs, ym, ctx, xm, init_state)
            pre = (Hs @ P['ff_logit_lstm_W'] + P['ff_logit_lstm_b'] + embs @ P['ff_logit_prev_W'] + P['ff_logit_prev_b']
                   + Cs @ P['ff_logit_ctx_W'] + P['ff_logit_ctx_b'])
            lg = (np.tanh(pre) @ P['ff_logit_W'] + P['ff_logit_b']).reshape(Ty * B, -1)
            mx = lg.max(1, keepdims=True)
            lse = mx[:, 0] + np.log(np.exp(lg - mx).sum(1))
            cost = ((lse - lg[np.arange(Ty * B), y.flatten()]).reshape(Ty, B) * ym).sum(0)
            ts.append(time.perf_counter() - t0)
        t = float(np.median(ts[1:]))
        return dict(value=float(ym.sum()) / t, ms=1e3 * t, sample='full batch (%d sentences), median of %d decoder-forward passes'
                    % (B, reps), cost=float(cost.mean()))
    return _with_threads(run, w)


def cpu_beam_steps(w, steps=6):
    """R3 on the host: the literal gen_sample restatement (SciPy-style O(k*ii) penalty loop included) driven by the float32
    oracle f_init / f_next, beam 10, `steps` beam steps (EOS suppressed so that all 10 hypotheses stay alive)."""
    def run():
        from oracle import nats_oracle as O
        opts = options_of(w)
        np.random.seed(1234)
        P = O.init_params(opts)
        P['ff_logit_b'] = P['ff_logit_b'].copy(); P['ff_logit_b'][0] = -1e9
        rng = np.random.RandomState(4321)
        x = np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1,)).tolist() + [0], dtype='int64').reshape(-1, 1)
        t0 = time.perf_counter()
        s0, ctx0 = O.f_init(P, x)
        t_init = time.perf_counter() - t0
        fi = lambda x_: (s0, ctx0)
        fn = lambda y_, c_, s_, ac_, aa_: O.f_next(P, y_, c_, s_.astype('float32'), ac_.astype('float32'), aa_.astype('float32'))
        t0 = time.perf_counter()
        O.gen_sample(fi, fn, x, k=10, maxlen=steps, stochastic=False, use_unk=True, kl_factor=1.0, ctx_factor=1.0, state_factor=1.0)
        dt = time.perf_counter() - t0
        live = 1 + 10 * (steps - 1)                      # hypotheses expanded: 1 at the first step, 10 afterwards
        return dict(value=live / dt, ms_per_step=1e3 * dt / steps, f_init_ms=1e3 * t_init,
                    sample='%d beam steps at beam 10 (src_len %d) of the restated gen_sample + 1 f_init' % (steps, w['Tx'] - 1))
    return _with_threads(run, w)


# ----------------------------------------------------------------------------------------------- GPU side helpers
def kernel_table(torch, run_step, steps=2):
    """Per-kernel device time of `steps` REPLAYED steps from the CUPTI activity trace (torch.profiler): the same graphs the
    headline timing replays -- no eager launches, no event brackets.  With programmatic dependent launch a kernel becomes
    resident (and starts its clock) while its predecessor is still running, so raw durations overlap; every kernel is
    therefore charged its EXCLUSIVE time = the part of [start, end] not already covered by kernels that started earlier.
    The exclusive times add up to the busy time of the GPU, which is <= the step time by construction.
    Returns {kernel name: (exclusive us, raw busy us, launches)}."""
    from torch.profiler import profile, ProfilerActivity
    run_step(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            run_step()
        torch.cuda.synchronize()
    evs = []
    for e in prof.events():
        if 'cuda' not in str(getattr(e, 'device_type', '')).lower():
            continue
        tr = e.time_range
        evs.append((float(tr.start), float(tr.end), e.name))
    evs.sort()
    rows, cover = {}, -1e30
    for st, en, name in evs:
        if 'nccl' in name.lower():
            # collectives run on their own stream UNDER the compute kernels (and spin while they wait for the peers): they
            # are listed with their raw duration and take no part in the exclusive-time attribution of the compute stream
            r = rows.setdefault(name, [0.0, 0.0, 0])
            r[1] += en - st; r[2] += 1
            continue
        excl = max(0.0, en - max(st, cover))
        cover = max(cover, en)
        r = rows.setdefault(name, [0.0, 0.0, 0])
        r[0] += excl; r[1] += en - st; r[2] += 1
    return dict((k, tuple(v)) for k, v in rows.items())


CLASSES = [   # (class, substring of the kernel name)
    ('enc_tc_fwd', 'enc_tc_kernel<32, false>'), ('enc_tc_fwd', 'enc_tc_kernel<64, false>'),
    ('enc_tc_fwd', 'enc_tc_kernelILi32ELb0'), ('enc_tc_fwd', 'enc_tc_kernelILi64ELb0'),
    ('enc_tc_bwd', 'enc_tc_kernel<32, true>'), ('enc_tc_bwd', 'enc_tc_kernel<64, true>'),
    ('enc_tc_bwd', 'enc_tc_kernelILi32ELb1'), ('enc_tc_bwd', 'enc_tc_kernelILi64ELb1'),
    ('tc_gemm_3xtf32_skinny', 'tma_gemm_ts_kernel'), ('tc_gemm_3xtf32', 'tma_gemm_kernel'), ('tc_gemm_3xtf32', 'tc_gemm_kernel'),
    ('sgemm_fp32', 'sgemm_kernel'), ('att_context', 'att_context_kernel'), ('att_scores', 'att_scores_kernel'),
    ('att_bwd_dalpha', 'att_bwd_dalpha'), ('att_bwd_softmax', 'att_bwd_softmax'), ('att_bwd_ctx', 'att_bwd_ctx'),
    ('att_bwd_reduce', 'att_bwd_reduce'), ('gru_gates_fwd', 'gru_gates_fwd'), ('gru_gates_bwd', 'gru_gates_bwd'),
    ('readout_nll', 'nll_rows'), ('readout_dlogits', 'dlogits'), ('optimizer', 'adadelta'), ('optimizer', 'grad_clip'),
    ('optimizer', 'clip_'), ('nccl', 'nccl'), ('memset', 'Memset'), ('memset', 'memset'), ('memcpy', 'Memcpy'),
]


def classify(rows, steps):
    out = {}
    for name, (excl_us, raw_us, cnt) in rows.items():
        cls = 'other'
        for c, sub in CLASSES:
            if sub in name:
                cls = c
                break
        d = out.setdefault(cls, {'ms_per_step': 0.0, 'raw_ms_per_step': 0.0, 'launches_per_step': 0.0})
        d['ms_per_step'] += excl_us / 1e3 / steps
        d['raw_ms_per_step'] += raw_us / 1e3 / steps
        d['launches_per_step'] += cnt / float(steps)
    for d in out.values():
        d['us_per_launch'] = 1e3 * d['ms_per_step'] / d['launches_per_step'] if d['launches_per_step'] else None
    return out


def algorithmic_work(graph, plan, f_update, accum):
    """algorithmic flops / bytes per step and kernel class from the library's own counters (one eager step; the counts do
    not depend on timing) -- merged into the CUPTI table for the roofline"""
    from nats_b200 import profiling
    k = profiling.probe(graph, plan, f_update, steps=1, accum=accum)
    return dict((n, (v['algo_gflop_per_step'], v['algo_gbytes_per_step'])) for n, v in k['classes'].items())


def region_r1(eng, _lib, graph, plan, tparams, w, tokens_per_step, n=10):
    """R1 = nats_decoder_scan_fwd + nats_readout_nll_fwd in one CUDA graph, CUDA events."""
    import ctypes
    import torch
    lib = eng.lib
    Tx, Ty, B = plan.shape
    vp = ctypes.c_void_p
    D = ctypes.byref(graph.dims)
    F, XM, Y, YM = vp(tparams.flat.data_ptr()), vp(plan.xm.data_ptr()), vp(plan.y.data_ptr()), vp(plan.ym.data_ptr())
    WS, C = vp(plan.ws.data_ptr()), vp(plan.cost.data_ptr())

    def r1():
        _lib.check(lib.nats_decoder_scan_fwd(eng.ctx, eng.stream(), D, F, Y, XM, YM, Tx, Ty, B, WS, plan.ws_bytes), 'scan')
        _lib.check(lib.nats_readout_nll_fwd(eng.ctx, eng.stream(), D, F, Y, YM, Tx, Ty, B, WS, plan.ws_bytes, C), 'readout')
    r1()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        r1()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    Dm, A, Cc = w['dim'], w['dim_att'], 2 * w['dim']
    step_bytes = 4.0 * (Tx * B * (Cc + A) + (12 * Dm * Dm + Dm * A) + B * (10 * Dm + 3 * Cc + 4 * Tx))   # SURVEY 8(d)
    hbm, _, src = load_peaks()
    ach = step_bytes * Ty / (ms * 1e-3) / 1e9
    rows = None
    try:
        rows = classify(kernel_table(torch, g.replay, 2), 2)
    except Exception as e:
        rows = {'error': repr(e)}
    return {'value': tokens_per_step / (ms * 1e-3), 'unit': 'tokens/s', 'ms': ms, 'us_per_decoder_step': 1e3 * ms / Ty,
            'region': 'decoder forward: gru_cond_layer scan + readout + softmax/NLL on a precomputed context (nats.py:737-770)',
            'roofline': {'bound': 'hbm', 'achieved': ach, 'peak': hbm, 'unit': 'GB/s', 'frac': ach / hbm,
                         'algo_bytes_per_decoder_step': step_bytes, 'hbm_floor_us_per_step': step_bytes / hbm / 1e3,
                         'peak_source': src, 'traffic': None},
            'kernels': rows, 'how': 'one CUDA graph, CUDA events, %d replays' % n}


def beam_run(nats, tparams, opts, w, steps, warm=True, kernels=False):
    """gen_sample at beam 10 with all three penalties; the EOS logit is pushed down so that all 10 hypotheses stay alive."""
    import torch
    rng = np.random.RandomState(4321)
    x = np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1,)).tolist() + [0], dtype='int64').reshape(-1, 1)
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    bsave = tparams['ff_logit_b'].get_value()
    bmod = bsave.copy()
    bmod[0] = -1e9
    tparams['ff_logit_b'].set_value(bmod)
    try:
        if warm:                                     # same maxlen as the timed run: buffers of that size, kernels loaded
            nats.gen_sample(tparams, f_init, f_next, x, opts, None, 10, steps, False, False, True, 1.0, 1.0, 1.0)
        torch.cuda.synchronize()
        f_init.device(x)                              # the call gen_sample makes (device tensors, no host copies); warm
        torch.cuda.synchronize()
        t1 = time.time()
        f_init.device(x)
        torch.cuda.synchronize()
        t_init = time.time() - t1
        t0 = time.time()
        result = nats.gen_sample(tparams, f_init, f_next, x, opts, None, 10, steps, False, False, True, 1.0, 1.0, 1.0)
        torch.cuda.synchronize()
        dt = time.time() - t0
    finally:
        tparams['ff_logit_b'].set_value(bsave)
    live = 1 + 10 * (steps - 1)
    out = {'ms_per_step': (dt - t_init) / steps * 1e3, 'f_init_ms': t_init * 1e3, 'steps': steps, 'sentence_ms': dt * 1e3,
           'hyp_tokens_per_s': live / max(dt - t_init, 1e-9),
           'how': 'gen_sample wall clock (host bookkeeping included) minus one f_init; beam 10, src_len %d, kl=ctx=state=1' % (w['Tx'] - 1)}
    samples, scores = result[0], result[1]
    toks = np.full((len(samples), max([len(s) for s in samples] + [1])), -1.0)
    for i, s in enumerate(samples):
        toks[i, :len(s)] = s
    outputs = {'beam_tokens': toks, 'beam_scores': np.asarray(scores, 'float64')}
    if kernels:
        # the same sentence under the CUPTI activity trace: launches and exclusive device time per kernel
        tparams['ff_logit_b'].set_value(bmod)
        try:
            rows = kernel_table(torch, lambda: nats.gen_sample(tparams, f_init, f_next, x, opts, None, 10, steps, False, False, True,
                                                               1.0, 1.0, 1.0), steps=1)
        finally:
            tparams['ff_logit_b'].set_value(bsave)
        launches = sum(v[2] for k_, v in rows.items() if 'memcpy' not in k_.lower() and 'memset' not in k_.lower())
        busy = sum(v[0] for v in rows.values())
        top = sorted(rows.items(), key=lambda kv: -kv[1][0])[:12]
        out['kernels'] = {'launches_per_sentence': int(launches), 'launches_per_step': launches / float(steps),
                          'gpu_busy_us_per_step_incl_f_init': busy / steps,
                          'top': [{'kernel': k_.replace('(anonymous namespace)::', '').replace('nats::', '').replace('void ', '').split('(')[0][:60],
                                   'excl_us': round(v[0], 1), 'launches': v[2]} for k_, v in top]}
    return out, outputs


def gen_throughput(nats, tparams, opts, w, n_sent=32, steps=25):
    """What gen.py does per worker: a stream of source sentences, beam 10 each.  With f_init.prefetch the 16 encoders run
    as ONE masked launch of the persistent kernel; without, one launch per sentence.  EOS is suppressed: every sentence
    runs all `steps` steps (a summary-sized output)."""
    import torch
    rng = np.random.RandomState(99)
    xs = [np.array(rng.randint(2, w['n_words'], size=(w['Tx'] - 1 - 7 * (i % 16),)).tolist() + [0], dtype='int64') for i in range(n_sent)]
    f_init, f_next = nats.build_sampler(tparams, opts, None)
    bsave = tparams['ff_logit_b'].get_value()
    bmod = bsave.copy()
    bmod[0] = -1e9
    tparams['ff_logit_b'].set_value(bmod)
    out = {}
    try:
        for mode in ('one_f_init_per_sentence', 'prefetch_16', 'prefetch_16_and_12_searches_in_flight'):
            for rep in range(2):                              # first pass warms buffers and kernels
                torch.cuda.synchronize()
                t0 = time.time()
                if mode == 'prefetch_16_and_12_searches_in_flight':
                    nats.gen_sample_many(tparams, f_init, f_next, xs, opts, None, 10, steps, True, 1.0, 1.0, 1.0, concurrency=12, chunk=16)
                else:
                    for i, x in enumerate(xs):
                        if mode == 'prefetch_16' and i % 16 == 0:
                            f_init.prefetch(xs[i:i + 16])
                        nats.gen_sample(tparams, f_init, f_next, x[:, None], opts, None, 10, steps, False, False, True, 1.0, 1.0, 1.0)
                torch.cuda.synchronize()
                dt = time.time() - t0
            out[mode] = {'sentences_per_s': n_sent / dt, 'ms_per_sentence': dt / n_sent * 1e3,
                         'hyp_tokens_per_s': n_sent * (1 + 10 * (steps - 1)) / dt}
    finally:
        tparams['ff_logit_b'].set_value(bsave)
    out['how'] = '%d sentences of src_len %d..%d, beam 10, %d steps each, kl=ctx=state=1; wall clock incl. f_init and result copies' % (
        n_sent, w['Tx'] - 1 - 7 * 15, w['Tx'] - 1, steps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--workload', default='c3', choices=sorted(WORKLOADS))
    ap.add_argument('--ragged', action='store_true', help='e2e on batches with lengths uniform in [T/2, T] (shape buckets)')
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--no-regions', action='store_true', help='skip the R1 (decoder forward) / R3 (beam step) measurements')
    ap.add_argument('--no-kernels', action='store_true', help='skip the CUPTI per-kernel table')
    ap.add_argument('--dump-outputs', metavar='DIR', help='write the outputs of the last timed step to DIR/<name>.npy')
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    w = WORKLOADS[args.workload]
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    warmup = max(args.warmup, 3) if args.impl == 'ours' else max(args.warmup, 1)
    beam = args.workload == 'c5'

    config = {'workload': w['name'],
              'region': 'beam step: f_next + distraction re-rank + bookkeeping (nats.py:957-1066)' if beam else
                        'train step: f_grad_shared + f_update (nats.py:1400-1411)',
              'global_batch': w['B'] * max(world, 1), 'src_len': w['Tx'] - (1 if beam else 0), 'tgt_len': w['Ty'],
              'parallelism': 'dp%d' % max(world, 1),
              'l2_policy': 'per-step working set (saved activations + weights, > 2 GB) exceeds the 50 MB L2'}
    if not beam:
        config.update({'optimizer': 'adadelta', 'clip_c': 100.0})

    if args.impl == 'reference':
        if rank != 0:
            return 0
        if beam:
            r = cpu_beam_steps(w, steps=min(args.steps, 8))
            ms = r['ms_per_step']
        else:
            r = cpu_train_step(w, args.steps, warmup)
            ms = r['ms_per_step']
        line = {'impl': 'reference', 'metric': METRIC, 'value': r['value'], 'unit': 'tokens/s', 'n_gpus': args.gpus,
                'steps': args.steps, 'warmup': warmup, 'ms_per_step': ms, 'higher_is_better': True,
                'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic', 'config': config,
                'cpu_baseline': {'value': r['value'], 'unit': 'tokens/s', 'cores': r['cores'], 'kind': 'port',
                                 'sample': r['sample']},
                'e2e': {'value': r['value'], 'unit': 'tokens/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
                'gpu_launches': 0,
                'note': 'reference = NumPy/OpenBLAS float32 restatement of scripts/nats.py (oracle/) on the full batch; '
                        'Python 2 + Theano are not installable here'}
        print(json.dumps(line))
        return 0

    os.environ.setdefault('NCCL_DEBUG_FILE', '/dev/stderr')     # keep NCCL's banner off the one-JSON-line stdout
    # NCCL prints its version banner on stdout: keep stdout clean for the ONE JSON line (restored before it is printed)
    sys.stdout.flush()
    saved_stdout = os.dup(1)
    os.dup2(2, 1)
    import torch
    if world > 1:
        torch.cuda.set_device(local)
        torch.distributed.init_process_group('nccl', device_id=torch.device('cuda', local))
    from nats_b200 import nats, _lib
    eng = nats.get_engine()
    opts = options_of(w)
    np.random.seed(1234)
    params = nats.init_params(opts)
    import io
    import contextlib
    with contextlib.redirect_stdout(io.StringIO()):
        tparams = nats.init_tparams(params)

    if beam:
        if rank != 0:
            return 0
        K = args.steps
        clk = ClockSampler(local)
        t0 = time.time()
        r, outputs = beam_run(nats, tparams, opts, w, K, kernels=not args.no_kernels)
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, outputs)
        full = beam_run(nats, tparams, opts, w, 100, warm=False)[0]
        clocks = clk.stop(t0, time.time())
        Tx5, k5 = w['Tx'], 10
        d2h_sentence = 2 * k5 * K * Tx5 * 4 + 2 * k5 * K * 4 + 3 * k5 * 4 + 32     # attention histories (live + retired), tokens, scores, counters
        line = {'metric': METRIC, 'value': r['hyp_tokens_per_s'], 'unit': 'tokens/s', 'n_gpus': 1, 'steps': K, 'warmup': 4,
                'ms_per_step': r['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
                'dtype': 'f32', 'data': 'synthetic', 'config': config, 'clocks': clocks,
                'e2e': {'value': r['hyp_tokens_per_s'], 'unit': 'tokens/s', 'h2d_bytes_per_step': 8.0 * Tx5 / K,
                        'd2h_bytes_per_step': d2h_sentence / float(K),
                        'note': 'gen_sample is the public API: host loop included; the source sentence goes up once per '
                                'sentence, the search state stays on the device, results come back once at the end'},
                'beam': r, 'full_sentence_100_steps': full, 'gen_stream': gen_throughput(nats, tparams, opts, w),
                'gpu_launches': (r.get('kernels') or {}).get('launches_per_sentence')}
        if not args.no_cpu_baseline:
            c = cpu_beam_steps(w, steps=6)
            line['cpu_baseline'] = {'value': c['value'], 'unit': 'tokens/s', 'cores': c['cores'], 'kind': 'port',
                                    'sample': c['sample'], 'ms_per_step': c['ms_per_step'], 'f_init_ms': c['f_init_ms']}
        sys.stdout.flush(); os.dup2(saved_stdout, 1)
        print(json.dumps(line))
        return 0

    graph = nats.build_model(tparams, opts)[-1].mean()
    graph.clip_c = 100.0
    graph.lazy_cost = True
    f_grad_shared, f_update = nats.adadelta('lr', tparams, graph, None, graph)
    K = args.steps
    batches = make_batches(w, warmup + K, seed=1234 + rank, ragged=args.ragged)
    tokens_per_step = float(batches[0][3].sum()) if not args.ragged else float(np.mean([b[3].sum() for b in batches[warmup:]]))
    graph.reserve(w['Tx'], w['Ty'], w['B'])

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], dtype=torch.float64, device=eng.device)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return float(t.item())

    # ---------------- e2e: host numpy in, host scalar out, every step (cost reads pipelined by one step) ----------------
    costs = []
    for i in range(warmup):
        costs.append(float(f_grad_shared(*batches[i])))
        f_update(0.01)
    barrier()
    launches0 = eng.launches
    clk = ClockSampler(local) if rank == 0 else None
    t_wall0 = time.time()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pending = None
    ev0.record()
    for i in range(K):
        c = f_grad_shared(*batches[warmup + i])
        f_update(0.01)
        if pending is not None:
            costs.append(float(pending))          # device->host read of the previous step's result
        pending = c
    costs.append(float(pending))
    ev1.record()
    barrier()
    e2e_ms = max_over_ranks(ev0.elapsed_time(ev1))
    abi_calls = eng.launches - launches0
    n_plans = len(graph._plans)
    plan = graph.plan(w['Tx'], w['Ty'], w['B'])
    h2d = plan.h2d_bytes()

    # ---------------- device-resident: same steps, inputs already in HBM (full-shape plan) ----------------
    if plan.uses < 2:                                  # --ragged may never have produced the full shape
        full = make_batches(w, 1, seed=99)[0]
        for _ in range(2):
            float(f_grad_shared(*full)); f_update(0.01)
    main_stream = torch.cuda.current_stream(eng.device)

    def device_step():
        if world == 1:
            plan.graph_step.replay()
        elif not graph.overlap_allreduce:
            plan.graph_fb.replay()
            torch.distributed.all_reduce(graph.grads)
            plan.graph_post.replay()
        else:
            plan.graph_fb.replay()
            graph._side.wait_stream(main_stream)
            with torch.cuda.stream(graph._side):
                w1 = torch.distributed.all_reduce(graph.grads[graph.split:], async_op=True, group=graph._pg_side)
            plan.graph_fb2.replay()
            torch.distributed.all_reduce(graph.grads[:graph.split])
            w1.wait()
            main_stream.wait_stream(graph._side)
            plan.graph_post.replay()
        f_update(0.01)

    have_graphs = (plan.graph_step is not None) if world == 1 else (plan.graph_fb is not None)
    dev_ms = None
    if have_graphs:
        for _ in range(3):
            device_step()
        barrier()
        ev0.record()
        for _ in range(K):
            device_step()
        ev1.record()
        barrier()
        dev_ms = max_over_ranks(ev0.elapsed_time(ev1))
    if args.dump_outputs and rank == 0:
        # the last timed step's results: per-sentence costs, the flat gradient and the parameters after the update
        dump_outputs(args.dump_outputs, {'cost': plan.cost.cpu().numpy(), 'grads': graph.grads[:tparams.total].cpu().numpy(),
                                         'params': tparams.flat.cpu().numpy()})
    t_wall1 = time.time()
    clocks = clk.stop(t_wall0, t_wall1) if clk is not None else None

    # ---------------- per-kernel table from the replayed step (CUPTI activity trace) ----------------
    kernels, roofline = None, None
    if have_graphs and not args.no_kernels:
        try:
            steps_p = 2
            rows = kernel_table(torch, device_step, steps_p)
            cls = classify(rows, steps_p)
            total = sum(v['ms_per_step'] for v in cls.values())
            for v in cls.values():
                v['share_of_step'] = v['ms_per_step'] / (dev_ms / K)
            if world == 1:
                try:
                    work = algorithmic_work(graph, plan, f_update, f_grad_shared.accum)
                    for n, (gf, gb) in work.items():
                        if n in cls:
                            cls[n]['algo_gflop_per_step'], cls[n]['algo_gbytes_per_step'] = gf, gb
                except Exception as e:
                    cls['_work_error'] = {'ms_per_step': 0.0, 'launches_per_step': 0.0, 'error': repr(e)}
            kernels = {'classes': cls, 'sum_kernel_ms_per_step': total, 'launches_per_step': sum(v['launches_per_step'] for v in cls.values()),
                       'how': 'CUPTI activity trace (torch.profiler) of %d replayed graph steps; ms_per_step = EXCLUSIVE time (a kernel '
                              'made resident early by programmatic dependent launch is not charged for the time its predecessor was still '
                              'running), raw_ms_per_step = start-to-end' % steps_p}
            roofline = roofline_of(cls, w, dev_ms / K)
        except Exception as e:
            kernels = {'error': repr(e)}
    if rank != 0:
        if world > 1:
            torch.distributed.destroy_process_group()
        return 0

    r1 = None
    if world == 1 and not args.no_regions:
        try:
            r1 = region_r1(eng, _lib, graph, plan, tparams, w, float(batches[0][3].sum()) if not args.ragged else w['B'] * w['Ty'])
        except Exception as e:       # diagnostics only
            r1 = {'error': repr(e)}
    r3 = None
    if world == 1 and args.workload == 'c3' and not args.no_regions:
        try:
            r3 = beam_run(nats, tparams, opts, WORKLOADS['c5'], 20)[0]
            r3['gen_stream'] = gen_throughput(nats, tparams, opts, WORKLOADS['c5'])      # sentences/s of the gen driver's loop
        except Exception as e:
            r3 = {'error': repr(e)}

    total_tokens = tokens_per_step * max(world, 1) * K
    value_ms = dev_ms if dev_ms is not None else e2e_ms
    dev_tokens = float(w['B'] * w['Ty']) * max(world, 1) * K
    line = {
        'metric': METRIC, 'value': dev_tokens / (value_ms * 1e-3), 'unit': 'tokens/s', 'n_gpus': max(world, 1),
        'steps': K, 'warmup': warmup, 'ms_per_step': value_ms / K, 'higher_is_better': True, 'scaling': 'weak',
        'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic', 'config': config,
        'e2e': {'value': total_tokens / (e2e_ms * 1e-3), 'unit': 'tokens/s', 'h2d_bytes_per_step': h2d,
                'd2h_bytes_per_step': 4, 'ms_per_step': e2e_ms / K, 'ragged': bool(args.ragged), 'plans_used': n_plans,
                'tokens_per_step': tokens_per_step,
                'how': 'f_grad_shared(host numpy) + f_update per step; packed pinned staging, one H2D copy, cost read back '
                       'every step (the read of step i is awaited after step i+1 is queued)'},
        'gpu_launches': None, 'abi_calls_timed': abi_calls,
        'clocks': clocks, 'roofline': roofline, 'r1': r1, 'r3_beam_step': r3, 'kernels': kernels,
        'cost_first_last': [costs[0], costs[-1]],
    }
    if kernels and 'launches_per_step' in kernels:
        line['gpu_launches'] = int(round(kernels['launches_per_step'] * K))
    if not args.no_cpu_baseline and world == 1:
        r = cpu_train_step(w, steps=2, warmup=1, budget_s=40)
        line['cpu_baseline'] = {'value': r['value'], 'unit': 'tokens/s', 'cores': r['cores'], 'kind': 'port',
                                'sample': r['sample'], 'ms_per_step': r['ms_per_step']}
        if r1 and 'value' in r1:
            c1 = cpu_decoder_forward(w)
            r1['cpu_baseline'] = {'value': c1['value'], 'unit': 'tokens/s', 'cores': c1['cores'], 'kind': 'port', 'sample': c1['sample'], 'ms': c1['ms']}
        if r3 and 'hyp_tokens_per_s' in r3:
            c3 = cpu_beam_steps(WORKLOADS['c5'], steps=5)
            r3['cpu_baseline'] = {'value': c3['value'], 'unit': 'tokens/s', 'cores': c3['cores'], 'kind': 'port', 'sample': c3['sample'],
                                  'ms_per_step': c3['ms_per_step'], 'f_init_ms': c3['f_init_ms']}
    sys.stdout.flush(); os.dup2(saved_stdout, 1)
    print(json.dumps(line))
    sys.stdout.flush()
    if world > 1:
        torch.distributed.destroy_process_group()
    return 0


def roofline_of(cls, w, step_ms):
    """`roofline` of the bench line for the dominant kernel class of the replayed step.
    enc_tc_*: tensor-bound by construction (weights stay on chip: no weight traffic) -> algorithmic fp32 flops of the
    recurrence / launch duration against the measured dense peak; the limiter is named.
    att_* / optimizer: HBM streams -> algorithmic bytes / duration against the measured copy bandwidth."""
    hbm, tf, src = load_peaks()
    name = max((k for k in cls if k not in ('other', 'memcpy', 'memset')), key=lambda k: cls[k]['ms_per_step'])
    k = cls[name]
    Tx, Ty, B, D, A = w['Tx'], w['Ty'], w['B'], w['dim'], w['dim_att']
    us = k['us_per_launch']
    base = {'kernel': name, 'share_of_step': k['ms_per_step'] / step_ms, 'us_per_launch': us, 'peak_source': src,
            'duration_source': 'CUPTI activity trace of the replayed graph step'}
    traffic = None
    if name.startswith('enc_tc'):
        flops = 2.0 * 2 * (Tx - 1) * B * D * 3 * D            # both directions, fp32-equivalent (each is 3 tf32 products)
        ach = flops / (us * 1e-6) / 1e12
        base.update({'bound': 'tensor', 'achieved': ach, 'peak': tf, 'unit': 'TFLOP/s', 'frac': ach / tf,
                     'algo_flops_per_launch': flops, 'traffic': traffic,
                     'limiter': 'inter-SM dependency latency: 2 L2 exchange hops per recurrent step (K partials, then h_t / dG_t); '
                                'the tensor pipe itself is busy a fraction of the step (3xTF32 wgmma per k-step, 189 x 32 x 256 per CTA and step)',
                     'us_per_recurrent_step': us / Tx})
        return base
    if name.startswith('tc_gemm'):
        gf = k.get('algo_gflop_per_step')
        ach = gf / k['ms_per_step'] if gf else None          # GFLOP / ms = TFLOP/s
        base.update({'bound': 'tensor', 'achieved': ach, 'peak': tf, 'unit': 'TFLOP/s', 'frac': ach / tf if ach else None, 'traffic': None,
                     'algo_gflop_per_step': gf,
                     'note': 'fp32-equivalent flops: every product is 3 tf32 wgmma MMAs (3xTF32), so the tensor pipe executes 3x this'})
        return base
    C = 2 * D
    bytes_per_launch = {'att_context': 4.0 * (Tx * B * C + 3 * B * C + 3 * B * Tx), 'att_bwd_dalpha': 4.0 * (Tx * B * C + 2 * B * C + B * Tx)}.get(name)
    ach = bytes_per_launch / (us * 1e-6) / 1e9 if bytes_per_launch else None
    base.update({'bound': 'hbm', 'achieved': ach, 'peak': hbm, 'unit': 'GB/s', 'frac': ach / hbm if ach else None,
                 'algo_bytes_per_launch': bytes_per_launch, 'traffic': None})
    return base


if __name__ == '__main__':
    sys.exit(main())
