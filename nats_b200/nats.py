"""
nats_b200.nats -- host side of the H100 implementation of lukecq1231/nats' hot path.

Same public surface as the reference's scripts/nats.py so that its drivers (train_nats.py, gen.py) keep working:

    init_params, init_tparams, load_params, zipp, unzip, itemlist, prepare_data,
    build_model, build_sampler, gen_sample, pred_probs, adadelta / adam / rmsprop / sgd, train

but there is no Theano graph underneath: every compiled callable of the reference (f_init, f_next, f_log_probs,
f_cost, f_grad_shared, f_update -- nats.py:817, 871, 1320, 1336, 1160, 1170) is a thin Python closure over
libnats_b200.so (include/nats_b200.h), called through ctypes with raw device pointers.  PyTorch is used as the
container for device memory, streams, CUDA graphs and NCCL only.

There is no CPU fallback: without the CUDA library and an H100 the compiled callables raise NatsB200Error.
Pure-host helpers (init_params, prepare_data, load_params, the beam bookkeeping of gen_sample) work anywhere.
"""
from collections import OrderedDict
import copy
import ctypes
import logging
import os
import pickle as pkl
import pprint
import sys
import time
import warnings

import numpy

from . import _lib
from . import parallel
from ._lib import Dims, NatsB200Error
from .data_iterator import TextIterator

logger = logging.getLogger(__name__)
profile = False


# ----------------------------------------------------------------------------------------------------------
# parameter dictionaries (reference: nats.py:31-46, 66-89, 118-142, 251-260, 271-302, 378-451, 613-654)
# ----------------------------------------------------------------------------------------------------------
def zipp(params, tparams):
    """push host arrays into the device store (nats.py:31-33)"""
    for kk, vv in params.items():
        tparams[kk].set_value(vv)


def unzip(zipped):
    """pull the device store into host arrays (nats.py:37-41)"""
    return OrderedDict((kk, vv.get_value()) for kk, vv in zipped.items())


def itemlist(tparams):
    return [vv for _, vv in tparams.items()]


def _p(pp, name):
    return '%s_%s' % (pp, name)


def ortho_weight(ndim):
    W = numpy.random.randn(ndim, ndim)
    u, _, _ = numpy.linalg.svd(W)
    return u.astype('float32')


def norm_weight(nin, nout=None, scale=0.01, ortho=True):
    if nout is None:
        nout = nin
    if nout == nin and ortho:
        return ortho_weight(nin)
    return (scale * numpy.random.randn(nin, nout)).astype('float32')


def param_init_fflayer(options, params, prefix='ff', nin=None, nout=None, ortho=True):
    nin = options['dim_proj'] if nin is None else nin
    nout = options['dim_proj'] if nout is None else nout
    params[_p(prefix, 'W')] = norm_weight(nin, nout, scale=0.01, ortho=ortho)
    params[_p(prefix, 'b')] = numpy.zeros((nout,), dtype='float32')
    return params


def param_init_gru(options, params, prefix='gru', nin=None, dim=None):
    nin = options['dim_proj'] if nin is None else nin
    dim = options['dim_proj'] if dim is None else dim
    params[_p(prefix, 'W')] = numpy.concatenate([norm_weight(nin, dim), norm_weight(nin, dim)], axis=1)
    params[_p(prefix, 'b')] = numpy.zeros((2 * dim,), dtype='float32')
    params[_p(prefix, 'U')] = numpy.concatenate([ortho_weight(dim), ortho_weight(dim)], axis=1)
    params[_p(prefix, 'Wx')] = norm_weight(nin, dim)
    params[_p(prefix, 'bx')] = numpy.zeros((dim,), dtype='float32')
    params[_p(prefix, 'Ux')] = ortho_weight(dim)
    return params


def param_init_gru_cond(options, params, prefix='gru_cond', nin=None, dim=None, dimctx=None, dimatt=None):
    nin = options['dim'] if nin is None else nin
    dim = options['dim'] if dim is None else dim
    dimctx = options['dim'] if dimctx is None else dimctx
    dimatt = options['dim'] if dimatt is None else dimatt
    z = lambda *s: numpy.zeros(s, dtype='float32')
    # GRU_2 (previous state -> intermediate state), input = target embedding
    params[_p(prefix, 'W')] = numpy.concatenate([norm_weight(nin, dim), norm_weight(nin, dim)], axis=1)
    params[_p(prefix, 'U')] = numpy.concatenate([ortho_weight(dim), ortho_weight(dim)], axis=1)
    params[_p(prefix, 'b')] = z(2 * dim)
    params[_p(prefix, 'Wx')] = norm_weight(nin, dim)
    params[_p(prefix, 'Ux')] = ortho_weight(dim)
    params[_p(prefix, 'bx')] = z(dim)
    # GRU_1 (intermediate state -> new state), input = context vector
    params[_p(prefix, 'U_1')] = numpy.concatenate([ortho_weight(dim), ortho_weight(dim)], axis=1)
    params[_p(prefix, 'W_1')] = norm_weight(dimctx, dim * 2)
    params[_p(prefix, 'b_1')] = z(2 * dim)
    params[_p(prefix, 'Wx_1')] = norm_weight(dimctx, dim)
    params[_p(prefix, 'Ux_1')] = ortho_weight(dim)
    params[_p(prefix, 'bx_1')] = z(dim)
    # attention MLP
    params[_p(prefix, 'W_att')] = norm_weight(dim, dimatt)
    params[_p(prefix, 'Wc_att')] = norm_weight(dimctx, dimatt)
    params[_p(prefix, 'b_att')] = z(dimatt)
    params[_p(prefix, 'U_att')] = norm_weight(dimatt, 1)
    params[_p(prefix, 'c_att')] = z(1)
    # distraction: over context vectors (W_con, U_con) and over attention weights (D_wei)
    params[_p(prefix, 'W_con')] = norm_weight(dimctx, 1)
    params[_p(prefix, 'U_con')] = norm_weight(dimctx, 1)
    params[_p(prefix, 'D_wei')] = norm_weight(1, dimatt)
    return params


layers = {'ff': ('param_init_fflayer', 'fflayer'),
          'gru': ('param_init_gru', 'gru_layer'),
          'gru_cond': ('param_init_gru_cond', 'gru_cond_layer')}


def _layer_is_fused(*_a, **_k):
    raise NatsB200Error('layer feed-forward functions are fused into libnats_b200 kernels; use build_model / '
                        'build_sampler')


fflayer = gru_layer = gru_cond_layer = _layer_is_fused


def get_layer(name):
    fns = layers[name]
    return (globals()[fns[0]], globals()[fns[1]])


def init_params(options):
    """The 43 tensors in the reference's order (nats.py:613-654); numpy's global RNG, like the reference."""
    if options.get('encoder', 'gru') != 'gru' or options.get('decoder', 'gru_cond') != 'gru_cond':
        raise ValueError("only encoder='gru', decoder='gru_cond' exist (as in the reference's layer registry)")
    params = OrderedDict()
    params['Wemb'] = norm_weight(options['n_words'], options['dim_word'])
    params = param_init_gru(options, params, prefix='encoder', nin=options['dim_word'], dim=options['dim'])
    params = param_init_gru(options, params, prefix='encoder_r', nin=options['dim_word'], dim=options['dim'])
    ctxdim = 2 * options['dim']
    params = param_init_fflayer(options, params, prefix='ff_state', nin=ctxdim, nout=options['dim'])
    params = param_init_gru_cond(options, params, prefix='decoder', nin=options['dim_word'], dim=options['dim'],
                                 dimctx=ctxdim, dimatt=options['dim_att'])
    params = param_init_fflayer(options, params, prefix='ff_logit_lstm', nin=options['dim'],
                                nout=options['dim_word'], ortho=False)
    params = param_init_fflayer(options, params, prefix='ff_logit_prev', nin=options['dim_word'],
                                nout=options['dim_word'], ortho=False)
    params = param_init_fflayer(options, params, prefix='ff_logit_ctx', nin=ctxdim, nout=options['dim_word'],
                                ortho=False)
    params = param_init_fflayer(options, params, prefix='ff_logit', nin=options['dim_word'],
                                nout=options['n_words'])
    return params


def load_params(path, params):
    """nats.py:81-89: fill `params` from an .npz archive, warn on (and skip) missing keys."""
    pp = numpy.load(path, allow_pickle=True)
    for kk in list(params.keys()):
        if kk not in pp:
            warnings.warn('%s is not in the archive' % kk)
            continue
        params[kk] = pp[kk]
    return params


def prepare_data(seqs_x, seqs_y, maxlen=None, n_words=30000):
    """Batch layout contract of the hot path (nats.py:200-247): long sequences are cut to maxlen-1 tokens,
    arrays are time-major and zero padded, masks carry len+1 ones (the implicit EOS row)."""
    def clip(seqs):
        if maxlen is None:
            return list(seqs)
        return [s[:maxlen - 1] if len(s) >= maxlen else s for s in seqs]
    seqs_x, seqs_y = clip(seqs_x), clip(seqs_y)
    if maxlen is not None and (len(seqs_x) < 1 or len(seqs_y) < 1):
        return None, None, None, None
    lx = [len(s) for s in seqs_x]
    ly = [len(s) for s in seqs_y]
    n_samples = len(seqs_x)
    x = numpy.zeros((max(lx) + 1, n_samples), dtype='int64')
    y = numpy.zeros((max(ly) + 1, n_samples), dtype='int64')
    x_mask = numpy.zeros(x.shape, dtype='float32')
    y_mask = numpy.zeros(y.shape, dtype='float32')
    for idx in range(n_samples):
        x[:lx[idx], idx] = seqs_x[idx]
        x_mask[:lx[idx] + 1, idx] = 1.
        y[:ly[idx], idx] = seqs_y[idx]
        y_mask[:ly[idx] + 1, idx] = 1.
    return x, x_mask, y, y_mask


# ----------------------------------------------------------------------------------------------------------
# device store: the replacement of theano.shared (nats.py:72-77)
# ----------------------------------------------------------------------------------------------------------
def _dims_from_shapes(shapes):
    V, W = shapes['Wemb']
    D = shapes['encoder_Ux'][0]
    A = shapes['decoder_W_att'][1]
    return int(V), int(W), int(D), int(A)


class DeviceParam(object):
    """One reference-named tensor living inside the flat device buffer (a strided view of the packed layout).
    Offers the two methods the reference uses on shared variables: get_value / set_value."""

    def __init__(self, store, name, offset, rows, cols, ld, ndim):
        self.store, self.name = store, name
        self.offset, self.rows, self.cols, self.ld, self.ndim = offset, rows, cols, ld, ndim

    @property
    def shape(self):
        return (self.cols,) if self.ndim == 1 else (self.rows, self.cols)

    def _view(self, flat):
        return flat.as_strided((self.rows, self.cols), (self.ld, 1), self.offset)

    def get_value(self, borrow=False):
        arr = self._view(self.store.flat).cpu().numpy()
        return arr.reshape(self.shape).copy()

    def set_value(self, value, borrow=False):
        import torch
        value = numpy.ascontiguousarray(numpy.asarray(value, dtype='float32')).reshape(self.rows, self.cols)
        self._view(self.store.flat).copy_(torch.from_numpy(value))

    def __repr__(self):
        return '<DeviceParam %s %s>' % (self.name, self.shape)


class TParams(OrderedDict):
    """OrderedDict name -> DeviceParam (reference order) + the flat device buffer they live in."""

    def __init__(self, dims, engine):
        super(TParams, self).__init__()
        import torch
        self.dims = dims                      # (V, W, D, A)
        self.engine = engine
        views, total = _lib.param_layout(*dims)
        self.total = total
        self.flat = torch.zeros(total, dtype=torch.float32, device=engine.device)
        for (name, off, rows, cols, ld, ndim) in views:
            OrderedDict.__setitem__(self, name, DeviceParam(self, name, off, rows, cols, ld, ndim))

    def view_of(self, flat_like):
        """dict name -> host array for another flat buffer with the same layout (gradients, optimiser state)"""
        return OrderedDict((k, v._view(flat_like).cpu().numpy().reshape(v.shape).copy()) for k, v in self.items())


def init_tparams(params, engine=None):
    """numpy dict -> device store (nats.py:72-77).  Needs an H100; prints 'name shape' like the reference."""
    shapes = OrderedDict((k, numpy.shape(v)) for k, v in params.items())
    dims = _dims_from_shapes(shapes)
    engine = engine or get_engine()
    tparams = TParams(dims, engine)
    if list(tparams.keys()) != list(params.keys()):
        raise ValueError('parameter names/order differ from the reference layout (nats.py:613-654)')
    for kk, pp in params.items():
        if tuple(tparams[kk].shape) != tuple(numpy.shape(pp)):
            raise ValueError('%s: shape %s, expected %s' % (kk, numpy.shape(pp), tparams[kk].shape))
        tparams[kk].set_value(pp)
        print(kk, numpy.shape(pp))
    return tparams


# ----------------------------------------------------------------------------------------------------------
# engine: context handle, workspaces, CUDA graphs
# ----------------------------------------------------------------------------------------------------------
_ENGINE = None


def get_engine():
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine()
    return _ENGINE


class Engine(object):
    def __init__(self, device_index=None):
        import torch
        self.torch = torch
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise NatsB200Error('no CUDA device visible: nats_b200 runs on H100 (sm_90a) only, there is no CPU path')
        if device_index is None:
            device_index = int(os.environ.get('LOCAL_RANK', torch.cuda.current_device()))
        torch.cuda.set_device(device_index)
        self.device = torch.device('cuda', device_index)
        h = ctypes.c_void_p()
        _lib.check(self.lib.nats_ctx_create(device_index, ctypes.byref(h)), 'nats_ctx_create')
        self.ctx = h
        self.launches = 0          # C-ABI calls issued (each one enqueues many kernels)
        self._ws = {}

    def stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def workspace(self, key, nbytes):
        t = self._ws.get(key)
        if t is None or t.numel() < nbytes:
            self._ws[key] = None
            t = self.torch.empty(int(nbytes), dtype=self.torch.uint8, device=self.device)
            self._ws[key] = t
        return t


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _bucket(n, q):
    """round n up to a multiple of q (q <= 1: no bucketing)"""
    return int(n) if q <= 1 else ((int(n) + q - 1) // q) * q


class _Arena(object):
    """Storage shared by every plan of a ModelGraph: ONE workspace sized for the largest shape seen, one packed device
    input buffer (x | y | x_mask | y_mask) and its pinned host mirror -> one H2D copy per step.  Plans are views; when the
    arena has to grow (a larger shape than any before) every captured CUDA graph is dropped with the old addresses."""

    def __init__(self, model):
        self.model = model
        self.ws = None
        self.ws_bytes = 0
        self.inp = None         # uint8 device buffer
        self.pin = None         # uint8 pinned host mirror
        self.inp_bytes = 0
        self.version = 0

    @staticmethod
    def input_layout(Tx, Ty, B):
        ox = 0
        oy = ox + Tx * B * 8
        oxm = oy + Ty * B * 8
        oym = oxm + Tx * B * 4
        return ox, oy, oxm, oym, oym + Ty * B * 4

    def reserve(self, Tx, Ty, B):
        eng = self.model.engine
        torch = eng.torch
        need_ws = int(eng.lib.nats_train_workspace_bytes(ctypes.byref(self.model.dims), Tx, Ty, B))
        if need_ws <= 0:
            raise NatsB200Error('nats_train_workspace_bytes failed')
        need_in = self.input_layout(Tx, Ty, B)[4]
        grown = False
        if need_ws > self.ws_bytes:
            self.ws = None
            self.ws = torch.empty(need_ws, dtype=torch.uint8, device=eng.device)
            self.ws_bytes = need_ws
            grown = True
        if need_in > self.inp_bytes:
            self.inp = torch.zeros(need_in, dtype=torch.uint8, device=eng.device)
            self.pin = torch.zeros(need_in, dtype=torch.uint8).pin_memory()
            self.inp_bytes = need_in
            grown = True
        if grown:
            self.version += 1
        return need_ws


class _TrainPlan(object):
    """Everything bound to one (Tx, Ty, B) shape: views of the arena's input buffers and workspace, optional CUDA graphs."""

    def __init__(self, model, Tx, Ty, B):
        torch = model.engine.torch
        arena = model.arena
        self.shape = (Tx, Ty, B)
        self.ws_bytes = arena.reserve(Tx, Ty, B)
        self.arena_version = arena.version
        self.ws = arena.ws
        ox, oy, oxm, oym, end = arena.input_layout(Tx, Ty, B)
        self.in_bytes = end

        def views(buf):
            return (buf[ox:oy].view(torch.int64).view(Tx, B), buf[oy:oxm].view(torch.int64).view(Ty, B),
                    buf[oxm:oym].view(torch.float32).view(Tx, B), buf[oym:end].view(torch.float32).view(Ty, B))
        self.x, self.y, self.xm, self.ym = views(arena.inp)
        self.hx, self.hy, self.hxm, self.hym = [t.numpy() for t in views(arena.pin)]      # numpy views of the pinned mirror
        self.dev_in, self.pin_in = arena.inp[:end], arena.pin[:end]
        self.cost = torch.zeros((B,), dtype=torch.float32, device=model.engine.device)
        self.graph_fwd = None      # forward only (f_log_probs)
        self.graph_fb = None       # forward + first half of the backward (data-parallel)
        self.graph_fb2 = None      # second half of the backward (encoder), overlapped with the first all-reduce
        self.graph_post = None     # L2 / clip / optimiser accumulators
        self.graph_step = None     # single GPU: forward + backward + post in one graph
        self.uses = 0

    def stage(self, x, x_mask, y, y_mask):
        """host arrays (any shape <= the plan's: the rest is zero padding, masked out) -> pinned mirror -> ONE H2D copy"""
        Tx, Ty, B = self.shape
        for dst, src in ((self.hx, x), (self.hxm, x_mask), (self.hy, y), (self.hym, y_mask)):
            t = src.shape[0]
            dst[:t] = src
            if t < dst.shape[0]:
                dst[t:] = 0
        self.dev_in.copy_(self.pin_in, non_blocking=True)

    def h2d_bytes(self):
        return int(self.in_bytes)


class LazyCost(object):
    """The scalar cost of a step whose device->host read is still in flight (pinned buffer + event).  float() / numpy
    conversion waits for it; the training loop of the reference converts immediately, a pipelined caller (bench.py)
    converts one step later and keeps the GPU queue full."""

    def __init__(self, host_buf, event, extra=0.0):
        self._buf, self._ev, self._extra, self._v = host_buf, event, extra, None

    def value(self):
        if self._v is None:
            self._ev.synchronize()
            self._v = numpy.float32(float(self._buf[0]) + self._extra)
        return self._v

    def __float__(self):
        return float(self.value())

    def __array__(self, dtype=None, copy=None):
        return numpy.asarray(self.value(), dtype=dtype)

    def __repr__(self):
        return repr(self.value())


class ModelGraph(object):
    """What build_model returns in place of the symbolic `cost` (nats.py:772): the training graph bound to a
    device store.  f_log_probs / f_cost / gradients are produced from it by train() and the optimiser factories."""

    MAX_PLANS = 64            # plans are views + CUDA graphs (the storage is shared): cheap

    def __init__(self, tparams, options):
        self.tparams = tparams
        self.engine = tparams.engine
        self.options = options
        V, W, D, A = tparams.dims
        self.dims = Dims(V, W, D, A)
        self.decay_c = 0.
        self.clip_c = -1.
        self.is_mean = False
        self._plans = OrderedDict()
        self.arena = _Arena(self)
        self.use_graphs = os.environ.get('NATS_CUDA_GRAPHS', '1') != '0'
        # shape buckets: padded source / target lengths are rounded up so that ragged batches reuse captured graphs
        # (zero-padded positions are masked out: cost and gradients do not change, nats.py:354,518,565,770)
        self.bucket_tx = int(os.environ.get('NATS_BUCKET_TX', '8'))
        self.bucket_ty = int(os.environ.get('NATS_BUCKET_TY', '5'))
        self.lazy_cost = False
        self.overlap_allreduce = os.environ.get('NATS_OVERLAP_ALLREDUCE', '1') != '0'
        torch = self.engine.torch
        self.grads = torch.zeros(tparams.total + _lib.GRAD_TAIL, dtype=torch.float32, device=self.engine.device)
        self.stats = torch.zeros(8, dtype=torch.float32, device=self.engine.device)
        self.rank, self.world = parallel.world()
        self.split = int(self.engine.lib.nats_grad_split(ctypes.byref(self.dims)))
        self._side = None
        self._pg_side = None
        self._pg_side_tried = False
        self._cost_ring = None
        self._cost_slot = 0

    # -- reference idiom: cost = cost.mean() (nats.py:1323)
    def mean(self):
        g = copy.copy(self)
        g.is_mean = True
        return g

    def reserve(self, Tx, Ty, B):
        """size the shared storage for the largest batch that will be seen (train() knows maxlen and batch_size), so
        that no later plan has to grow it (growing drops every captured graph)"""
        self.arena.reserve(_bucket(Tx, self.bucket_tx), _bucket(Ty, self.bucket_ty), B)

    def plan(self, Tx, Ty, B):
        key = (_bucket(Tx, self.bucket_tx), _bucket(Ty, self.bucket_ty), B)
        p = self._plans.get(key)
        if p is not None and p.arena_version != self.arena.version:
            self._plans.clear()               # the arena moved: every captured graph holds stale addresses
            p = None
        if p is None:
            while len(self._plans) >= self.MAX_PLANS:
                self._plans.popitem(last=False)
            v0 = self.arena.version
            p = _TrainPlan(self, *key)
            if self.arena.version != v0:
                self._plans.clear()
            self._plans[key] = p
        else:
            self._plans.move_to_end(key)
        return p

    # -- raw enqueue helpers (no host sync)
    def _train_args(self, p):
        Tx, Ty, B = p.shape
        return (self.engine.ctx, self.engine.stream(), ctypes.byref(self.dims), _ptr(self.tparams.flat), _ptr(p.x), _ptr(p.xm),
                _ptr(p.y), _ptr(p.ym), Tx, Ty, B, _ptr(p.ws), p.ws_bytes)

    def enqueue_fwd(self, p):
        eng = self.engine
        _lib.check(eng.lib.nats_train_fwd(*(self._train_args(p) + (_ptr(p.cost),))), 'nats_train_fwd')
        eng.launches += 1

    def enqueue_bwd(self, p, scale, part=0):
        """part 0: whole backward; 1: readout + decoder (grads[split:] final); 2: encoder (grads[:split] final)"""
        eng = self.engine
        fn = (eng.lib.nats_train_bwd, eng.lib.nats_train_bwd_begin, eng.lib.nats_train_bwd_finish)[part]
        _lib.check(fn(*(self._train_args(p) + (ctypes.c_float(scale), _ptr(self.grads)))), 'nats_train_bwd')
        eng.launches += 1

    def enqueue_clip(self):
        eng = self.engine
        _lib.check(eng.lib.nats_grad_clip(eng.ctx, eng.stream(), self.tparams.total, _ptr(self.tparams.flat),
                                          _ptr(self.grads), ctypes.c_float(self.decay_c),
                                          ctypes.c_float(self.clip_c), _ptr(self.stats)), 'nats_grad_clip')
        eng.launches += 1

    def _run(self, p, attr, body):
        """run `body` eagerly the first time a shape is seen, then capture + replay it as a CUDA graph"""
        torch = self.engine.torch
        g = getattr(p, attr)
        if g is not None:
            g.replay()
            return
        if self.use_graphs and p.uses >= 1:
            torch.cuda.synchronize(self.engine.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                body()
            setattr(p, attr, g)
            g.replay()
            return
        body()

    # -- compiled callables
    def f_log_probs(self, x, x_mask, y, y_mask):
        """per-sample negative log-likelihood [B] (nats.py:1320)"""
        p = self.plan(x.shape[0], y.shape[0], x.shape[1])
        p.stage(x, x_mask, y, y_mask)
        self._run(p, 'graph_fwd', lambda: self.enqueue_fwd(p))
        p.uses += 1
        return p.cost.cpu().numpy()

    def f_cost(self, x, x_mask, y, y_mask):
        """mean cost (+ L2) (nats.py:1323-1336)"""
        c = float(self.f_log_probs(x, x_mask, y, y_mask).mean(dtype='float64'))
        if self.decay_c > 0.:
            c += self.decay_c * float((self.tparams.flat.double() ** 2).sum().item())
        return numpy.float32(c)

    def _read_cost(self):
        """device->host read of the step result: async copy into a pinned ring slot + event"""
        torch = self.engine.torch
        if self._cost_ring is None:
            self._cost_ring = [(torch.zeros(2, dtype=torch.float32).pin_memory(), torch.cuda.Event()) for _ in range(4)]
        buf, ev = self._cost_ring[self._cost_slot]
        self._cost_slot = (self._cost_slot + 1) % len(self._cost_ring)
        buf[:1].copy_(self.grads[self.tparams.total:self.tparams.total + 1], non_blocking=True)
        if self.decay_c > 0.:
            buf[1:2].copy_(self.stats[1:2], non_blocking=True)
        ev.record()
        hb = buf.numpy()

        class _B(object):           # buf[0] (+ decay_c * ||p||^2 once the event has completed)
            def __getitem__(s, i):
                return hb[0] + (self.decay_c * hb[1] if self.decay_c > 0. else 0.0)
        return LazyCost(_B(), ev)

    def grad_step(self, x, x_mask, y, y_mask, after_grads, global_batch=None):
        """forward + backward (+ allreduce) + L2/clip + `after_grads()` (the optimiser's accumulator update);
        returns the scalar cost like f_grad_shared (nats.py:1160).  `global_batch`: number of sentence pairs of the
        whole data-parallel step (default: local batch x world size).  x = None: this rank's shard is empty; it only
        contributes zeros to the all-reduce."""
        torch = self.engine.torch
        world = self.world
        if x is None:
            assert world > 1, 'empty batch'
            self.grads.zero_()
            parallel.allreduce_flat(self.grads)
            self.enqueue_clip()
            after_grads()
            c = self._read_cost()
            return c if self.lazy_cost else c.value()
        p = self.plan(x.shape[0], y.shape[0], x.shape[1])
        p.stage(x, x_mask, y, y_mask)
        B = x.shape[1]
        scale = parallel.grad_scale(B, world, global_batch)   # d mean(cost) over the GLOBAL batch (nats.py:1323)

        def post():
            self.enqueue_clip()
            after_grads()

        if world == 1:
            self._run(p, 'graph_step', lambda: (self.enqueue_fwd(p), self.enqueue_bwd(p, scale), post()))
        elif not self.overlap_allreduce:
            self._run(p, 'graph_fb', lambda: (self.enqueue_fwd(p), self.enqueue_bwd(p, scale)))
            parallel.allreduce_flat(self.grads)               # ONE collective: gradients + cost tail
            self._run(p, 'graph_post', post)
        else:
            # the decoder / readout / ff_state gradients (grads[split:], ~65 % of the buffer, + the cost slot) are final
            # before the encoder backward starts: their all-reduce runs on a side stream UNDER the encoder backward,
            # only the encoder slice is reduced after it
            if self._side is None:
                self._side = torch.cuda.Stream(device=self.engine.device)
            if not self._pg_side_tried:                       # collective call: every rank reaches this in its first step
                self._pg_side_tried = True
                self._pg_side = parallel.side_group(int(os.environ.get('NATS_NCCL_SIDE_CTAS', '4')))
            main = torch.cuda.current_stream(self.engine.device)
            self._run(p, 'graph_fb', lambda: (self.enqueue_fwd(p), self.enqueue_bwd(p, scale, 1)))
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                w1 = parallel.allreduce_flat(self.grads[self.split:], async_op=True, group=self._pg_side)
            self._run(p, 'graph_fb2', lambda: self.enqueue_bwd(p, scale, 2))
            parallel.allreduce_flat(self.grads[:self.split])
            if w1 is not None:
                w1.wait()
            main.wait_stream(self._side)
            self._run(p, 'graph_post', post)
        p.uses += 1
        c = self._read_cost()
        return c if self.lazy_cost else c.value()


def build_model(tparams, options):
    """Reference signature (nats.py:658-772).  Returns the same 8-tuple; the symbolic inputs are replaced by
    their names and `cost` by a ModelGraph bound to `tparams`."""
    opt_ret = dict()
    trng = numpy.random.RandomState(1234)
    use_noise = _HostFlag(0.)
    graph = ModelGraph(tparams, options)
    return trng, use_noise, 'x', 'x_mask', 'y', 'y_mask', opt_ret, graph


class _HostFlag(object):
    def __init__(self, v):
        self.v = v

    def set_value(self, v):
        self.v = v

    def get_value(self):
        return self.v


# ----------------------------------------------------------------------------------------------------------
# optimisers: name(lr, tparams, grads, inp, cost) -> (f_grad_shared, f_update)   (nats.py:1104-1221)
# `grads` is the ModelGraph (it owns the flat gradient buffer; clipping / L2 were configured on it by train()).
# ----------------------------------------------------------------------------------------------------------
def _zeros_like_flat(graph):
    torch = graph.engine.torch
    return torch.zeros(graph.tparams.total, dtype=torch.float32, device=graph.engine.device)


def adadelta(lr, tparams, grads, inp, cost, epsilon=1e-6, rho=0.95):
    graph = grads
    eng = graph.engine
    running_up2, running_grads2 = _zeros_like_flat(graph), _zeros_like_flat(graph)
    n = tparams.total

    def accum():
        _lib.check(eng.lib.nats_adadelta_grad_shared(eng.ctx, eng.stream(), n, _ptr(graph.grads),
                                                     _ptr(running_grads2), ctypes.c_float(rho)),
                   'nats_adadelta_grad_shared')
        eng.launches += 1

    def f_grad_shared(x, x_mask, y, y_mask, global_batch=None):
        return graph.grad_step(x, x_mask, y, y_mask, accum, global_batch=global_batch)

    def f_update(lr_value=None):
        _lib.check(eng.lib.nats_adadelta_update(eng.ctx, eng.stream(), n, _ptr(tparams.flat), _ptr(graph.grads),
                                                _ptr(running_up2), _ptr(running_grads2), ctypes.c_float(rho),
                                                ctypes.c_float(epsilon)), 'nats_adadelta_update')
        eng.launches += 1
        return []

    f_grad_shared.state = dict(running_up2=running_up2, running_grads2=running_grads2)
    f_grad_shared.accum = accum
    return f_grad_shared, f_update


def adam(lr, tparams, grads, inp, cost):
    graph = grads
    eng = graph.engine
    m, v = _zeros_like_flat(graph), _zeros_like_flat(graph)
    n = tparams.total
    step = numpy.zeros(1, dtype='int64')

    def f_grad_shared(x, x_mask, y, y_mask, global_batch=None):
        return graph.grad_step(x, x_mask, y, y_mask, lambda: None, global_batch=global_batch)

    def f_update(lr_value=None):
        _lib.check(eng.lib.nats_adam_update(eng.ctx, eng.stream(), n, _ptr(tparams.flat), _ptr(graph.grads),
                                            _ptr(m), _ptr(v), int(step[0])), 'nats_adam_update')
        eng.launches += 1
        step[0] += 1
        return []

    f_grad_shared.state = dict(m=m, v=v, step=step)
    return f_grad_shared, f_update


def rmsprop(lr, tparams, grads, inp, cost):
    graph = grads
    eng = graph.engine
    rg, rg2, ud = _zeros_like_flat(graph), _zeros_like_flat(graph), _zeros_like_flat(graph)
    n = tparams.total

    def accum():
        _lib.check(eng.lib.nats_rmsprop_grad_shared(eng.ctx, eng.stream(), n, _ptr(graph.grads), _ptr(rg),
                                                    _ptr(rg2)), 'nats_rmsprop_grad_shared')
        eng.launches += 1

    def f_grad_shared(x, x_mask, y, y_mask, global_batch=None):
        return graph.grad_step(x, x_mask, y, y_mask, accum, global_batch=global_batch)

    def f_update(lr_value=None):
        _lib.check(eng.lib.nats_rmsprop_update(eng.ctx, eng.stream(), n, _ptr(tparams.flat), _ptr(graph.grads),
                                               _ptr(ud), _ptr(rg), _ptr(rg2)), 'nats_rmsprop_update')
        eng.launches += 1
        return []

    f_grad_shared.state = dict(running_grads=rg, running_grads2=rg2, updir=ud)
    return f_grad_shared, f_update


def sgd(lr, tparams, grads, inp, cost):
    """The reference's sgd has a 7-argument signature that train() never matches (dead code, nats.py:1209);
    provided here with the common 5-argument form: p <- p - lr * g."""
    graph = grads

    def f_grad_shared(x, x_mask, y, y_mask, global_batch=None):
        return graph.grad_step(x, x_mask, y, y_mask, lambda: None, global_batch=global_batch)

    def f_update(lr_value):
        tparams.flat.add_(graph.grads[:tparams.total], alpha=-float(lr_value))
        return []

    return f_grad_shared, f_update


_OPTIMIZERS = {'adadelta': adadelta, 'adam': adam, 'rmsprop': rmsprop, 'sgd': sgd}


# ----------------------------------------------------------------------------------------------------------
# sampler (nats.py:776-874)
# ----------------------------------------------------------------------------------------------------------
class DeviceBackedArray(numpy.ndarray):
    """Host copy of an encoder context that remembers its device-resident original (and the projected context
    pctx).  numpy.tile / broadcast_to keep the subclass, so f_next can recognise `tile(ctx0, [live_k, 1])`
    (nats.py:958) and read the ONE device copy with a zero batch stride instead of re-uploading k copies."""

    def __new__(cls, arr, handle=None):
        obj = numpy.asarray(arr).view(cls)
        obj._nats_handle = handle
        return obj

    def __array_finalize__(self, obj):
        self._nats_handle = getattr(obj, '_nats_handle', None)

    # the handle stands for "these values are the encoder context on the device": anything computed FROM the array
    # (ufuncs) is a plain ndarray, and writing into the array drops the handle
    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        plain = [numpy.asarray(i) if isinstance(i, DeviceBackedArray) else i for i in inputs]
        if 'out' in kwargs:
            for o in kwargs['out']:
                if isinstance(o, DeviceBackedArray):
                    o._nats_handle = None
            kwargs['out'] = tuple(numpy.asarray(o) if isinstance(o, DeviceBackedArray) else o for o in kwargs['out'])
        return getattr(ufunc, method)(*plain, **kwargs)

    def __setitem__(self, key, value):
        self._nats_handle = None
        b = self.base
        while isinstance(b, numpy.ndarray):                 # writing through a view invalidates the owner as well
            if isinstance(b, DeviceBackedArray):
                b._nats_handle = None
            b = b.base
        numpy.ndarray.__setitem__(self, key, value)


class _CtxHandle(object):
    def __init__(self, ctx_dev, pctx_dev, host):
        self.ctx_dev, self.pctx_dev, self.host = ctx_dev, pctx_dev, host
        Tx = host.shape[0]
        self.probe_t = numpy.unique(numpy.linspace(0, Tx - 1, num=min(Tx, 8)).astype('int64'))

    def matches(self, ctx):
        """is `ctx` [Tx,n,C] the broadcast of the single-sentence context this handle owns?"""
        h = self.host
        if h.shape[1] != 1 or ctx.ndim != 3 or ctx.shape[0] != h.shape[0] or ctx.shape[2] != h.shape[2]:
            return False
        a = numpy.asarray(ctx)[self.probe_t]
        return bool(numpy.array_equal(a, numpy.broadcast_to(h[self.probe_t], a.shape)))


class DeviceArray(object):
    """What f_next returns in place of a host ndarray: a device tensor that is copied to the host the first time
    NumPy needs its values (`numpy.log(a)`, `a[0]`, `a[:, 1] = v` ...).  Row selection with an index list
    (`a[parents]`) and `.copy()` stay on the device, so gen_sample can hand states and accumulators straight back
    to f_next without a host round trip (SURVEY 8(f).1)."""
    __array_priority__ = 1000

    def __init__(self, tensor):
        self._t = tensor
        self._h = None
        self._dirty = False

    shape = property(lambda self: tuple(self._t.shape))
    ndim = property(lambda self: self._t.dim())
    dtype = property(lambda self: numpy.dtype(str(self._t.dtype).replace('torch.', '')))
    size = property(lambda self: int(self._t.numel()))

    def __len__(self):
        return int(self._t.shape[0])

    def host(self):
        if self._h is None:
            self._h = self._t.cpu().numpy()
        return self._h

    def tensor(self):
        """the device tensor (re-uploaded if the host copy was written to)"""
        if self._dirty:
            self._t.copy_(self._t.new_tensor(self._h))
            self._dirty = False
        return self._t

    def __array__(self, dtype=None, copy=None):
        h = self.host()
        return h if dtype is None else h.astype(dtype, copy=False)

    def __getitem__(self, idx):
        rows = isinstance(idx, (list, numpy.ndarray)) and numpy.asarray(idx).ndim == 1 and \
            numpy.asarray(idx).dtype.kind in 'iu'
        if rows and not self._dirty:
            import torch
            ii = torch.as_tensor(numpy.asarray(idx, dtype='int64'), device=self._t.device)
            return DeviceArray(self._t.index_select(0, ii))
        return self.host()[idx]

    def __setitem__(self, idx, value):
        self.host()[idx] = value
        self._dirty = True

    def copy(self):
        if self._h is not None:
            return self._h.copy()
        return DeviceArray(self._t.clone())

    def argmax(self, *a, **k):
        return self.host().argmax(*a, **k)

    def flatten(self):
        return self.host().flatten()

    def __repr__(self):
        return 'DeviceArray(%r)' % (self.host(),)


def _binop(name):
    def f(self, other):
        return getattr(self.host(), name)(other.host() if isinstance(other, DeviceArray) else other)
    return f


for _n in ('__add__', '__radd__', '__sub__', '__rsub__', '__mul__', '__rmul__', '__truediv__', '__rtruediv__',
           '__lt__', '__le__', '__gt__', '__ge__', '__eq__', '__ne__'):
    setattr(DeviceArray, _n, _binop(_n))
DeviceArray.__hash__ = None


def build_sampler(tparams, options, trng=None):
    """-> f_init, f_next with the reference signatures (nats.py:817, 869-871)."""
    eng = tparams.engine
    torch = eng.torch
    V, W, D, A = tparams.dims
    C = 2 * D
    dims = Dims(V, W, D, A)
    seed = 1234
    counter = [0]

    def ws_for(Tx, n, slot=0):
        """sampler workspace; one per `slot`: calls that may be in flight at the same time (searches on different streams,
        the batched encoder) must not share it"""
        nbytes = eng.lib.nats_sampler_workspace_bytes(ctypes.byref(dims), Tx, n)
        if nbytes <= 0:
            raise NatsB200Error('nats_sampler_workspace_bytes failed')
        return eng.workspace(('sampler', slot), nbytes), int(nbytes)

    def f_init(x):
        x = numpy.ascontiguousarray(x, dtype='int64')
        Tx, n = x.shape
        xd = torch.from_numpy(x).to(eng.device)
        ws, nbytes = ws_for(Tx, n)
        init_state = torch.empty((n, D), dtype=torch.float32, device=eng.device)
        ctx = torch.empty((Tx, n, C), dtype=torch.float32, device=eng.device)
        pctx = torch.empty((Tx, n, A), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.nats_sampler_init(eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(xd), None,
                                             Tx, n, _ptr(ws), nbytes, _ptr(init_state), _ptr(ctx), _ptr(pctx)),
                   'nats_sampler_init')
        eng.launches += 1
        host = ctx.cpu().numpy()
        return [init_state.cpu().numpy(), DeviceBackedArray(host, _CtxHandle(ctx, pctx, host))]

    # ---- device-side f_init for the device-resident beam search: no host copies, and SEVERAL sentences per encoder launch.
    # The persistent encoder kernel costs the same ~7 us per source position for 1 or 32 sentences, and at summary lengths
    # f_init is more than half of a sentence's time: gen.py hands the next sentences to prefetch(), which encodes them in one
    # masked launch (the training encoder's masks, nats.py:700-724) and parks the per-sentence slices.
    cache = {}

    def _key(x):
        return numpy.ascontiguousarray(x, dtype='int64').reshape(-1).tobytes()

    def encode(vs, slot='init'):
        """vs: source sentences (1-d word ids) -> init_state [n, D], ctx [Tx, n, C], pctx [Tx, n, A] of ONE masked encoder
        launch (Tx = the longest; rows t >= len(vs[i]) of column i are padding)"""
        n = len(vs)
        Tx = max(len(v) for v in vs)
        xb = numpy.zeros((Tx, n), dtype='int64')
        mb = numpy.zeros((Tx, n), dtype='float32')
        for i, v in enumerate(vs):
            xb[:len(v), i] = v
            mb[:len(v), i] = 1.
        xd, md = torch.from_numpy(xb).to(eng.device), torch.from_numpy(mb).to(eng.device)
        ws, nbytes = ws_for(Tx, n, slot)
        f32 = dict(dtype=torch.float32, device=eng.device)
        init_state, ctx, pctx = torch.empty((n, D), **f32), torch.empty((Tx, n, C), **f32), torch.empty((Tx, n, A), **f32)
        _lib.check(eng.lib.nats_sampler_init(eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(xd), _ptr(md),
                                             Tx, n, _ptr(ws), nbytes, _ptr(init_state), _ptr(ctx), _ptr(pctx)),
                   'nats_sampler_init')
        eng.launches += 1
        return init_state, ctx, pctx

    def prefetch(xs, max_batch=32):
        """xs: iterable of source sentences ([Tx_i] or [Tx_i, 1] word ids, EOS included); encodes those not parked yet"""
        todo = []
        for x in xs:
            k_ = _key(x)
            if k_ not in cache and all(k_ != t[0] for t in todo):
                todo.append((k_, numpy.ascontiguousarray(x, dtype='int64').reshape(-1)))
        for lo in range(0, len(todo), max_batch):
            grp = todo[lo:lo + max_batch]
            init_state, ctx, pctx = encode([v for _, v in grp])
            for i, (k_, v) in enumerate(grp):
                L = len(v)
                cache[k_] = (init_state[i].clone(), ctx[:L, i].contiguous(), pctx[:L, i].contiguous())
        while len(cache) > 4 * max_batch:                     # sentences that were never asked for
            cache.pop(next(iter(cache)))

    def init_device(x):
        """-> (init_state [D], ctx [Tx, C], pctx [Tx, A]) device tensors of ONE sentence; parked results are used once"""
        hit = cache.pop(_key(x), None)
        if hit is not None:
            return hit
        x = numpy.ascontiguousarray(x, dtype='int64').reshape(-1, 1)
        Tx = x.shape[0]
        xd = torch.from_numpy(x).to(eng.device)
        ws, nbytes = ws_for(Tx, 1, ('init', eng.stream()))        # per stream: a search on another stream may be initialising too
        f32 = dict(dtype=torch.float32, device=eng.device)
        init_state, ctx, pctx = torch.empty((1, D), **f32), torch.empty((Tx, 1, C), **f32), torch.empty((Tx, 1, A), **f32)
        _lib.check(eng.lib.nats_sampler_init(eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(xd), None,
                                             Tx, 1, _ptr(ws), nbytes, _ptr(init_state), _ptr(ctx), _ptr(pctx)),
                   'nats_sampler_init')
        eng.launches += 1
        return init_state.reshape(D), ctx.reshape(Tx, C), pctx.reshape(Tx, A)

    def init_group(xs):
        """-> (init_state [S, D], ctx [Tx, S, C], pctx [Tx, S, A], source lengths) of a group of S sentences, used in place by
        the grouped beam search; ONE sentence goes through init_device (a sentence parked by prefetch is used once)"""
        if len(xs) == 1:
            s0, c0, p0 = init_device(xs[0])
            Tx = int(c0.shape[0])
            return s0.reshape(1, D), c0.reshape(Tx, 1, C), p0.reshape(Tx, 1, A), [Tx]
        vs = [numpy.ascontiguousarray(x, dtype='int64').reshape(-1) for x in xs]
        init_state, ctx, pctx = encode(vs, ('init', eng.stream()))     # per stream, like init_device
        return init_state, ctx, pctx, [len(v) for v in vs]

    f_init.prefetch = prefetch
    f_init.device = init_device
    f_init.group = init_group

    def f_next(y, ctx, init_state, acc_ctx, acc_alpha):
        y = numpy.ascontiguousarray(y, dtype='int64')
        n = y.shape[0]
        Tx = ctx.shape[0]
        handle = getattr(ctx, '_nats_handle', None)
        if handle is not None and handle.matches(ctx):
            ctx_d, pctx_d = handle.ctx_dev, handle.pctx_dev
            cts, cbs, pts, pbs = C, 0, A, 0                   # one source shared by all n hypotheses
            pptr = _ptr(pctx_d)
        else:                                                 # arbitrary context: upload, recompute pctx (nats.py:493)
            ctx_d = torch.from_numpy(numpy.ascontiguousarray(ctx, dtype='float32')).to(eng.device)
            if ctx_d.shape[1] != n:
                raise ValueError('ctx has %d columns, y has %d' % (ctx_d.shape[1], n))
            cts, cbs, pts, pbs = n * C, C, 0, 0
            pptr = ctypes.c_void_p(0)
        def up(a, shp):
            if isinstance(a, DeviceArray):                    # came out of a previous f_next: already on the device
                return a.tensor().reshape(shp).contiguous()
            return torch.from_numpy(numpy.ascontiguousarray(a, dtype='float32').reshape(shp)).to(eng.device)
        yd = torch.from_numpy(y).to(eng.device)
        st_d, ac_d, aa_d = up(init_state, (n, D)), up(acc_ctx, (n, C)), up(acc_alpha, (n, Tx))
        ws, nbytes = ws_for(Tx, n)
        f32 = dict(dtype=torch.float32, device=eng.device)
        probs = torch.empty((n, V), **f32)
        sample = torch.empty((n,), dtype=torch.int64, device=eng.device)
        state_o, alphaT, ctxs = torch.empty((n, D), **f32), torch.empty((n, Tx), **f32), torch.empty((n, C), **f32)
        acc_ctx_o, acc_alpha_o = torch.empty((n, C), **f32), torch.empty((n, Tx), **f32)
        _lib.check(eng.lib.nats_sampler_next(
            eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(yd), _ptr(ctx_d), cts, cbs, pptr,
            pts, pbs, _ptr(st_d), _ptr(ac_d), _ptr(aa_d), Tx, n, seed, counter[0], _ptr(ws), nbytes, _ptr(probs),
            _ptr(sample), _ptr(state_o), _ptr(alphaT), _ptr(ctxs), _ptr(acc_ctx_o), _ptr(acc_alpha_o)),
            'nats_sampler_next')
        eng.launches += 1
        counter[0] += 1
        f_next.last_device = dict(alpha=alphaT, ctx=ctxs, state=state_o, probs=probs)
        # same seven outputs in the same order (nats.py:869-870); each becomes a host array on first NumPy access
        return [DeviceArray(probs), DeviceArray(sample), DeviceArray(state_o), DeviceArray(alphaT), DeviceArray(ctxs),
                DeviceArray(acc_ctx_o), DeviceArray(acc_alpha_o)]

    def topk(probs_dev, kk, mask_unk):
        """(p [n,kk] float32, idx [n,kk] int32) host arrays: the kk most probable words of every row"""
        n = int(probs_dev.shape[0])
        tp = torch.empty((n, kk), dtype=torch.float32, device=eng.device)
        ti = torch.empty((n, kk), dtype=torch.int32, device=eng.device)
        _lib.check(eng.lib.nats_beam_topk(eng.ctx, eng.stream(), _ptr(probs_dev), n, int(probs_dev.shape[1]), kk,
                                          1 if mask_unk else 0, _ptr(tp), _ptr(ti)), 'nats_beam_topk')
        eng.launches += 1
        return tp.cpu().numpy(), ti.cpu().numpy()

    def next_device(y_d, ctx_d, pctx_d, st_d, ac_d, aa_d, Tx, n, outs):
        """f_next entirely on device tensors (rows of ONE source: zero batch stride), outputs into preallocated `outs`;
        outs[1] = None skips the multinomial draw (beam search never reads it)"""
        ws, nbytes = ws_for(Tx, n)
        _lib.check(eng.lib.nats_sampler_next(
            eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(y_d), _ptr(ctx_d), C, 0, _ptr(pctx_d), A, 0,
            _ptr(st_d), _ptr(ac_d), _ptr(aa_d), Tx, n, seed, counter[0], _ptr(ws), nbytes, _ptr(outs[0]), _ptr(outs[1]),
            _ptr(outs[2]), _ptr(outs[3]), _ptr(outs[4]), _ptr(outs[5]), _ptr(outs[6])), 'nats_sampler_next')
        eng.launches += 1
        counter[0] += 1

    def bind_next(y_d, ctx_d, pctx_d, st_d, ac_d, aa_d, Tx, n, outs):
        """next_device with every pointer argument converted ONCE: a zero-argument callable for the beam-search loop (the
        tensors must stay alive and in place, which the caller's ping-pong buffers do)"""
        ws, nbytes = ws_for(Tx, n)
        args = (eng.ctx, eng.stream(), ctypes.byref(dims), _ptr(tparams.flat), _ptr(y_d), _ptr(ctx_d), C, 0, _ptr(pctx_d), A, 0,
                _ptr(st_d), _ptr(ac_d), _ptr(aa_d), Tx, n, seed, 0, _ptr(ws), nbytes) + tuple(_ptr(o) for o in outs)
        fn = eng.lib.nats_sampler_next

        def call():
            rc = fn(*args)
            if rc != 0:
                _lib.check(rc, 'nats_sampler_next')
        call.keep = (ws, y_d, ctx_d, pctx_d, st_d, ac_d, aa_d, outs)
        return call

    f_next.last_device = None
    f_next.engine = eng
    f_next.bind_next = bind_next
    f_next.beam_env = (ws_for, tparams, dims)      # what nats_beam_step needs besides the search buffers
    f_next.topk = topk
    f_next.next_device = next_device
    f_next.dims = (V, W, D, A)
    return f_init, f_next


# ----------------------------------------------------------------------------------------------------------
# beam search with distraction (nats.py:879-1076)
# ----------------------------------------------------------------------------------------------------------
class DistractionScorer(object):
    """Device-resident attention / context / state histories of the live hypotheses and the lambda_1..3 penalties
    of nats.py:981-995 computed by nats_beam_distraction_scores (replaces O(k*ii) SciPy calls per step)."""

    def __init__(self, engine, k, maxlen, Tx, C, D):
        torch = engine.torch
        self.eng, self.k, self.cap = engine, k, maxlen
        self.dims = (Tx, C, D)
        mk = lambda d: [torch.zeros((k, maxlen, d), dtype=torch.float32, device=engine.device) for _ in range(2)]
        self.hist = [mk(Tx), mk(C), mk(D)]       # [alpha, ctx, state] x ping-pong
        self.cur = 0
        self.len = 0
        self.scratch = torch.zeros(3 * k * maxlen + 16, dtype=torch.float32, device=engine.device)
        self.out = torch.zeros(3 * k, dtype=torch.float32, device=engine.device)

    def _dev(self, arr):
        torch = self.eng.torch
        if isinstance(arr, torch.Tensor):
            return arr
        return torch.from_numpy(numpy.ascontiguousarray(arr, dtype='float32')).to(self.eng.device)

    def penalties(self, cur_alpha, cur_ctx, cur_state, live_k, kl, cf, sf):
        eng = self.eng
        Tx, C, D = self.dims
        a, c, s = self._dev(cur_alpha), self._dev(cur_ctx), self._dev(cur_state)
        h = [self.hist[i][self.cur] for i in range(3)]
        _lib.check(eng.lib.nats_beam_distraction_scores(
            eng.ctx, eng.stream(), _ptr(h[0]), _ptr(h[1]), _ptr(h[2]), self.cap, self.len, live_k, Tx, C, D,
            _ptr(a), _ptr(c), _ptr(s), ctypes.c_float(kl), ctypes.c_float(cf), ctypes.c_float(sf),
            _ptr(self.scratch), _ptr(self.out)), 'nats_beam_distraction_scores')
        eng.launches += 1
        return self.out[:3 * live_k].cpu().numpy().reshape(3, live_k)

    def advance(self, cur_alpha, cur_ctx, cur_state, parents):
        """histories of the surviving hypotheses j <- history of parents[j] + the current step's vectors"""
        eng = self.eng
        torch = eng.torch
        if len(parents) == 0:
            return
        par = torch.tensor(list(map(int, parents)), dtype=torch.int32, device=eng.device)
        curs = [self._dev(cur_alpha), self._dev(cur_ctx), self._dev(cur_state)]
        for i in range(3):
            src, dst = self.hist[i][self.cur], self.hist[i][self.cur ^ 1]
            _lib.check(eng.lib.nats_beam_reorder_append(eng.ctx, eng.stream(), _ptr(src), _ptr(dst), _ptr(curs[i]),
                                                        _ptr(par), len(parents), self.cap, self.len, self.dims[i]),
                       'nats_beam_reorder_append')
            eng.launches += 1
        self.cur ^= 1
        self.len += 1


def _tile_ctx(ctx0, live_k):
    """numpy.tile(ctx0, [live_k, 1]) (nats.py:958) without materialising live_k copies"""
    if ctx0.shape[1] == 1:
        return numpy.broadcast_to(ctx0, (ctx0.shape[0], live_k, ctx0.shape[2]), subok=True)
    return numpy.tile(ctx0, [live_k, 1])


class _DeviceBeam(object):
    """Beam search with every piece of bookkeeping on the device (SURVEY 8(f).1, replaces the host loop of
    nats.py:1001-1066), for a GROUP of S source sentences at once: per step ONE f_next on S*k rows (row s*k + j is row j of
    sentence s and attends to its own source; rows >= live_k of a sentence are ignored), the distraction penalties, a
    per-row top-k, nats_beam_select (one warp per sentence: candidate merge, re-ranking, EOS retirement) and
    nats_beam_advance (state / accumulator / history gathers within each sentence).  The weights are read once per step for
    all S*k rows.  The host reads one 4-byte flag per step, the number of sentences that are done, two steps late (the GPU
    queue never drains), and copies tokens, scores and attention histories back once at the end.  Each sentence gets the
    reference's three lists, as its own search would return them.

    One search = one object: __init__ encodes the group (one masked encoder launch; its [Tx, S, C] output is used in place)
    and allocates and binds everything on `stream`, step() issues one iteration (False once every sentence is over),
    result() fetches the hypotheses.  gen_sample runs a group of one on the current stream; gen_sample_many keeps several
    groups in flight on separate streams (workspace slot = stream).

    Device memory per group, by count, at S = 16, k = 10, maxlen = 100, Tx = 800, dim = 1000: the ping-pong histories
    2 x S*k x maxlen x (Tx + 3*dim) floats = 0.49 GB (0.10 GB without penalties), out_alpha S*k x maxlen x Tx floats =
    0.05 GB, and the f_next workspace of S*k rows, whose encoder part (Tx x S*k x 6*dim floats, unused by the search) makes
    it 3.2 GB."""

    def __init__(self, f_init, f_next, xs, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace=None, slot=0,
                 stream=None):
        torch = f_next.engine.torch
        self.tstream = stream if stream is not None else torch.cuda.current_stream(f_next.engine.device)
        with torch.cuda.stream(self.tstream):
            self._setup(f_init, f_next, xs, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace, slot)

    def _setup(self, f_init, f_next, xs, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace, slot):
        eng = f_next.engine
        torch = eng.torch
        lib = eng.lib
        V, W, D, A = f_next.dims
        C = 2 * D
        S = len(xs)
        if _trace is not None and S != 1:
            raise ValueError('the step trace covers a group of one sentence')
        init_state, ctx_d, pctx_d, src_lens = f_init.group(xs)        # device tensors [S, D], [Tx, S, C], [Tx, S, A]
        Tx = int(ctx_d.shape[0])
        n = S * k
        dev = eng.device
        f32 = dict(dtype=torch.float32, device=dev)
        i32 = dict(dtype=torch.int32, device=dev)
        distract = kl_factor > 0. or ctx_factor > 0. or state_factor > 0.
        # state of the live rows (ping-pong), f_next outputs, histories, results
        state = [torch.zeros((n, D), **f32) for _ in range(2)]
        acc_ctx = [torch.zeros((n, C), **f32) for _ in range(2)]
        acc_alpha = [torch.zeros((n, Tx), **f32) for _ in range(2)]
        state[0].view(S, k, D)[:, 0].copy_(init_state.reshape(S, D))
        outs = [torch.empty((n, V), **f32), None, torch.empty((n, D), **f32),
                torch.empty((n, Tx), **f32), torch.empty((n, C), **f32), torch.empty((n, C), **f32), torch.empty((n, Tx), **f32)]
        hist_alpha = [torch.zeros((n, maxlen, Tx), **f32) for _ in range(2)]
        hist_ctx = [torch.zeros((n, maxlen, C), **f32) for _ in range(2)] if distract else [None, None]
        hist_state = [torch.zeros((n, maxlen, D), **f32) for _ in range(2)] if distract else [None, None]
        out_alpha = torch.zeros((S, k, maxlen, Tx), **f32)
        c0 = getattr(eng, '_beam_counters0', None)               # live_k, dead_k, done, finished, last effective step
        if c0 is None:                                           # (a host list -> device tensor is a synchronous copy: once)
            c0 = eng._beam_counters0 = torch.tensor([1, 0, 0, 0, -1, 0, 0, 0], **i32)
        counters = c0.repeat(S)
        src_len_h = torch.tensor(src_lens, dtype=torch.int32).pin_memory()
        src_len = src_len_h.to(dev, non_blocking=True)
        scores = torch.zeros((2, n), **f32)
        tokens = torch.zeros((2, n, maxlen), **i32)
        parents = torch.zeros((n,), **i32)
        fin_parent = torch.zeros((n,), **i32)
        next_w = torch.full((n,), -1, dtype=torch.int64, device=dev)          # BOS marker -> zero embedding
        out_tokens = torch.zeros((S, k, maxlen), **i32)
        out_len = torch.zeros((S, k), **i32)
        out_score = torch.zeros((S, k), **f32)
        top_p, top_i = torch.empty((n, k), **f32), torch.empty((n, k), **i32)
        pen = torch.zeros((3 * n,), **f32)
        scratch = torch.zeros((3 * n * maxlen + 16,), **f32)
        # the number of sentences that are done reaches the host without a copy: nats_beam_select mirrors it into pinned host
        # memory, the loop looks at it two steps late (after that step's event), so the GPU queue never drains.  All pointer
        # arguments are converted once, per ping-pong parity: the loop body is one C call on a prebuilt struct.
        host_cnt = torch.zeros(8, dtype=torch.int32).pin_memory()
        host_np = host_cnt.numpy()
        events = [torch.cuda.Event() for _ in range(2)]
        P, cf = _ptr, ctypes.c_float
        stream = ctypes.c_void_p(self.tstream.cuda_stream)
        if _trace is not None:                                   # five separate calls per step (single sentence, [Tx, C])
            ctx1, pctx1 = ctx_d.reshape(Tx, C), pctx_d.reshape(Tx, A)
            step_next = [f_next.bind_next(next_w, ctx1, pctx1, state[c], acc_ctx[c], acc_alpha[c], Tx, k, outs) for c in (0, 1)]
            pen_head = [(eng.ctx, stream, P(hist_alpha[c]), P(hist_ctx[c]), P(hist_state[c]), maxlen) for c in (0, 1)]
            pen_tail = (k, Tx, C, D, P(outs[3]), P(outs[4]), P(outs[2]), cf(kl_factor), cf(ctx_factor), cf(state_factor), P(scratch),
                        P(pen))
            topk_args = (eng.ctx, stream, P(outs[0]), k, V, k, 0 if use_unk else 1, P(top_p), P(top_i))
            sel_head = (eng.ctx, stream, P(top_p), P(top_i))
            sel_tail = (P(counters), P(scores), P(tokens), P(parents), P(next_w), P(out_tokens), P(out_len), P(out_score),
                        P(fin_parent), P(host_cnt))
            pen_ptr, no_ptr = P(pen), P(None)
            adv_head = (eng.ctx, stream, P(parents), P(fin_parent), P(counters), k, maxlen)
            adv_tail = [(Tx, C, D, P(outs[2]), P(state[c ^ 1]), P(outs[5]), P(acc_ctx[c ^ 1]), P(outs[6]), P(acc_alpha[c ^ 1]),
                         P(outs[3]), P(outs[4]), P(outs[2]), P(hist_alpha[c]), P(hist_alpha[c ^ 1]), P(hist_ctx[c]),
                         P(hist_ctx[c ^ 1]), P(hist_state[c]), P(hist_state[c ^ 1]), P(out_alpha)) for c in (0, 1)]
        check = _lib.check
        # without a trace the whole step is ONE foreign call (nats_beam_step_many) on a prebuilt argument struct per parity
        ws_for, tp_, dims_ = f_next.beam_env
        ws_t, ws_bytes = ws_for(Tx, n, slot)
        one_call = []
        for c in (0, 1):
            m = _lib.BeamStepMany()
            m.n_src, m.src_len = S, src_len.data_ptr()
            a = m.beam
            a.params, a.next_w, a.ctx, a.pctx = tp_.flat.data_ptr(), next_w.data_ptr(), ctx_d.data_ptr(), pctx_d.data_ptr()
            a.Tx, a.k, a.maxlen, a.use_unk = Tx, k, maxlen, 1 if use_unk else 0
            a.ws, a.ws_bytes = ws_t.data_ptr(), ws_bytes
            a.state_in, a.acc_ctx_in, a.acc_alpha_in = state[c].data_ptr(), acc_ctx[c].data_ptr(), acc_alpha[c].data_ptr()
            a.probs, a.state_out, a.alphaT, a.ctxs = outs[0].data_ptr(), outs[2].data_ptr(), outs[3].data_ptr(), outs[4].data_ptr()
            a.acc_ctx_out, a.acc_alpha_out = outs[5].data_ptr(), outs[6].data_ptr()
            a.kl_factor, a.ctx_factor, a.state_factor = kl_factor, ctx_factor, state_factor
            a.hist_alpha_in = hist_alpha[c].data_ptr()
            a.hist_ctx_in = hist_ctx[c].data_ptr() if distract else None
            a.hist_state_in = hist_state[c].data_ptr() if distract else None
            a.scratch, a.pen, a.top_p, a.top_i = scratch.data_ptr(), pen.data_ptr(), top_p.data_ptr(), top_i.data_ptr()
            a.counters, a.scores, a.tokens, a.parents = counters.data_ptr(), scores.data_ptr(), tokens.data_ptr(), parents.data_ptr()
            a.fin_parent, a.out_tokens, a.out_len = fin_parent.data_ptr(), out_tokens.data_ptr(), out_len.data_ptr()
            a.out_score, a.out_alpha, a.host_counters = out_score.data_ptr(), out_alpha.data_ptr(), host_cnt.data_ptr()
            a.state_next, a.acc_ctx_next, a.acc_alpha_next = state[c ^ 1].data_ptr(), acc_ctx[c ^ 1].data_ptr(), acc_alpha[c ^ 1].data_ptr()
            a.hist_alpha_out = hist_alpha[c ^ 1].data_ptr()
            a.hist_ctx_out = hist_ctx[c ^ 1].data_ptr() if distract else None
            a.hist_state_out = hist_state[c ^ 1].data_ptr() if distract else None
            one_call.append((eng.ctx, stream, ctypes.byref(dims_), ctypes.byref(m)))
        # every local becomes an attribute: step() / result() use a dozen of them, and ALL the tensors above must outlive the
        # search because their addresses sit in the prebuilt argument structs (a tensor dropped here would be a dangling pointer)
        keep = dict(locals())
        keep.pop('self')
        self.__dict__.update(keep)
        self.ii = 0

    def step(self):
        """issue iteration self.ii; False when the search has ended (every sentence retired all its hypotheses or
        maxlen was reached)"""
        ii, maxlen, torch = self.ii, self.maxlen, self.torch
        if ii >= maxlen:
            return False
        cur = ii & 1
        events = self.events
        if ii >= 2:
            events[cur].synchronize()                         # step ii-2 is through: its counters are in host memory
            if self.host_np[5] >= self.S:
                self.ii = maxlen
                return False
        self.ii = ii + 1
        eng = self.eng
        if self._trace is None:
            rc = self.lib.nats_beam_step_many(*self.one_call[cur], ii)
            if rc != 0:
                self.check(rc, 'nats_beam_step_many')
            eng.launches += 1
            events[cur].record(self.tstream)
            return True
        lib, check, k = self.lib, self.check, self.k
        with torch.cuda.stream(self.tstream):
            self.step_next[cur]()
            use_pen = self.distract and ii > 0
            if use_pen:
                check(lib.nats_beam_distraction_scores(*self.pen_head[cur], ii, *self.pen_tail), 'nats_beam_distraction_scores')
                live_now = int(self.counters[0].item())
                self._trace.append(dict(ii=ii, pen=self.pen.cpu().numpy().reshape(3, k)[:, :live_now].copy()))
            check(lib.nats_beam_topk(*self.topk_args), 'nats_beam_topk')
            check(lib.nats_beam_select(*self.sel_head, self.pen_ptr if use_pen else self.no_ptr, k, maxlen, ii, *self.sel_tail),
                  'nats_beam_select')
            check(lib.nats_beam_advance(*self.adv_head, ii, *self.adv_tail[cur]), 'nats_beam_advance')
            eng.launches += 5
            events[cur].record(self.tstream)
        return True

    def result(self):
        """per sentence of the group, the reference's three lists (nats.py:1068-1076): retired hypotheses first, then what
        is still alive; attention rows are cut to the sentence's own length"""
        torch = self.torch
        with torch.cuda.stream(self.tstream):
            out = self._result()
        return out

    def _result(self):
        S, k = self.S, self.k
        self.tstream.synchronize()
        cnt = self.counters.cpu().numpy().reshape(S, 8)
        # with the late flag up to two steps may have run after `done`: nats_beam_select leaves a done sentence untouched
        fin_tok, fin_len, fin_sc = self.out_tokens.cpu().numpy(), self.out_len.cpu().numpy(), self.out_score.cpu().numpy()
        fin_al = self.out_alpha.cpu().numpy()
        live = {}                                             # parity -> host copies of the live rows' buffers
        res = []
        for s in range(S):
            live_k, n_fin, Ls = int(cnt[s, 0]), int(cnt[s, 3]), self.src_lens[s]
            sample, sample_score, sample_dec_alphas = [], [], []
            for f in range(n_fin):
                L = int(fin_len[s, f])
                sample.append([int(t) for t in fin_tok[s, f, :L]])
                sample_score.append(numpy.float32(fin_sc[s, f]))
                sample_dec_alphas.append(list(fin_al[s, f, :L, :Ls].copy()))     # one copy; the rows are views of it
            if live_k > 0:                                    # dump what is still alive (nats.py:1068-1074)
                s_last = int(cnt[s, 4])                       # step s_last wrote the rows of parity (s_last + 1) & 1
                par, L = (s_last + 1) & 1, s_last + 1
                if par not in live:
                    live[par] = (self.tokens[par].cpu().numpy(), self.scores[par].cpu().numpy(),
                                 self.hist_alpha[par].cpu().numpy())
                lt, ls, ha = live[par]
                for j in range(s * k, s * k + live_k):
                    sample.append([int(t) for t in lt[j, :L]])
                    sample_score.append(numpy.float32(ls[j]))
                    sample_dec_alphas.append(list(ha[j, :L, :Ls].copy()))
            res.append((sample, sample_score, sample_dec_alphas))
        return res


def _gen_sample_device(f_init, f_next, x, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace):
    """one device-resident beam search (a group of one sentence) on the current stream (see _DeviceBeam)"""
    b = _DeviceBeam(f_init, f_next, [x], k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace)
    while b.step():
        pass
    return b.result()[0]


def gen_sample_many(tparams, f_init, f_next, xs, options, trng=None, k=5, maxlen=30, use_unk=False, kl_factor=0,
                    ctx_factor=0, state_factor=0, concurrency=12, chunk=16):
    """Beam search (nats.py:879-1076, stochastic=False) of a LIST of source sentences -> list of gen_sample's three lists.
    Every `chunk` consecutive sentences form one group: one masked encoder launch, then one device step advances the beams
    of all of them (S = chunk sentences x k rows per f_next; see _DeviceBeam), so the decoder and readout weights are read
    once per step for the whole group.  `concurrency` groups run interleaved, each on its own CUDA stream with its own
    workspace.  Results are those of gen_sample sentence by sentence, in order (the sentences of a group do not interact).
    Device memory per group in flight: see _DeviceBeam (3.7 GB at chunk = 16, beam 10, 100 steps, 800 source words,
    dim 1000)."""
    eng = f_next.engine
    torch = eng.torch
    if k > 32 or getattr(f_init, 'device', None) is None or os.environ.get('NATS_DEVICE_BEAM', '1') == '0':
        return [gen_sample(tparams, f_init, f_next, numpy.asarray(x).reshape(-1, 1), options, trng, k, maxlen, False, False,
                           use_unk, kl_factor, ctx_factor, state_factor) for x in xs]
    chunk = max(1, int(chunk))
    streams = getattr(eng, '_beam_streams', None)
    if streams is None:
        streams = eng._beam_streams = []
    while len(streams) < concurrency:
        streams.append(torch.cuda.Stream(device=eng.device))
    main = torch.cuda.current_stream(eng.device)
    results = [None] * len(xs)
    nxt, active = 0, {}

    def start(slot):
        nonlocal nxt
        grp = [numpy.asarray(x).reshape(-1) for x in xs[nxt:nxt + chunk]]
        streams[slot].wait_stream(main)                           # whatever the current stream queued comes first
        b = _DeviceBeam(f_init, f_next, grp, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, None, slot + 1,
                        streams[slot])
        active[slot] = (nxt, b)
        nxt += len(grp)
        b.step()

    for slot in range(min(concurrency, (len(xs) + chunk - 1) // chunk)):
        start(slot)
    while active:
        finished = []
        for slot in list(active):
            idx, b = active[slot]
            if not b.step():
                finished.append((idx, b))
                del active[slot]
                if nxt < len(xs):
                    start(slot)              # queued behind the finished group on the same stream (same workspace slot)
        for idx, b in finished:              # fetching a result waits for that group only; the others have work queued
            res = b.result()
            results[idx:idx + len(res)] = res
    return results


def gen_sample(tparams, f_init, f_next, x, options, trng=None, k=1, maxlen=30, stochastic=True, argmax=False,
               use_unk=False, kl_factor=0, ctx_factor=0, state_factor=0, _scorer_factory=None, _trace=None):
    """Stochastic sampling or beam search with distraction re-ranking; same arguments, return values and
    hypothesis bookkeeping as the reference (nats.py:879-1076).  Candidate costs stay un-penalised (nats.py:1004);
    the three penalties only re-rank (nats.py:997-999)."""
    if k > 1:
        assert not stochastic, 'Beam search does not support stochastic sampling'
    if (not stochastic and _scorer_factory is None and getattr(f_next, 'next_device', None) is not None and k <= 32
            and os.environ.get('NATS_DEVICE_BEAM', '1') != '0' and numpy.ndim(x) == 2 and numpy.shape(x)[1] == 1
            and getattr(f_init, '__module__', None) == __name__ and hasattr(f_init, 'device')):
        return _gen_sample_device(f_init, f_next, x, k, maxlen, use_unk, kl_factor, ctx_factor, state_factor, _trace)

    sample, sample_score, sample_dec_alphas = [], [], []
    if stochastic:
        sample_score = 0

    live_k, dead_k = 1, 0
    hyp_samples = [[]]
    hyp_scores = numpy.zeros(live_k, dtype='float32')
    hyp_dec_alphas = [[]]

    next_state, ctx0 = f_init(x)
    next_w = -1 * numpy.ones((1,), dtype='int64')        # BOS marker -> zero embedding
    acc_ctx = numpy.zeros((live_k, ctx0.shape[2]), dtype='float32')
    acc_alpha = numpy.zeros((live_k, ctx0.shape[0]), dtype='float32')

    distract = (not stochastic) and (kl_factor > 0. or ctx_factor > 0. or state_factor > 0.)
    scorer = None
    if distract:
        if _scorer_factory is not None:
            scorer = _scorer_factory(k, maxlen, ctx0.shape[0], ctx0.shape[2], next_state.shape[1])
        else:
            eng = getattr(f_next, 'engine', None) or get_engine()
            scorer = DistractionScorer(eng, k, maxlen, ctx0.shape[0], ctx0.shape[2], next_state.shape[1])

    for ii in range(maxlen):
        ctx = _tile_ctx(ctx0, live_k)
        next_p, next_w, next_state, dec_alphas, ctxs, acc_ctx, acc_alpha = f_next(next_w, ctx, next_state, acc_ctx,
                                                                                  acc_alpha)
        if stochastic:
            nw = next_p[0].argmax() if argmax else next_w[0]
            sample.append(nw)
            sample_score += next_p[0, nw]
            if nw == 0:
                break
            continue

        dev = getattr(f_next, 'last_device', None) or {}
        cur = (dev.get('alpha', dec_alphas), dev.get('ctx', ctxs), dev.get('state', next_state))
        n_keep = k - dead_k
        topk = getattr(f_next, 'topk', None)
        if topk is not None and dev.get('probs') is not None and isinstance(next_p, DeviceArray) and \
                next_p._h is None and n_keep <= next_p.shape[1]:
            # Hypothesis scores and penalties are constant per row, so the best n_keep candidates overall are among
            # each row's n_keep most probable words: select those on the device (nats_beam_topk) instead of sorting
            # all live_k*|V| scores on the host; same ranking rule, same un-penalised stored cost (nats.py:997-1004).
            top_p, top_i = topk(dev['probs'], n_keep, not use_unk)
            with numpy.errstate(divide='ignore'):
                cand_scores = hyp_scores[:, None] - numpy.log(top_p)
            cand_flat = cand_scores.flatten()
            if distract and ii > 0:
                pen = scorer.penalties(cur[0], cur[1], cur[2], live_k, kl_factor, ctx_factor, state_factor)
                if _trace is not None:
                    _trace.append(dict(ii=ii, pen=numpy.array(pen)))
                ranked = (cand_scores + pen[0][:, None] + pen[1][:, None] + pen[2][:, None]).flatten()
            else:
                ranked = cand_flat
            ranked = numpy.where(top_i.flatten() < 0, numpy.float32(numpy.inf), ranked)
            ranks_flat = ranked.argsort(kind='stable')[:n_keep]
            trans_indices = ranks_flat // n_keep
            word_indices = top_i.flatten()[ranks_flat].astype('int64')
            costs = cand_flat[ranks_flat]
        else:
            if not use_unk:
                next_p[:, 1] = 1e-20
            cand_scores = hyp_scores[:, None] - numpy.log(next_p)
            cand_flat = cand_scores.flatten()
            if distract and ii > 0:
                pen = scorer.penalties(cur[0], cur[1], cur[2], live_k, kl_factor, ctx_factor, state_factor)
                if _trace is not None:
                    _trace.append(dict(ii=ii, pen=numpy.array(pen)))
                ranked = (cand_scores + pen[0][:, None] + pen[1][:, None] + pen[2][:, None]).flatten()
                ranks_flat = ranked.argsort()[:n_keep]
            else:
                ranks_flat = cand_flat.argsort()[:n_keep]

            voc_size = next_p.shape[1]
            trans_indices = ranks_flat // voc_size
            word_indices = ranks_flat % voc_size
            costs = cand_flat[ranks_flat]

        survivors = []                    # (parent index, word, cost) of the hypotheses that stay alive
        for ti, wi, ci in zip(trans_indices, word_indices, costs):
            grown = hyp_samples[ti] + [wi]
            alphas = hyp_dec_alphas[ti] + [dec_alphas[ti].copy()]
            if wi == 0:                   # finished: move to the result lists (nats.py:1037-1041)
                sample.append(grown)
                sample_score.append(numpy.float32(ci))
                sample_dec_alphas.append(alphas)
                dead_k += 1
            else:
                survivors.append((int(ti), grown, numpy.float32(ci), alphas))

        live_k = len(survivors)
        if live_k < 1 or dead_k >= k:
            hyp_samples = [s[1] for s in survivors]
            hyp_scores = numpy.array([s[2] for s in survivors], dtype='float32')
            hyp_dec_alphas = [s[3] for s in survivors]
            break
        parents = [s[0] for s in survivors]
        if distract:
            scorer.advance(cur[0], cur[1], cur[2], parents)
        hyp_samples = [s[1] for s in survivors]
        hyp_scores = numpy.array([s[2] for s in survivors], dtype='float32')
        hyp_dec_alphas = [s[3] for s in survivors]
        next_w = numpy.array([w[-1] for w in hyp_samples], dtype='int64')
        next_state = next_state[parents].copy()      # DeviceArray: a device-side row gather
        acc_ctx = acc_ctx[parents].copy()
        acc_alpha = acc_alpha[parents].copy()

    if not stochastic and live_k > 0:     # dump what is still alive (nats.py:1068-1074)
        for idx in range(live_k):
            sample.append(hyp_samples[idx])
            sample_score.append(hyp_scores[idx])
            sample_dec_alphas.append(hyp_dec_alphas[idx])
    return sample, sample_score, sample_dec_alphas


# ----------------------------------------------------------------------------------------------------------
# validation cost and the training loop (nats.py:1080-1101, 1230-1539)
# ----------------------------------------------------------------------------------------------------------
def pred_probs(f_log_probs, prepare_data, options, iterator, verbose=True):
    probs = []
    n_done = 0
    for x, y in iterator:
        n_done += len(x)
        x, x_mask, y, y_mask = prepare_data(x, y, n_words=options['n_words'])
        probs.extend(f_log_probs(x, x_mask, y, y_mask))
        if numpy.isnan(numpy.mean(probs)):
            raise FloatingPointError('NaN validation cost')      # the reference drops into pdb here (:1095)
        if verbose:
            print('%d samples computed' % n_done, file=sys.stderr)
    return numpy.array(probs)


def _load_pickle(path):
    with open(path, 'rb') as f:
        try:
            return pkl.load(f)
        except UnicodeDecodeError:          # python-2 pickles written by the reference (nats.py:1434)
            f.seek(0)
            return pkl.load(f, encoding='latin1')


def _words(ids, worddicts_r):
    out = []
    for vv in ids:
        if vv == 0:
            break
        out.append(worddicts_r.get(vv, 'UNK'))
    return ' '.join(out)


def _prefetched(gen, depth):
    """run generator `gen` in a background thread, `depth` items ahead (0: inline).  The consumer spends its time inside
    cudaStreamSynchronize (GIL released), so the next batch is padded and ready when the step returns."""
    if depth <= 0:
        for item in gen:
            yield item
        return
    import queue
    import threading
    q = queue.Queue(maxsize=depth)
    END = object()

    def work():
        try:
            for item in gen:
                q.put(item)
            q.put(END)
        except BaseException as e:          # surfaced in the consumer
            q.put(e)
    th = threading.Thread(target=work, daemon=True)
    th.start()
    while True:
        item = q.get()
        if item is END:
            break
        if isinstance(item, BaseException):
            raise item
        yield item
    th.join()


def save_optimizer_state_file(path, f_grad_shared):
    """optimiser accumulators (flat buffers, packed layout of the parameter store) next to the model file; the model
    npz / pkl keep the reference's key set (nats.py:1427-1435)."""
    st = getattr(f_grad_shared, 'state', None) or {}
    out = {}
    for k, v in st.items():
        out[k] = v.detach().cpu().numpy() if hasattr(v, 'detach') else numpy.asarray(v)
    numpy.savez(path, **out)


def load_optimizer_state(path, f_grad_shared):
    import torch
    st = getattr(f_grad_shared, 'state', None) or {}
    z = numpy.load(path)
    for k, v in st.items():
        if k not in z.files:
            warnings.warn('%s is not in the optimizer archive' % k)
            continue
        if hasattr(v, 'copy_'):
            v.copy_(torch.from_numpy(z[k]))
        else:
            v[...] = z[k]


def train(dim_word=100, dim=1000, dim_att=100, encoder='gru', decoder='gru_cond', patience=10, max_epochs=5000,
          finish_after=10000000, dispFreq=100, decay_c=0., clip_c=-1., lrate=0.01, n_words=100000, maxlen=100,
          optimizer='adadelta', batch_size=16, valid_batch_size=16, saveto='model.npz', validFreq=1000,
          saveFreq=1000, sampleFreq=100, datasets=[], valid_datasets=[], dictionary='', use_dropout=False,
          reload_=False, verbose=False, bucket_batches=0, save_optimizer_state=False, prefetch=2):
    """Same keyword surface, side effects (npz + options pickle, log lines) and return value as the reference's
    train() (nats.py:1230-1539).  Ours, all defaulting to the reference behaviour:
      bucket_batches        k > 0: the training iterator sorts k batches by source length before cutting them;
      save_optimizer_state  also write / reload `<saveto>.opt.npz` (the reference loses the accumulators, nats.py:1433);
      prefetch              batches prepared ahead by a background thread (0 = inline as the reference).
    Under torchrun (one process per GPU, NCCL) every rank reads the same files; each global batch is sharded over the
    ranks, gradients are all-reduced once per update, rank 0 alone saves / samples / logs."""
    logging.basicConfig(level=logging.DEBUG, format="%(asctime)s: %(name)s: %(levelname)s: %(message)s")
    model_options = locals().copy()
    for _k in ('save_optimizer_state', 'prefetch'):      # not part of the reference's option pickle
        model_options.pop(_k)
    rank, world = parallel.world()
    is_main = rank == 0

    worddicts = _load_pickle(dictionary)
    worddicts_r = dict((vv, kk) for kk, vv in worddicts.items())

    if reload_ and os.path.exists(saveto):
        print('Reload options')
        model_options = _load_pickle('%s.pkl' % saveto)
    logger.debug(pprint.pformat(model_options))

    print('Loading data')
    train_it = TextIterator(datasets[0], datasets[1], dictionary, n_words=n_words, batch_size=batch_size,
                            bucket_batches=bucket_batches)
    valid_it = TextIterator(valid_datasets[0], valid_datasets[1], dictionary, n_words=n_words,
                            batch_size=valid_batch_size)

    print('Building model')
    params = init_params(model_options)
    if reload_ and os.path.exists(saveto):
        print('Reload parameters')
        params = load_params(saveto, params)
    tparams = init_tparams(params)

    trng, use_noise, x, x_mask, y, y_mask, opt_ret, cost = build_model(tparams, model_options)
    inps = [x, x_mask, y, y_mask]
    print('Buliding sampler')
    f_init, f_next = build_sampler(tparams, model_options, trng)

    print('Building f_log_probs...', end=' ')
    f_log_probs = cost.f_log_probs
    print('Done')
    cost = cost.mean()
    cost.decay_c = float(decay_c) if decay_c > 0. else 0.          # nats.py:1326-1332
    print('Building f_cost...', end=' ')
    f_cost = cost.f_cost                                           # noqa: F841 (compiled, unused: as the reference)
    print('Done')
    print('Computing gradient...', end=' ')
    cost.clip_c = float(clip_c)                                    # nats.py:1344-1353
    grads = cost
    print('Done')

    lr = 'lr'
    print('Building optimizers...', end=' ')
    f_grad_shared, f_update = _OPTIMIZERS[optimizer](lr, tparams, grads, inps, cost)
    print('Done')
    opt_path = '%s.opt.npz' % saveto
    if save_optimizer_state and reload_ and os.path.exists(opt_path):
        print('Reload optimizer state')
        load_optimizer_state(opt_path, f_grad_shared)
    # one workspace for the largest batch this run can produce: no regrowth (= no graph re-capture) later
    grads.reserve(maxlen + 1, maxlen + 1, max(1, (batch_size + world - 1) // world))
    print('Optimization')

    history_errs = []
    if reload_ and os.path.exists(saveto):
        print('Reload history error')
        history_errs = list(numpy.load(saveto, allow_pickle=True)['history_errs'])
    best_p = None
    bad_counter = 0

    if validFreq == -1 or saveFreq == -1 or sampleFreq == -1:
        n_train = sum(1 for _ in open(datasets[0], 'r'))
        per_epoch = max(1, n_train // batch_size)
        validFreq = per_epoch if validFreq == -1 else validFreq
        saveFreq = per_epoch if saveFreq == -1 else saveFreq
        sampleFreq = per_epoch if sampleFreq == -1 else sampleFreq

    def _prepared(it):
        """global batch -> this rank's shard -> padded arrays (host work a background thread can do ahead of time)"""
        for bx, by in it:
            n_global = len(bx)
            if world > 1:
                bx, by, n_global = parallel.shard_batch(bx, by, rank, world)
            if len(bx) == 0:
                yield None, None, None, None, n_global, 0
                continue
            x_, xm_, y_, ym_ = prepare_data(bx, by, maxlen=maxlen, n_words=n_words)
            yield x_, xm_, y_, ym_, n_global, len(bx)

    uidx = 0
    estop = False
    for eidx in range(max_epochs):
        n_samples = 0
        for x, x_mask, y, y_mask, n_global, n_local in _prefetched(_prepared(train_it), prefetch):
            n_samples += n_global
            uidx += 1
            use_noise.set_value(1.)
            if x is None and world == 1:
                print('Minibatch with zero sample under length ', maxlen)
                uidx -= 1
                continue

            ud_start = time.time()
            cost_v = f_grad_shared(x, x_mask, y, y_mask, global_batch=n_global)
            if verbose and clip_c > 0.:
                norm_g = float(numpy.sqrt(grads.stats[0].item()))
            f_update(lrate)
            ud = time.time() - ud_start

            if numpy.isnan(cost_v) or numpy.isinf(cost_v):
                print('NaN detected')
                return 1., 1., 1.

            if numpy.mod(uidx, dispFreq) == 0 and is_main:
                logger.debug('Epoch {0} Update {1} Cost {2} UD {3}'.format(eidx, uidx, cost_v, ud))
                if verbose and clip_c > 0.:
                    logger.debug('Grad {0}'.format(norm_g))

            if numpy.mod(uidx, saveFreq) == 0 and is_main:
                print('Saving...', end=' ')
                params = best_p if best_p is not None else unzip(tparams)
                numpy.savez(saveto, history_errs=history_errs, **params)
                with open('%s.pkl' % saveto, 'wb') as f:
                    pkl.dump(model_options, f, protocol=2)
                if save_optimizer_state:
                    save_optimizer_state_file(opt_path, f_grad_shared)
                print('Done')

            if numpy.mod(uidx, sampleFreq) == 0 and is_main and x is not None:
                for jj in range(int(numpy.minimum(5, x.shape[1]))):
                    sample, score, dec_alphas = gen_sample(tparams, f_init, f_next, x[:, jj][:, None], model_options,
                                                           trng=trng, k=1, maxlen=30, stochastic=True, argmax=False)
                    print('Source ', jj, ': ', _words(x[:, jj], worddicts_r))
                    print('Truth ', jj, ' : ', _words(y[:, jj], worddicts_r))
                    print('Sample ', jj, ': ', _words(sample, worddicts_r))

            if numpy.mod(uidx, validFreq) == 0:
                use_noise.set_value(0.)
                valid_errs = pred_probs(f_log_probs, prepare_data, model_options, valid_it)
                valid_err = valid_errs.mean()
                history_errs.append(valid_err)
                if uidx == 0 or valid_err <= numpy.array(history_errs).min():
                    best_p = unzip(tparams)
                    bad_counter = 0
                if patience == 0:
                    if len(history_errs) > 1 and valid_err >= numpy.array(history_errs)[:-1].min():
                        print('Early Stop!')
                        estop = True
                        break
                elif len(history_errs) > patience and valid_err >= numpy.array(history_errs)[:-patience].min():
                    bad_counter += 1
                    if bad_counter > patience:
                        print('Early Stop!')
                        estop = True
                        break
                if numpy.isnan(valid_err):
                    raise FloatingPointError('NaN validation error')
                print('Valid ', valid_err)

            if uidx >= finish_after:
                print('Finishing after %d iterations!' % uidx)
                estop = True
                break

        print('Seen %d samples' % n_samples)
        if estop:
            break

    if best_p is not None:
        zipp(best_p, tparams)
    use_noise.set_value(0.)
    valid_err = pred_probs(f_log_probs, prepare_data, model_options, valid_it).mean()
    print('Valid ', valid_err)

    params = copy.copy(best_p) if best_p is not None else unzip(tparams)
    if is_main:
        numpy.savez(saveto, zipped_params=best_p, history_errs=history_errs, **params)
        if save_optimizer_state:
            save_optimizer_state_file(opt_path, f_grad_shared)
    logger.debug('Done')
    return valid_err


if __name__ == '__main__':
    pass
