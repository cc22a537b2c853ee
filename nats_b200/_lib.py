"""ctypes binding of libnats_b200.so (include/nats_b200.h).  There is NO fallback: if the CUDA library is
missing or fails to load, importing the product path raises."""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint64,
                    c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libnats_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'nats_b200.h')

NUM_PARAMS = 43
GRAD_TAIL = 32


class Dims(Structure):
    _fields_ = [('n_words', c_int32), ('dim_word', c_int32), ('dim', c_int32), ('dim_att', c_int32)]


class ParamView(Structure):
    _fields_ = [('name', c_char * 32), ('offset', c_int64), ('rows', c_int32), ('cols', c_int32),
                ('ld', c_int32), ('ndim', c_int32)]


_P = c_void_p     # device pointers travel as integers (tensor.data_ptr())


class BeamStep(Structure):
    """nats_beam_step_t of include/nats_b200.h, field for field"""
    _fields_ = ([('params', _P), ('next_w', _P), ('ctx', _P), ('pctx', _P),
                 ('Tx', c_int32), ('k', c_int32), ('maxlen', c_int32), ('use_unk', c_int32),
                 ('ws', _P), ('ws_bytes', c_int64)] +
                [(n, _P) for n in ('state_in', 'acc_ctx_in', 'acc_alpha_in', 'probs', 'state_out', 'alphaT', 'ctxs',
                                   'acc_ctx_out', 'acc_alpha_out')] +
                [('kl_factor', c_float), ('ctx_factor', c_float), ('state_factor', c_float)] +
                [(n, _P) for n in ('hist_alpha_in', 'hist_ctx_in', 'hist_state_in', 'scratch', 'pen', 'top_p', 'top_i',
                                   'counters', 'scores', 'tokens', 'parents', 'fin_parent', 'out_tokens', 'out_len',
                                   'out_score', 'out_alpha', 'host_counters', 'state_next', 'acc_ctx_next',
                                   'acc_alpha_next', 'hist_alpha_out', 'hist_ctx_out', 'hist_state_out')])


class BeamStepMany(Structure):
    """nats_beam_step_many_t of include/nats_b200.h: a group of n_src sentences x k rows"""
    _fields_ = [('beam', BeamStep), ('n_src', c_int32), ('src_len', _P)]

# name -> (restype, argtypes); mirrors include/nats_b200.h one to one (checked by tests/test_abi.py)
SIGNATURES = {
    'nats_last_error': (c_char_p, []),
    'nats_version': (c_int, []),
    'nats_ctx_create': (c_int, [c_int, POINTER(c_void_p)]),
    'nats_ctx_destroy': (c_int, [c_void_p]),
    'nats_param_layout': (c_int, [POINTER(Dims), POINTER(ParamView), POINTER(c_int64)]),
    'nats_train_workspace_bytes': (c_int64, [POINTER(Dims), c_int, c_int, c_int]),
    'nats_train_fwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64, _P]),
    'nats_train_bwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64,
                               c_float, _P]),
    'nats_grad_split': (c_int64, [POINTER(Dims)]),
    'nats_train_bwd_begin': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64,
                                     c_float, _P]),
    'nats_train_bwd_finish': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64,
                                      c_float, _P]),
    'nats_encoder_fwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, c_int, c_int, c_int, _P, c_int64]),
    'nats_decoder_scan_fwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64]),
    'nats_readout_nll_fwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, c_int, c_int, c_int, _P, c_int64, _P]),
    'nats_readout_nll_bwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, c_int, c_int, c_int, _P, c_int64,
                                     c_float, _P]),
    'nats_decoder_scan_bwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64,
                                      _P]),
    'nats_encoder_bwd': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, _P, c_int, c_int, c_int, _P, c_int64, _P]),
    'nats_train_ws_view': (c_void_p, [POINTER(Dims), c_int, c_int, c_int, _P, c_char_p]),
    'nats_sampler_workspace_bytes': (c_int64, [POINTER(Dims), c_int, c_int]),
    'nats_sampler_init': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, c_int, c_int, _P, c_int64, _P, _P, _P]),
    'nats_sampler_next': (c_int, [c_void_p, _P, POINTER(Dims), _P, _P, _P, c_int64, c_int64, _P, c_int64, c_int64,
                                  _P, _P, _P, c_int, c_int, c_uint64, c_uint64, _P, c_int64,
                                  _P, _P, _P, _P, _P, _P, _P]),
    'nats_grad_clip': (c_int, [c_void_p, _P, c_int64, _P, _P, c_float, c_float, _P]),
    'nats_adadelta_grad_shared': (c_int, [c_void_p, _P, c_int64, _P, _P, c_float]),
    'nats_adadelta_update': (c_int, [c_void_p, _P, c_int64, _P, _P, _P, _P, c_float, c_float]),
    'nats_adam_update': (c_int, [c_void_p, _P, c_int64, _P, _P, _P, _P, c_int64]),
    'nats_rmsprop_grad_shared': (c_int, [c_void_p, _P, c_int64, _P, _P, _P]),
    'nats_rmsprop_update': (c_int, [c_void_p, _P, c_int64, _P, _P, _P, _P, _P]),
    'nats_beam_distraction_scores': (c_int, [c_void_p, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                             _P, _P, _P, c_float, c_float, c_float, _P, _P]),
    'nats_beam_topk': (c_int, [c_void_p, _P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    'nats_beam_reorder_append': (c_int, [c_void_p, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int]),
    'nats_beam_select': (c_int, [c_void_p, _P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'nats_beam_advance': (c_int, [c_void_p, _P] + [_P] * 3 + [c_int] * 6 + [_P] * 16),
    'nats_beam_step': (c_int, [c_void_p, _P, POINTER(Dims), POINTER(BeamStep), c_int]),
    'nats_beam_step_many': (c_int, [c_void_p, _P, POINTER(Dims), POINTER(BeamStepMany), c_int]),
    'nats_debug_gemm': (c_int, [c_void_p, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P, c_int, _P, c_int,
                                _P, c_int, c_int, c_int, c_int64, c_int64, c_int64]),
    'nats_profile_enable': (c_int, [c_void_p, c_int]),
    'nats_profile_num_classes': (c_int, []),
    'nats_profile_class_name': (c_char_p, [c_int]),
    'nats_profile_read': (c_int, [c_void_p, c_int, POINTER(c_double), POINTER(c_double), POINTER(c_double),
                                  POINTER(c_int64)]),
}

_lib = None


class NatsB200Error(RuntimeError):
    pass


def load():
    """Load libnats_b200.so (once).  Raises NatsB200Error when it is absent -- there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NatsB200Error('%s not found: build it with `python nats_b200/csrc/build.py` '
                            '(or __graft_entry__.build()); nats_b200 has no CPU fallback' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=''):
    if rc != 0:
        msg = load().nats_last_error()
        raise NatsB200Error('%s failed (rc=%d): %s' % (what or 'libnats_b200 call', rc,
                                                      msg.decode() if msg else '?'))


def param_layout(n_words, dim_word, dim, dim_att):
    """-> (list of (name, offset, rows, cols, ld, ndim) in the reference order, total_floats).  Pure host call."""
    lib = load()
    d = Dims(n_words, dim_word, dim, dim_att)
    views = (ParamView * NUM_PARAMS)()
    total = c_int64(0)
    check(lib.nats_param_layout(ctypes.byref(d), views, ctypes.byref(total)), 'nats_param_layout')
    out = [(v.name.decode(), v.offset, v.rows, v.cols, v.ld, v.ndim) for v in views]
    return out, total.value
