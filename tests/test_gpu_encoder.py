"""The bidirectional GRU encoder recurrence (persistent kernel `enc_tc_kernel`, nats_b200/csrc/enc_tc.cu, and the
per-step path for the shapes it does not take) against the float64 oracle, case by case across the kernel's tile plans.

Each case drives the C ABI directly on its own workspace:
  * forward:  nats_encoder_fwd; the `ctx` and `init_state` views against O.gru_layer_fwd of both directions (every
    position, padding included: the state is carried there) and the oracle's init_state;
  * backward: nats_train_fwd + nats_train_bwd_begin, snapshot of the gradient buffer, nats_train_bwd_finish.  The `dcc` /
    `dmean` views hold the gradient the encoder backward consumed; exactly those float32 values go through
    O.gru_layer_bwd of both directions (O.model_bwd, the encoder part), and the result is compared with the encoder
    gradients and the source-side part of the Wemb gradient (after the finish minus the snapshot);
  * path:     the profiler counts the persistent launches (once per pass, or zero on the per-step path), so a plan
    change cannot quietly move a case to the other path.

Errors are in three families with one bound each: the states (forward max abs error), the gradients that come from the
recurrence alone (the bias gradients are column sums of dGx; the source-side Wemb gradient is dGx . Wcat^T), and those
fed through the d[U|Ux] / d[W|Wx] products (U, Ux, W, Wx).  test_bounds_reject_a_degraded_kernel (no GPU) emulates the
kernel's arithmetic on the same inputs and shows that each bound is at most a quarter of the error of a kernel that
drops one of the two 3xTF32 correction terms, or of single-pass TF32."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import nats_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V, W, A, TY = 64, 16, 8, 3          # a cheap decoder: D and the batch are what the encoder's plans depend on

# What each case reaches in plan() (enc_tc.cu) on an H100 (132 SMs, 227 KB of shared memory per block).  BN: batch
# columns of the MMA tile; forward tiles are NT row tiles x S K chunks of D, backward ones x S K chunks of 3D; Kc: the K
# chunk (kc = forward, backward, for the emulation); a CTA finishes dps units of its tile per step.  Ragged masks with a
# full-length column and a column of length 1, except where n = 1.
CASES = [
    # smallest eligible D, Tx = 1: no recurrent step at all (the product never runs)
    dict(n=1, D=96, Tx=1, persistent=True, kc=(32, 32)),
    # BN = 32 with 31 zero-filled batch rows; forward 20 tiles of 5 units x 3 chunks: the last tile holds 1 unit, so two
    # of its CTAs finish none (nds = 0); backward 7 x 9, three CTAs of the last tile finish none; forward also with
    # x_mask NULL
    dict(n=1, D=96, Tx=7, persistent=True, kc=(32, 32)),
    # forward last K chunk 36 deep (one full and one partial k-block); backward last chunk 12 deep
    dict(n=5, D=100, Tx=23, persistent=True, kc=(64, 32)),
    # forward last K chunk exactly one k-step (8 deep); CTAs with no units in both passes
    dict(n=32, D=200, Tx=40, persistent=True, kc=(64, 64)),
    # BN = 64 with 31 empty batch rows: EPT = 4, the non-deferred gate branch; backward 5 x 12 chunks
    dict(n=33, D=256, Tx=31, persistent=True, kc=(64, 64)),
    # BASELINE config 2 shape: BN = 64, two warpgroups in both passes, 12 backward K chunks, a 4-stage ring
    dict(n=64, D=500, Tx=120, persistent=True, kc=(128, 128)),
    # three warpgroups in both passes: 144-row forward and 154-row backward tiles
    dict(n=17, D=768, Tx=25, persistent=True, kc=(192, 192)),
    # NS = 2 ring under 8 (forward) / 12 (backward) k-blocks per step; three forward warpgroups (189 rows)
    dict(n=64, D=1000, Tx=40, persistent=True, kc=(256, 384)),
    # not eligible (n > 64, D % 4 != 0): the per-step path, against the same oracle and bounds
    dict(n=65, D=256, Tx=20, persistent=False, kc=None),
    dict(n=8, D=98, Tx=15, persistent=False, kc=None),
]
for _c in CASES:
    _c['id'] = 'n%d_d%d_t%d' % (_c['n'], _c['D'], _c['Tx'])
    _c['seed'] = 7919 * _c['n'] + 31 * _c['D'] + _c['Tx']

DIRS = ('encoder', 'encoder_r')
GEMM_FED = ('U', 'Ux', 'W', 'Wx')
RECURRENCE = ('b', 'bx', 'Wemb')

# Measured on an H100 80GB HBM3 at a 700 W power limit: per case, the forward max abs error (ctx and init_state) and
# each gradient's relative error ||g - g*|| / ||g*|| (the worse of the two directions; Wemb: the source-side part).
# U / Ux at D >= 500 are limited by the d[U|Ux] product itself (fp32 accumulation over K = (Tx - 1) n = 7616 / 2496),
# which both encoder paths share.
#                      fwd     U       Ux      W       Wx      b       bx      Wemb
MEASURED = {
    'n1_d96_t1':     (5.8e-8, 0.0,    0.0,    9.8e-8, 8.5e-8, 9.3e-8, 8.0e-8, 2.0e-7),
    'n1_d96_t7':     (2.2e-7, 3.8e-7, 2.3e-7, 2.4e-7, 1.8e-7, 4.3e-7, 1.4e-7, 2.2e-7),
    'n5_d100_t23':   (2.5e-7, 7.7e-7, 6.4e-7, 3.4e-7, 2.8e-7, 3.4e-7, 1.7e-7, 6.4e-7),
    'n32_d200_t40':  (3.2e-7, 7.7e-7, 6.8e-7, 3.2e-7, 3.1e-7, 5.4e-7, 2.1e-7, 9.2e-7),
    'n33_d256_t31':  (3.1e-7, 8.1e-7, 6.8e-7, 3.6e-7, 3.4e-7, 4.3e-7, 2.0e-7, 8.6e-7),
    'n64_d500_t120': (5.5e-7, 4.1e-6, 5.0e-6, 9.9e-7, 1.1e-6, 7.9e-7, 3.0e-7, 9.1e-7),
    'n17_d768_t25':  (6.6e-7, 1.3e-6, 1.1e-6, 4.2e-7, 4.1e-7, 6.7e-7, 2.8e-7, 3.6e-7),
    'n64_d1000_t40': (6.6e-7, 4.5e-6, 4.7e-6, 9.0e-7, 9.2e-7, 1.1e-6, 4.9e-7, 8.9e-7),
    'n65_d256_t20':  (3.0e-7, 6.9e-7, 5.6e-7, 3.0e-7, 2.9e-7, 3.3e-7, 1.5e-7, 5.2e-7),
    'n8_d98_t15':    (1.5e-7, 3.1e-7, 2.2e-7, 2.7e-7, 2.5e-7, 1.9e-7, 9.2e-8, 5.3e-7),
    # NATS_ENC_TC=0: the per-step path on shapes the persistent kernel takes
    'n5_d100_t23 per-step':   (1.5e-7, 5.9e-7, 5.3e-7, 2.6e-7, 2.5e-7, 2.0e-7, 9.5e-8, 6.4e-7),
    'n64_d500_t120 per-step': (2.1e-7, 3.8e-6, 4.9e-6, 9.1e-7, 9.5e-7, 2.4e-7, 1.3e-7, 8.7e-7),
}
MEASURED_COLUMNS = ('fwd', 'U', 'Ux', 'W', 'Wx', 'b', 'bx', 'Wemb')

# About four times the worst measured value of each family.  A backward without A_lo.B_raw measured 1.9-2.1e-4 on
# every encoder gradient at D = 500 and 1000 (same card).
BOUND = {'fwd': 3e-6, 'recurrence': 5e-6, 'gemm': 2e-5}


def _options(D):
    return dict(dim_word=W, dim=D, dim_att=A, n_words=V, encoder='gru', decoder='gru_cond')


def _params(case):
    """Reference init (orthogonal U / Ux) under the case's seed, non-zero biases and a livelier source side: with
    dim_word = 16 the reference scales (Wemb and W / Wx at N(0, 0.01^2)) would leave the input projection near zero."""
    np.random.seed(case['seed'])
    P = O.init_params(_options(case['D']))
    rng = np.random.RandomState(case['seed'] + 1)
    for k in P:
        if P[k].ndim == 1:
            P[k] = (0.1 * rng.randn(*P[k].shape)).astype('float32')
    P['Wemb'] = (P['Wemb'] * 30).astype('float32')
    for d in DIRS:
        P[d + '_W'] = (P[d + '_W'] * 30).astype('float32')
        P[d + '_Wx'] = (P[d + '_Wx'] * 30).astype('float32')
    P['ff_logit_W'] = (P['ff_logit_W'] * 40).astype('float32')
    P['decoder_U_att'] = (P['decoder_U_att'] * 30).astype('float32')
    return P


def _batch(case):
    n, Tx = case['n'], case['Tx']
    rs = np.random.RandomState(case['seed'] + 2)
    lx = rs.randint(1, Tx + 1, size=n)          # valid positions per column, EOS included
    ly = rs.randint(1, TY + 1, size=n)
    lx[0], ly[0] = Tx, TY
    if n > 1:
        lx[1] = 1
    sx = [list(rs.randint(2, V, size=L - 1)) for L in lx]
    sy = [list(rs.randint(2, V, size=L - 1)) for L in ly]
    batch = O.prepare_data(sx, sy, n_words=V)
    assert batch[0].shape == (Tx, n) and batch[2].shape == (TY, n)
    return batch


def _relerr(g, ref):
    nr = np.linalg.norm(ref)
    if nr == 0.0:
        return 0.0 if not np.any(g) else np.inf
    return float(np.linalg.norm(np.asarray(g, 'float64') - ref) / nr)


def _oracle_fwd(P, x, xm):
    """float64 encoder forward as O.model_fwd runs it (nats.py:700-724): both directions, ctx, init_state"""
    Tx, n = x.shape
    emb = P['Wemb'][x.flatten()].reshape(Tx, n, -1)
    xm = xm.astype('float64')
    Hf, cf = O.gru_layer_fwd(P, 'encoder', emb, xm)
    Hr, cr = O.gru_layer_fwd(P, 'encoder_r', emb[::-1], xm[::-1])
    ctx = np.concatenate([Hf, Hr[::-1]], axis=2)
    xsum = xm.sum(0)
    mean = (ctx * xm[:, :, None]).sum(0) / xsum[:, None]
    init = np.tanh(mean @ P['ff_state_W'] + P['ff_state_b'])
    return ctx, init, cf, cr, xsum


def _family_errors(errs):
    out = {'fwd': errs['fwd']}
    out['recurrence'] = max(errs[k] for k in RECURRENCE)
    out['gemm'] = max(errs[k] for k in GEMM_FED)
    return out


# ------------------------------------------------------------------------------------------------ device
def _launches(lib, eng):
    n = lib.nats_profile_num_classes()
    ms, fl, by, la = (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_int64 * n)()
    from nats_b200 import _lib
    _lib.check(lib.nats_profile_read(eng.ctx, n, ms, fl, by, la), 'nats_profile_read')
    lib.nats_profile_enable(eng.ctx, 0)
    names = [lib.nats_profile_class_name(i).decode() for i in range(n)]
    return {k: int(la[names.index(k)]) for k in ('enc_tc_fwd', 'enc_tc_bwd')}


def _device_run(case, P32, batch, null_mask=False, repeat=1):
    """the case through the C ABI; returns the forward views, the dcc / dmean views, the gradients before / after the
    encoder backward and the persistent launches of each part (one dict per repetition on the same workspace)"""
    import torch
    from nats_b200 import nats, _lib
    eng = nats.get_engine()
    lib = eng.lib
    tparams = nats.init_tparams(P32)
    D, C = case['D'], 2 * case['D']
    x, xm, y, ym = batch
    Tx, n = x.shape
    dims = _lib.Dims(V, W, D, A)
    dev = eng.device
    xd, xmd, yd, ymd = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in batch]
    ones = torch.ones_like(xmd)
    nbytes = int(lib.nats_train_workspace_bytes(ctypes.byref(dims), Tx, TY, n))
    assert nbytes > 0
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    cost = torch.zeros(n, dtype=torch.float32, device=dev)
    grads = torch.zeros(tparams.total + _lib.GRAD_TAIL, dtype=torch.float32, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    st = eng.stream()

    def view(name, shape):
        ptr = lib.nats_train_ws_view(ctypes.byref(dims), Tx, TY, n, p(ws), name.encode())
        assert ptr, name
        off = (ptr - ws.data_ptr()) // 4
        return ws.view(torch.float32)[off:off + int(np.prod(shape))].cpu().numpy().reshape(shape).copy()

    def enc_fwd(mask):
        _lib.check(lib.nats_encoder_fwd(eng.ctx, st, ctypes.byref(dims), p(tparams.flat), p(xd), p(mask), Tx, TY, n,
                                        p(ws), nbytes), 'nats_encoder_fwd')

    train = lambda fn: _lib.check(fn(eng.ctx, st, ctypes.byref(dims), p(tparams.flat), p(xd), p(xmd), p(yd), p(ymd),
                                     Tx, TY, n, p(ws), nbytes, ctypes.c_float(1.0 / n), p(grads)), 'nats_train_bwd')
    runs = []
    for _ in range(repeat):
        out = {}
        _lib.check(lib.nats_profile_enable(eng.ctx, 1), 'nats_profile_enable')
        enc_fwd(xmd)
        out['fwd_launches'] = _launches(lib, eng)
        out['ctx'] = view('ctx', (Tx, n, C))
        out['init_state'] = view('init_state', (n, D))
        if null_mask:
            enc_fwd(None)
            out['ctx_null'] = view('ctx', (Tx, n, C))
            out['init_null'] = view('init_state', (n, D))
            enc_fwd(ones)
            out['ctx_ones'] = view('ctx', (Tx, n, C))
        _lib.check(lib.nats_profile_enable(eng.ctx, 1), 'nats_profile_enable')
        _lib.check(lib.nats_train_fwd(eng.ctx, st, ctypes.byref(dims), p(tparams.flat), p(xd), p(xmd), p(yd), p(ymd),
                                      Tx, TY, n, p(ws), nbytes, p(cost)), 'nats_train_fwd')
        train(lib.nats_train_bwd_begin)
        before = grads.clone()
        train(lib.nats_train_bwd_finish)
        out['train_launches'] = _launches(lib, eng)
        out['dcc'] = view('dcc', (Tx, n, C))
        out['dmean'] = view('dmean', (n, C))
        out['G0'] = tparams.view_of(before)
        out['G'] = tparams.view_of(grads)
        runs.append(out)
    torch.cuda.synchronize()
    return runs


def _device_errors(P, batch, out):
    """forward max abs error and per-tensor gradient relative errors of one device run against float64"""
    x, xm = batch[0], batch[1]
    Tx, n = x.shape
    D = P['encoder_Ux'].shape[1]
    ctx, init, cf, cr, xsum = _oracle_fwd(P, x, xm)
    errs = {'fwd': float(max(np.abs(out['ctx'] - ctx).max(), np.abs(out['init_state'] - init).max()))}
    # the gradient the encoder consumed, exactly as the device holds it (nats.py:717: dmean is not yet divided by the
    # length; the kernel multiplies it by xinv)
    xm64 = xm.astype('float64')
    dctx = out['dcc'].astype('float64') + xm64[:, :, None] * (out['dmean'].astype('float64') / xsum[:, None])[None]
    G = O.zero_grads(P)
    demb_f = O.gru_layer_bwd(P, 'encoder', cf, dctx[:, :, :D], G)
    demb_r = O.gru_layer_bwd(P, 'encoder_r', cr, dctx[::-1, :, D:], G)
    Wsrc = np.zeros_like(P['Wemb'])
    np.add.at(Wsrc, x.flatten(), demb_f.reshape(Tx * n, -1))
    np.add.at(Wsrc, x[::-1].flatten(), demb_r.reshape(Tx * n, -1))
    for t in GEMM_FED + ('b', 'bx'):
        errs[t] = max(_relerr(out['G'][d + '_' + t], G[d + '_' + t]) for d in DIRS)
    errs['Wemb'] = _relerr(out['G']['Wemb'].astype('float64') - out['G0']['Wemb'], Wsrc)
    return errs


def _expected_launches(case):
    on = os.environ.get('NATS_ENC_TC', '1')
    return (int(case['persistent'] and on in ('1', '2')), int(case['persistent'] and on in ('1', '3')))


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c['id'] for c in CASES])
def test_encoder_vs_float64(case):
    P32 = _params(case)
    P = O.cast_params(P32, 'float64')
    batch = _batch(case)
    null_mask = case['n'] == 1
    out = _device_run(case, P32, batch, null_mask=null_mask)[0]
    pf, pb = _expected_launches(case)
    assert out['fwd_launches'] == {'enc_tc_fwd': pf, 'enc_tc_bwd': 0}, out['fwd_launches']
    assert out['train_launches'] == {'enc_tc_fwd': pf, 'enc_tc_bwd': pb}, out['train_launches']
    if null_mask:                       # x_mask NULL = all ones (the f_init encoder), bit for bit
        assert np.all(batch[1] == 1)
        np.testing.assert_array_equal(out['ctx_null'], out['ctx'])
        np.testing.assert_array_equal(out['ctx_ones'], out['ctx'])
        np.testing.assert_array_equal(out['init_null'], out['init_state'])
    errs = _device_errors(P, batch, out)
    print('encoder errors', case['id'], json.dumps(errs))
    fam = _family_errors(errs)
    assert fam['fwd'] <= BOUND['fwd'], (case['id'], errs)
    for t in RECURRENCE:
        assert errs[t] <= BOUND['recurrence'], (case['id'], t, errs)
    for t in GEMM_FED:
        assert errs[t] <= BOUND['gemm'], (case['id'], t, errs)


@pytest.mark.gpu
def test_encoder_is_deterministic():
    """The K partials of a row tile are summed in a fixed order: two runs on the same workspace give the same bits.
    This also checks that the step tags and the tile counters are reset between launches."""
    case = next(c for c in CASES if c['D'] == 1000)
    r1, r2 = _device_run(case, _params(case), _batch(case), repeat=2)
    np.testing.assert_array_equal(r1['ctx'], r2['ctx'])
    np.testing.assert_array_equal(r1['init_state'], r2['init_state'])
    for d in DIRS:
        for t in GEMM_FED + ('b', 'bx'):
            np.testing.assert_array_equal(r1['G'][d + '_' + t], r2['G'][d + '_' + t], err_msg=d + '_' + t)


@pytest.mark.gpu
def test_per_step_path_vs_float64():
    """NATS_ENC_TC=0 (read at context creation, hence a fresh process): two cases the persistent kernel would take run
    on the per-step path (grouped split-K product + gate kernel per step), with no persistent launch, under the same
    bounds."""
    env = dict(os.environ, NATS_ENC_TC='0')
    r = subprocess.run([sys.executable, '-m', 'pytest', '-x', '-q', '-s', '-m', 'gpu', 'tests/test_gpu_encoder.py', '-k',
                        'test_encoder_vs_float64 and (n5_d100_t23 or n64_d500_t120)'],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print('\n'.join(l for l in r.stdout.splitlines() if l.startswith('encoder errors')))
    assert r.returncode == 0 and '2 passed' in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ emulation (no GPU)
def _tf32(x):
    """the tf32 operand the tensor core reads from a raw fp32 word: its upper 19 bits (truncation)"""
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _kernel_product(b, a, kc, variant):
    """b [n, K] (the moving operand: h_{t-1} / dG) times a [K, M] (the stationary weights) as enc_tc_kernel forms it:
    per K chunk of kc, acc_hh = A_raw.B_raw and acc_x = A_raw.B_lo + A_lo.B_raw (raw = the word read as tf32,
    lo = resid(word)), the chunk's partial acc_hh + acc_x in fp32, the partials summed in ascending chunk order.
    variant: '3x', 'no_a_lo' (without A_lo.B_raw), 'no_b_lo' (without A_raw.B_lo) or '1x' (single pass)."""
    b = np.asarray(b, np.float32)
    a = np.asarray(a, np.float32)
    out = np.zeros((b.shape[0], a.shape[1]), np.float32)
    for k0 in range(0, a.shape[0], kc):
        bc, ac = b[:, k0:k0 + kc], a[k0:k0 + kc]
        bh, ah = _tf32(bc), _tf32(ac)
        hh = bh.astype(np.float64) @ ah.astype(np.float64)
        x = np.zeros_like(hh)
        if variant in ('3x', 'no_a_lo'):
            x += (bc - bh).astype(np.float64) @ ah.astype(np.float64)
        if variant in ('3x', 'no_b_lo'):
            x += bh.astype(np.float64) @ (ac - ah).astype(np.float64)
        out += hh.astype(np.float32) + x.astype(np.float32)
    return out


def _sig32(v):
    return (1.0 / (1.0 + np.exp(-v))).astype(np.float32)


def _emulate_fwd(P, prefix, emb, mask, kc, variant):
    """the forward gate arithmetic of enc_tc_kernel in fp32 (nats.py:336-356) around _kernel_product"""
    D = P[prefix + '_Ux'].shape[1]
    Ucat = np.concatenate([P[prefix + '_U'], P[prefix + '_Ux']], axis=1).astype(np.float32)
    xp = np.concatenate([emb @ P[prefix + '_W'] + P[prefix + '_b'], emb @ P[prefix + '_Wx'] + P[prefix + '_bx']],
                        axis=2).astype(np.float32)
    T, n = mask.shape
    h = np.zeros((n, D), np.float32)
    H = np.zeros((T, n, D), np.float32)
    for t in range(T):
        pre = _kernel_product(h, Ucat, kc, variant) if t > 0 else np.zeros((n, 3 * D), np.float32)
        r = _sig32(pre[:, :D] + xp[t, :, :D])
        u = _sig32(pre[:, D:2 * D] + xp[t, :, D:2 * D])
        c = np.tanh(pre[:, 2 * D:] * r + xp[t, :, 2 * D:])
        m = mask[t][:, None].astype(np.float32)
        h = m * (u * h + (1 - u) * c) + (1 - m) * h
        H[t] = h
    return H


def _emulate_bwd(P, prefix, cache, dH, kc, variant):
    """the backward gate arithmetic of enc_tc_kernel in fp32 around _kernel_product, on the float64 forward's saved
    gates (rounded to fp32, as the device saves them); the weight gradients and d emb from its dG / dGx in float64"""
    D = P[prefix + '_Ux'].shape[1]
    Ucat_t = np.concatenate([P[prefix + '_U'], P[prefix + '_Ux']], axis=1).T.astype(np.float32)
    f32 = lambda k: cache[k].astype(np.float32)
    R, Ug, Cn, Pp, H = f32('R'), f32('U'), f32('C'), f32('P'), f32('H')
    mask = cache['mask']
    T, n = mask.shape
    dG = np.zeros((T, n, 3 * D), np.float32)
    dGx = np.zeros((T, n, 3 * D), np.float32)
    carry = np.zeros((n, D), np.float32)
    prod = np.zeros((n, D), np.float32)
    for t in range(T - 1, -1, -1):
        m = mask[t][:, None].astype(np.float32)
        hp = H[t - 1] if t > 0 else np.zeros((n, D), np.float32)
        r, u, c, p = R[t], Ug[t], Cn[t], Pp[t]
        dh = dH[t].astype(np.float32) + carry + prod
        dhn = m * dh
        du = dhn * (hp - c)
        dc = dhn * (1 - u)
        dpc = dc * (1 - c * c)
        dgr = dpc * p * r * (1 - r)
        dgu = du * u * (1 - u)
        dG[t] = np.concatenate([dgr, dgu, dpc * r], axis=1)
        dGx[t] = np.concatenate([dgr, dgu, dpc], axis=1)
        carry = (1 - m) * dh + dhn * u
        prod = _kernel_product(dG[t], Ucat_t, kc, variant) if t > 0 else prod
    dG, dGx = dG.astype(np.float64), dGx.astype(np.float64)
    Hp = np.concatenate([np.zeros((1, n, D)), H[:-1].astype(np.float64)], axis=0).reshape(T * n, D)
    dUcat = Hp.T @ dG.reshape(T * n, 3 * D)
    e2 = cache['emb'].reshape(T * n, -1)
    dWcat = e2.T @ dGx.reshape(T * n, 3 * D)
    g = {'U': dUcat[:, :2 * D], 'Ux': dUcat[:, 2 * D:], 'W': dWcat[:, :2 * D], 'Wx': dWcat[:, 2 * D:],
         'b': dGx.sum((0, 1))[:2 * D], 'bx': dGx.sum((0, 1))[2 * D:]}
    Wcat = np.concatenate([P[prefix + '_W'], P[prefix + '_Wx']], axis=1)
    return g, dGx @ Wcat.T


def _emulated_errors(case, variants):
    """-> {variant: per-tensor errors} of the emulated kernel against float64 on the case's inputs.  The forward is
    emulated alone; the backward is emulated on the float64 forward, with the gradient arriving at the states taken from
    the oracle's own model_bwd (its decoder backward), so each pass is judged in isolation."""
    P = O.cast_params(_params(case), 'float64')
    batch = _batch(case)
    x = batch[0]
    Tx, n = x.shape
    _, cache = O.model_fwd(P, *batch)
    seen = {}
    orig = O.gru_layer_bwd

    def capture(P_, prefix, c, dH, G):
        seen[prefix] = (c, dH)
        return orig(P_, prefix, c, dH, G)

    O.gru_layer_bwd = capture
    try:
        G = O.model_bwd(P, cache, np.full(n, 1.0 / n))
    finally:
        O.gru_layer_bwd = orig
    Wsrc = np.zeros_like(P['Wemb'])
    for d, xs in zip(DIRS, (x, x[::-1])):
        c, dH = seen[d]
        Gd = O.zero_grads(P)
        np.add.at(Wsrc, xs.flatten(), orig(P, d, c, dH, Gd).reshape(Tx * n, -1))
    kf, kb = case['kc']
    out = {}
    for v in variants:
        errs = {'fwd': 0.0}
        Wem = np.zeros_like(P['Wemb'])
        for d, xs in zip(DIRS, (x, x[::-1])):
            c, dH = seen[d]
            Hd = _emulate_fwd(P, d, c['emb'], c['mask'], kf, v)
            errs['fwd'] = max(errs['fwd'], float(np.abs(Hd - c['H']).max()))
            g, demb = _emulate_bwd(P, d, c, dH, kb, v)
            for t in g:
                errs[t] = max(errs.get(t, 0.0), _relerr(g[t], G[d + '_' + t]))
            np.add.at(Wem, xs.flatten(), demb.reshape(Tx * n, -1))
        errs['Wemb'] = _relerr(Wem, Wsrc)
        out[v] = errs
    return out


# the persistent cases with at least one recurrent step up to D = 256, and the D = 500 case at a shorter Tx (the
# degraded error hardly depends on D or Tx)
EMULATED = ([c for c in CASES if c['persistent'] and c['Tx'] > 1 and c['D'] <= 256] +
            [dict(c, Tx=30, id='n64_d500_t30') for c in CASES if c['id'] == 'n64_d500_t120'])


def test_bounds_reject_a_degraded_kernel():
    """Every bound sits at most at a quarter of the smallest error, over the emulated cases, of an emulated kernel that
    drops A_lo.B_raw or A_raw.B_lo, or runs single-pass TF32 -- in the forward for the state bound, in the backward for
    the two gradient bounds -- and above every recorded device error of its family.  The emulated 3xTF32 kernel itself
    stays within the bounds."""
    for case, errs in MEASURED.items():
        e = dict(zip(MEASURED_COLUMNS, errs))
        for fam, v in _family_errors(e).items():
            assert v <= BOUND[fam], (case, fam, v)
    worst = {}
    for case in EMULATED:
        res = _emulated_errors(case, ('3x', 'no_a_lo', 'no_b_lo', '1x'))
        print(case['id'], json.dumps(res))
        for v, errs in res.items():
            for fam, e in _family_errors(errs).items():
                if v == '3x':
                    assert e <= BOUND[fam], (case['id'], fam, e)
                else:
                    # the degraded kernel must fail every tensor of the family, not only the worst one
                    low = errs['fwd'] if fam == 'fwd' else min(errs[t] for t in (RECURRENCE if fam == 'recurrence'
                                                                                  else GEMM_FED))
                    worst[fam] = min(worst.get(fam, np.inf), low)
    print('smallest degraded error per family', worst)
    for fam in BOUND:
        assert BOUND[fam] <= worst[fam] / 4, (fam, BOUND[fam], worst[fam])
