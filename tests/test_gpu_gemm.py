"""The library's GEMM engine (FFMA and wgmma 3xTF32 paths) against numpy float64, through nats_debug_gemm."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(path, M, N, K, ta, tb, bias=False, accumulate=False, splitk=1, batch=1, seed=0, pad=0):
    import torch
    from nats_b200 import nats, _lib
    eng = nats.get_engine()
    rng = np.random.RandomState(seed)
    lda = (M if ta else K) + pad
    ldb = (K if tb else N) + pad
    ldc = N + pad
    A = rng.randn(batch, K if ta else M, lda).astype('float32')
    B = rng.randn(batch, N if tb else K, ldb).astype('float32')
    C0 = rng.randn(batch, M, ldc).astype('float32')
    bv = rng.randn(N).astype('float32')
    dev = eng.device
    Ad, Bd = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
    nsl = splitk if splitk > 1 else 1
    assert batch == 1 or splitk == 1
    Cd = torch.from_numpy(np.tile(C0, (nsl, 1, 1)).copy()).to(dev)          # [nsl or batch, M, ldc]
    bd = torch.from_numpy(bv).to(dev)
    rc = eng.lib.nats_debug_gemm(eng.ctx, eng.stream(), path, int(ta), int(tb), M, N, K,
                                 ctypes.c_void_p(Ad.data_ptr()), lda, ctypes.c_void_p(Bd.data_ptr()), ldb,
                                 ctypes.c_void_p(Cd.data_ptr()), ldc,
                                 ctypes.c_void_p(bd.data_ptr()) if bias else ctypes.c_void_p(0), int(accumulate),
                                 splitk, batch, A[0].size, B[0].size, C0[0].size)
    _lib.check(rc, 'nats_debug_gemm')
    torch.cuda.synchronize()
    out = Cd.cpu().numpy()
    ref = np.zeros((batch, M, N))
    for b in range(batch):
        a = A[b].astype('float64'); bb = B[b].astype('float64')
        a = a[:, :M].T if ta else a[:, :K]
        bb = bb[:, :K].T if tb else bb[:, :N]
        ref[b] = a @ bb
    if splitk > 1:
        got = out[:, :, :N].astype('float64').sum(0)[None]
        np.testing.assert_array_equal(out[:, :, N:], np.tile(C0[:, :, N:], (nsl, 1, 1)))   # padding untouched
    else:
        got = out[..., :N]
        np.testing.assert_array_equal(out[..., N:], C0[..., N:])
    if bias:
        ref = ref + bv[None, None, :]
    if accumulate:
        ref = ref + C0[..., :N]
    scale = np.sqrt(K) + (np.abs(C0).max() if accumulate else 0)
    return np.abs(got - ref).max() / scale


# max |err| / sqrt(K) for N(0,1) operands.  FFMA: fp32 rounding only.  3xTF32: the dropped lo.lo term and the
# accumulation on the tensor core; single-pass TF32 would sit at ~5e-4, i.e. an order of magnitude above this bound.
TOL = {0: 1e-5, 1: 5e-5, 2: 5e-5, 3: 5e-5}

SHAPES = [
    (128, 128, 32), (128, 128, 64), (256, 384, 96), (1000, 3000, 130), (960, 100, 1000), (100, 30000, 64),
    (32, 3000, 1000), (32, 1000, 3000), (64, 1500, 500), (17, 259, 77), (200, 37, 300), (5, 129, 33), (400, 2000, 30),
]


@pytest.mark.parametrize('path', [0, 1, 2, 3])
@pytest.mark.parametrize('ta,tb', [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_shapes(path, ta, tb):
    for (M, N, K) in SHAPES:
        pad = (-(M if ta else K)) % 4 if path >= 2 else 0        # TMA path: leading dimensions multiple of 4
        if path >= 2 and ((M if ta else K) + pad) % 4 + ((K if tb else N) + pad) % 4:
            continue
        err = _run(path, M, N, K, ta, tb, seed=M + N + K, pad=pad)
        assert err < TOL[path], (path, ta, tb, M, N, K, err)


@pytest.mark.parametrize('path', [0, 1, 2, 3])
def test_gemm_epilogues(path):
    assert _run(path, 300, 260, 200, 0, 0, bias=True) < TOL[path]
    assert _run(path, 300, 260, 200, 1, 0, accumulate=True) < TOL[path]
    assert _run(path, 300, 260, 200, 0, 1, bias=True, accumulate=True, pad=4) < TOL[path]
    assert _run(path, 32, 3000, 1000, 0, 0, bias=True, pad=8) < TOL[path]           # swapped roles: bias on the 128-row side
    assert _run(path, 32, 1000, 3000, 0, 1, splitk=7) < TOL[path]
    assert _run(path, 32, 3000, 1000, 0, 0, splitk=6) < TOL[path]
    assert _run(path, 500, 700, 1000, 1, 0, splitk=3) < TOL[path]
    assert _run(path, 132, 200, 30, 1, 0, batch=5, accumulate=True) < TOL[path]
    if path < 2:
        assert _run(path, 33, 257, 65, 0, 0, pad=1) < TOL[path]                     # unaligned leading dimensions
