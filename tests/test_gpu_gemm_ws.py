"""The persistent warp-specialized 3xTF32 kernel (tma_gemm_kernel_ws: every TMA-eligible product whose N side of the tile is
wider than 64) against numpy float64, through nats_debug_gemm."""
import ctypes

import numpy as np
import pytest

from tests.test_gpu_gemm import TOL, _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('ta,tb', [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_ws_tails_and_tile_counts(ta, tb):
    for (M, N, K) in [
        (300, 260, 200),       # 9 tiles: fewer than the SMs
        (1000, 3000, 132),     # 192 tiles: not a multiple of 132, every CTA strides over a second tile or not
        (260, 132, 40),        # M and N 4 past a tile; K: two k-blocks, fewer than the raw stages
        (200, 100, 76),        # K not a multiple of 32; the N side of 100 is still wider than 64
        (12800, 100, 100),     # tall: 100 tiles in one column
    ]:
        err = _run(2, M, N, K, ta, tb, seed=M + N + K)
        assert err < TOL[2], (ta, tb, M, N, K, err)


@pytest.mark.parametrize('ta,tb', [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_ws_deep_product(ta, tb):
    """the encoder weight gradient's shape: 1000 x 3000, K = 12768, in three K splits.  Unsplit, the 12768-deep tensor-core
    accumulation sits at ~8e-5 of sqrt(K) for this kernel and for the 128 x 64 one it replaces alike (same sums)."""
    err = _run(2, 1000, 3000, 12768, ta, tb, seed=7, splitk=3)
    assert err < TOL[2], (ta, tb, err)


def test_ws_epilogues():
    assert _run(2, 300, 260, 200, 0, 0, bias=True) < TOL[2]
    assert _run(2, 100, 3000, 200, 0, 0, bias=True, pad=4) < TOL[2]                  # swapped roles: bias on the 128-row side
    assert _run(2, 100, 3000, 200, 1, 1, accumulate=True) < TOL[2]                   # swapped roles: column-stride output
    assert _run(2, 300, 200, 96, 1, 0, batch=3, accumulate=True) < TOL[2]
    assert _run(2, 300, 200, 72, 0, 1, batch=4, bias=True) < TOL[2]
    assert _run(2, 500, 700, 1000, 1, 0, splitk=3) < TOL[2]
    assert _run(2, 960, 100, 3000, 0, 1, splitk=5) < TOL[2]
    assert _run(2, 200, 300, 64, 0, 0, splitk=4) < TOL[2]                            # splits 2 and 3 have no k-block


def test_ws_deterministic():
    import torch
    from nats_b200 import nats, _lib
    eng = nats.get_engine()
    M, N, K = 1000, 3000, 2000
    g = torch.Generator().manual_seed(3)
    A = torch.randn(K, M, generator=g).to(eng.device)          # transA: stored [K, M]
    B = torch.randn(K, N, generator=g).to(eng.device)
    outs = []
    for _ in range(2):
        C = torch.zeros(M, N, device=eng.device)
        rc = eng.lib.nats_debug_gemm(eng.ctx, eng.stream(), 2, 1, 0, M, N, K, ctypes.c_void_p(A.data_ptr()), M,
                                     ctypes.c_void_p(B.data_ptr()), N, ctypes.c_void_p(C.data_ptr()), N, ctypes.c_void_p(0),
                                     0, 1, 1, 0, 0, 0)
        _lib.check(rc, 'nats_debug_gemm')
        torch.cuda.synchronize()
        outs.append(C.cpu().numpy())
    np.testing.assert_array_equal(outs[0], outs[1])
