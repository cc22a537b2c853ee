"""tma_gemm_kernel_ws feeds the raw fp32 word as the tf32 hi operand and its residual as the lo operand (the tensor core
reads the upper 19 bits of the word), and a K-major B box straight from the TMA stage.  Against numpy float64, through
nats_debug_gemm."""
import pytest

from tests.test_gpu_gemm import TOL, _run

pytestmark = pytest.mark.gpu

# max |err| / sqrt(K) of the unsplit 1000 x 3000 x 12768 product (seed 7) with the earlier split (hi and lo both rounded
# to tf32), measured on an H100 80GB HBM3.  The raw-word split may not make it worse by more than 10 %.  (The raw-word
# split measured 8.34e-5, 8.20e-5, 8.13e-5, 8.10e-5 on the same card.)
UNSPLIT_DEEP_ERR = {(0, 0): 8.338e-5, (0, 1): 8.048e-5, (1, 0): 7.648e-5, (1, 1): 7.981e-5}


@pytest.mark.parametrize('ta,tb', [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_ws_deep_product_unsplit(ta, tb):
    """d[U|Ux] of one encoder direction in one pass: 399 k-blocks into the same three accumulators"""
    err = _run(2, 1000, 3000, 12768, ta, tb, seed=7)
    assert err <= 1.1 * UNSPLIT_DEEP_ERR[(ta, tb)], (ta, tb, err)


def test_ws_kmajor_b_tail():
    """K-major B (the raw stage is the wgmma B_hi operand): K not a multiple of 32, so the last k-block reads past K.
    The padded leading dimensions hold random values there; only TMA's zero fill keeps them out of the sum."""
    assert _run(2, 300, 260, 45, 0, 1, pad=3) < TOL[2]                      # one partial k-block
    assert _run(2, 260, 200, 141, 0, 1, pad=3) < TOL[2]                     # four full k-blocks and a 13-deep tail
    assert _run(2, 100, 3000, 77, 0, 1, pad=3) < TOL[2]                     # swapped roles: op(A) is the K-major B side
    assert _run(2, 960, 100, 1013, 0, 1, splitk=3, pad=3) < TOL[2]          # split-K: only the last split has a tail
    assert _run(2, 300, 200, 70, 0, 1, batch=2, pad=2) < TOL[2]             # batched
    assert _run(2, 302, 200, 70, 1, 1, batch=2, pad=2) < TOL[2]             # MN-major A beside the K-major B
