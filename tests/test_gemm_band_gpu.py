"""GPU: the banded tile order of weight-dominated GEMMs (the lm_head at thousands of rows) changes only which CTA
computes which tile and when, so its output must be bit-identical to the plain m-fastest order."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run(A, W, b, band):
    from seal_b200._lib import lib, check
    M, K = A.shape
    N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm_ex(3, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, out.ctypes.data, 0, 0,
                                    C.byref(us), band, 1))
    return out


# (M, N, K, band): the lm_head at 1 000 queries x 15 beams with the band gemm_impl picks (-1: 16 tiles at K = 1 024),
# forced bands with a ragged last band and a ragged last tile, one band wider than the problem, and a small M where
# gemm_impl uses no bands
CASES = [(15000, 50265, 1024, -1), (2000, 3003, 1024, 3), (1100, 4097, 256, 4), (640, 2048, 512, 100),
         (700, 50265, 1024, -1)]


@pytest.mark.parametrize("M,N,K,band", CASES)
def test_banded_order_is_bit_identical(M, N, K, band):
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((M, K), dtype=np.float32)
    W = (rng.standard_normal((N, K), dtype=np.float32) * 0.05).astype(np.float32)
    b = rng.standard_normal(N, dtype=np.float32)
    ref = run(A, W, b, 0)
    got = run(A, W, b, band)
    assert np.isfinite(ref).all()
    assert np.array_equal(ref.view(np.uint32), got.view(np.uint32))
