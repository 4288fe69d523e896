"""GPU: the 3xFP16 GEMM on 2-CTA clusters sharing the W tile (sealdec_debug_gemm_ex mode 5) is bit-identical to the
one-CTA-per-tile kernel (mode 3): the same wgmma sequence per 256-K register chunk and the same promotions, only the W
tile arrives by multicast and a stage is released to both CTAs' producers.  Checked at the benchmark's decoder,
encoder and lm_head shapes (rows reduced where the host copies would dominate), ragged M (odd and even numbers of
128-row tiles, a last cluster with an empty second CTA), ragged N and K, with and without the GELU epilogue.
tools/gemm_cluster_bench.py times the two kernels against each other on the premise this test holds."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_gemm(mode, A, W, b, gelu):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm_ex(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                    out.ctypes.data, gelu, 0, C.byref(us), -1, 1))
    return out


def inputs(M, N, K, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    return A, W, b


def same_bits(x, y):
    return np.array_equal(x.view(np.uint32), y.view(np.uint32))


SHAPES = [
    (15000, 1024, 1024, 0), (7500, 3072, 1024, 0), (7500, 4096, 1024, 1), (7500, 1024, 4096, 0),   # decoder
    (20000, 1024, 1024, 0),                                                                         # encoder
    (700, 50265, 1024, 0),                                                                          # lm_head
    (1100, 1003, 1024, 1), (1300, 1000, 512, 0), (129, 384, 128, 0), (300, 2000, 192, 1),          # ragged M / N / K
]


@pytest.mark.parametrize("M,N,K,gelu", SHAPES)
def test_cluster_gemm_bit_identical(M, N, K, gelu):
    A, W, b = inputs(M, N, K, M + N + K)
    one = run_gemm(3, A, W, b, gelu)
    pair = run_gemm(5, A, W, b, gelu)
    assert np.isfinite(one).all()
    assert same_bits(one, pair), np.abs(one - pair).max()
