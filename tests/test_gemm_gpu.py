"""GPU: the GEMM back-ends of the BART path -- 3xFP16 (one CTA per tile, 2-CTA clusters) and the 3xTF32 range-safe
fallback, all wgmma -- against a float64 reference of the same op (C = A W^T + b, optional exact GELU): they must stay within a
few fp32 ulps of it (that is what the 1e-4 beam-score parity rests on)."""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_gemm(mode, A, W, b, gelu, iters=0):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                 out.ctypes.data, int(gelu), iters, C.byref(us)))
    return out, us.value


def ref_gemm(A, W, b, gelu):
    y = A.astype(np.float64) @ W.astype(np.float64).T
    if b is not None:
        y = y + b.astype(np.float64)
    if gelu:
        from math import erf
        y = 0.5 * y * (1.0 + np.vectorize(erf)(y / math.sqrt(2.0)))
    return y


SHAPES = [(5, 128, 128, False), (77, 384, 128, False), (300, 1024, 1024, False), (129, 4096, 1024, True),
          (513, 1024, 4096, False), (200, 1003, 1024, False), (6, 50265, 1024, False)]


# gemm_mode 5 (2-CTA clusters sharing the W tile) takes over once a problem fills the machine; these shapes do (odd
# and even numbers of 128-row tiles, ragged N, K = 4096, GELU epilogue), the small SHAPES run its split-K fallback
SHAPES_PAIR = [(2600, 1024, 1024, False), (1300, 4096, 1024, True), (2400, 1003, 4096, False), (700, 50265, 1024, False),
               (1024, 3072, 1024, False)]


@pytest.mark.parametrize("M,N,K,gelu", SHAPES_PAIR + SHAPES[:4])
def test_gemm_cta_pair_matches_float64(M, N, K, gelu):
    test_gemm_matches_float64(5, M, N, K, gelu)


@pytest.mark.parametrize("mode", [2, 3])
@pytest.mark.parametrize("M,N,K,gelu", SHAPES)
def test_gemm_matches_float64(mode, M, N, K, gelu):
    rng = np.random.default_rng(M * 7 + N)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    got, _ = run_gemm(mode, A, W, b, gelu)
    exp = ref_gemm(A, W, b, gelu)
    scale = np.abs(exp).max()
    err = np.abs(got - exp).max()
    print(f"mode {mode} {M}x{N}x{K} gelu={gelu}: max abs err {err:.3e} (scale {scale:.2f})")
    assert np.isfinite(got).all()
    assert err <= 3e-6 * max(scale, 1.0) * math.sqrt(K / 128.0), (mode, err)


def test_gemm_throughput_report():
    """Not an assertion on speed — records achieved TFLOP/s of both back-ends at the decode shapes."""
    rng = np.random.default_rng(0)
    for (M, N, K) in [(15000, 4096, 1024), (15000, 1024, 4096), (15000, 3072, 1024), (3000, 50265, 1024)]:
        A = rng.standard_normal((M, K)).astype(np.float32); W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
        b = np.zeros(N, dtype=np.float32)
        for mode in (2, 3, 5):
            _, us = run_gemm(mode, A, W, b, False, iters=5)
            print(f"GEMM {M}x{N}x{K} mode {mode}: {us:.1f} us, {2.0 * M * N * K / us / 1e6:.1f} TFLOP/s (fp32-equivalent)")


def test_gemm_small_m_report():
    """Latency of the small-problem path (batch 20 x beam 15 = 300 decoder rows; 125 queries per GPU under strong
    scaling = 1 875 rows): split-K over up to 8 CTAs per 128 x 256 tile + finish pass (a record, not an assertion)."""
    rng = np.random.default_rng(0)
    for (M, N, K) in [(300, 3072, 1024), (300, 1024, 1024), (300, 4096, 1024), (300, 1024, 4096), (1875, 1024, 1024), (1875, 1024, 4096)]:
        A = rng.standard_normal((M, K)).astype(np.float32); W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
        b = np.zeros(N, dtype=np.float32)
        _, us = run_gemm(5, A, W, b, False, iters=50)
        print(f"GEMM {M}x{N}x{K} mode 5: {us:.1f} us per call (launches back to back)")
