"""GPU: the GEMM tile epilogue's bias, which the kernel stages per work unit in shared memory during the K loop.  The
bias is the epilogue's last addition, and the weight unscale is a power of two, so without an activation C(A, W, b)
must equal fp32(C(A, W, no bias) + b) bit for bit in every gemm_mode.  The shapes give each CTA many work units (the
one staging buffer is refilled unit after unit), a ragged last n tile (columns past N stage as 0), a single k-block
(the K loop barely outlasts the staging), ragged row tiles, and skinny M (split-K: the kernel runs without a bias and
the slices' sum adds it)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPES = [(2000, 3000, 128), (1300, 1003, 1024), (700, 50265, 64), (2600, 1024, 64), (100, 1003, 1024)]


def run_gemm(mode, A, W, b):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    check(lib.sealdec_debug_gemm(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                 out.ctypes.data, 0, 0, C.byref(C.c_double(0))))
    return out


@pytest.mark.parametrize("mode", [2, 3, 5, 6])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_bias_is_the_last_addition(mode, M, N, K):
    rng = np.random.default_rng(M + 3 * N + K + mode)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    plain = run_gemm(mode, A, W, None)
    got = run_gemm(mode, A, W, b)
    exp = plain + b                                             # float32 + float32: one rounding, as the epilogue's FMA
    assert np.isfinite(got).all()
    bad = np.flatnonzero(got.view(np.uint32) != exp.view(np.uint32))
    assert bad.size == 0, f"{bad.size} elements differ, first at {np.unravel_index(bad[0], got.shape)}"


def test_head_epilogue_matches_plain_gemm():
    """The lm_head statistics epilogue (HEAD) reads the same staged bias: every logit it stores equals the plain
    GEMM's bit for bit (all of n tile 0, the allowed tokens, eos and pad elsewhere; the rest stays poisoned), and each
    (row, n tile) maximum is that tile's maximum of the plain output.  N is ragged and each CTA runs many units."""
    from seal_b200._lib import lib, check
    M, N, K, eos, pad = 2000, 3000, 128, 2, 1
    rng = np.random.default_rng(5)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    words, n_tiles, mpad = (N + 31) // 32, (N + 127) // 128, (M + 127) // 128 * 128
    mask = np.zeros((M, words), dtype=np.uint32)
    mask[np.arange(M)[:, None], rng.integers(0, words, size=(M, 6))] = rng.integers(1, 2 ** 32, size=(M, 6), dtype=np.uint32)
    plain = run_gemm(3, A, W, b)
    out = np.empty((mpad, N), dtype=np.float32)
    stats = np.empty((mpad, n_tiles, 2), dtype=np.float32)
    fused = C.c_int32(0)
    check(lib.sealdec_debug_head(M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, mask.ctypes.data, eos, pad,
                                 out.ctypes.data, stats.ctypes.data, C.byref(fused)))
    assert fused.value == 1
    cols = np.arange(N)
    allowed = ((mask[:, cols // 32] >> (cols % 32).astype(np.uint32)) & 1).astype(bool)
    allowed[:, :128] = True
    allowed[:, [eos, pad]] = True
    got = out[:M]
    assert np.array_equal(got[allowed].view(np.uint32), plain[allowed].view(np.uint32))
    assert np.isnan(got[~allowed]).all()
    tile_max = np.stack([plain[:, t * 128:(t + 1) * 128].max(axis=1) for t in range(n_tiles)], axis=1)
    assert np.array_equal(stats[:M, :, 0], tile_max)
