"""GPU: the GEMM back-ends against float64 element by element, over the range of activation magnitudes.

test_gemm_gpu.py bounds the error by one scale for the whole output, which leaves rows of small magnitude unchecked.
Here every element j of row i is held to the standard dot-product bound
    |C - C64| <= REL * sum_k |a_ik w_jk| + ULP * |C64|                      (3xTF32, gemm_mode 2)
plus, for the 3xFP16 modes 3 / 5, an absolute floor
    + FLOOR * sum_k |w_jk|
because activations enter the fp16 split unscaled (operand_split.cuh, split_value): the low half h2 = rn_half(x - h1)
has |x - h1| <= 2^-11 |x|, so below |x| ~ 2^-3 it is an fp16 subnormal with an absolute spacing of 2^-24 (below 2^-14
h1 is too), each such activation carries an error of up to 2^-25 whatever its size, and values below 2^-25 flush to
zero.  Standard-normal rows have entries on both sides of 2^-3; rows scaled by 2^-6 and less sit entirely below it.
Activations of magnitude >= 2^-3 are held to the bound without the floor in every mode."""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
REL = 2.0 ** -18          # 64 u: the split drops terms of ~2^-22 relative; the rest is fp32 accumulation (chunks of 48)
ULP = 2.0 ** -22          # the epilogue's scale-and-bias rounding
FLOOR = 2.0 ** -24        # twice the 2^-25 worst activation error of the fp16 split
ROW_SCALES = [1.0, 2.0 ** -6, 2.0 ** -12, 2.0 ** -20, 2.0 ** -30]


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


def run_gemm(mode, A, W, b, act):
    """act: 0 none, 1 GELU, 2 ReLU"""
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                 out.ctypes.data, act, 0, C.byref(us)))
    return out


def gelu64(x):
    from scipy.special import erf
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def make_a(kind, M, K, rng):
    if kind == "scaled":      # row i scaled by ROW_SCALES[i % 5] (M = 1: 2^-12)
        scale = np.array([ROW_SCALES[i % 5] if M > 1 else 2.0 ** -12 for i in range(M)])
        return (rng.standard_normal((M, K)) * scale[:, None]).astype(np.float32)
    # a GELU output, as fc2 sees it: many small negative entries, a few large positive ones
    return gelu64(rng.standard_normal((M, K)) * 3.0).astype(np.float32)


def check_elementwise(mode, A, W, b, act, label, floor_ok=True):
    got = run_gemm(mode, A, W, b, act)
    A64, W64 = A.astype(np.float64), W.astype(np.float64)
    pre = A64 @ W64.T + (b.astype(np.float64) if b is not None else 0.0)
    mag = np.abs(A64) @ np.abs(W64).T
    tol = REL * mag + ULP * np.abs(pre)
    floor = FLOOR * np.abs(W64).sum(1)[None, :] * np.ones_like(pre)
    if mode != 2 and floor_ok:
        tol = tol + floor
    exp = pre
    if act == 1:          # |gelu'| <= 1.13; erff's own error is relative to |x| where 1 + erf cancels
        exp = gelu64(pre)
        tol = 1.2 * tol + ULP * (np.abs(pre) + np.abs(exp))
    elif act == 2:        # |relu(x) - relu(y)| <= |x - y|: the same bound
        exp = np.maximum(pre, 0.0)
    assert np.isfinite(got).all(), label
    err = np.abs(got - exp)
    worst = np.unravel_index(np.argmax(err / tol), err.shape)
    no_floor = REL * mag + ULP * np.abs(pre)
    print(f"{label}: worst err/bound {(err / tol).max():.3f} at {tuple(int(i) for i in worst)} (|err| {err[worst]:.2e}); "
          f"max err / (u sum|a||w|) {(err / (U * np.maximum(mag, 1e-300))).max():.3g}; "
          f"worst err / bound without the floor {(err / no_floor).max():.3g}")
    assert (err <= tol).all(), (label, worst, err[worst], tol[worst])


@pytest.mark.parametrize("act", [0, 2], ids=["none", "relu"])
@pytest.mark.parametrize("mode", [2, 3, 5])
@pytest.mark.parametrize("kind", ["scaled", "gelu_rows"])
@pytest.mark.parametrize("M", [1, 129])
@pytest.mark.parametrize("N", [1, 3, 129])
@pytest.mark.parametrize("K", [64, 320])        # one k-block; five, the last promotion chunk partly filled
def test_gemm_per_element_vs_float64(mode, kind, M, N, K, act):
    rng = np.random.default_rng(M * 1000 + N * 10 + K)
    A = make_a(kind, M, K, rng)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) if N != 3 else None
    check_elementwise(mode, A, W, b, act, f"mode {mode} {kind} {M}x{N}x{K} act={act}")


@pytest.mark.parametrize("mode", [3, 5])
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "gelu", "relu"])
@pytest.mark.parametrize("K", [512, 2048])
def test_gemm_split_k_per_element_vs_float64(mode, act, K):
    """129 x 129: four tiles, so K is split over 4 (K = 512) or 8 (K = 2048) CTAs and summed by the finish pass"""
    rng = np.random.default_rng(K + act)
    for kind in ("scaled", "gelu_rows"):
        A = make_a(kind, 129, K, rng)
        W = (rng.standard_normal((129, K)) * 0.05).astype(np.float32)
        b = rng.standard_normal(129).astype(np.float32) if kind == "scaled" else None
        check_elementwise(mode, A, W, b, act, f"mode {mode} split-K {kind} 129x129x{K} act={act}")


@pytest.mark.parametrize("mode", [2, 3, 5])
@pytest.mark.parametrize("M,N,K", [(1, 129, 64), (129, 129, 320), (129, 129, 2048)])
def test_gemm_fp32_level_above_fp16_floor(mode, M, N, K):
    """every activation of magnitude in [2^-3, 4): both fp16 halves are normal, no floor term is needed"""
    rng = np.random.default_rng(M + N + K + mode)
    A = (np.exp2(rng.uniform(-3.0, 2.0, size=(M, K))) * rng.choice([-1.0, 1.0], size=(M, K))).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    check_elementwise(mode, A, W, b, 0, f"mode {mode} |a| in [2^-3, 4) {M}x{N}x{K}", floor_ok=False)


@pytest.mark.parametrize("mode", [3, 5])
def test_fp16_modes_reject_k_not_multiple_of_64(mode):
    from seal_b200._lib import SealB200Error
    A = np.ones((4, 96), dtype=np.float32); W = np.ones((8, 96), dtype=np.float32)
    with pytest.raises(SealB200Error) as ei:
        run_gemm(mode, A, W, None, 0)
    assert ei.value.code == -1
    run_gemm(2, A, W, None, 0)                # 3xTF32 takes K in steps of 32
