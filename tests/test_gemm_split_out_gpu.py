"""GPU: the GEMM's outputs besides its fp32 C, through sealdec_debug_gemm_split, against exact references
(test_gemm_split_out_host.py; test_bf16_host.split3 for 3xBF16) on every store path of the tile epilogue and of the
split-K finish pass:

  1. the operand split of the next GEMM (3xTF32 hi / lo, 3xFP16 halves, 3xBF16 pieces) is the split of the GEMM's own
     fp32 output, bit for bit -- -0.0 from GELU and +0 from ReLU included -- with and without the fp32 C, in every mode
     and activation: full tiles (gemm_mode 5: a last cluster whose second CTA has no rows), the ragged n tile's
     single-column store, a 1 x 3 output, split-K finish passes, and a skinny fc1 (GELU, split only);
  2. the fp16 range flag at its exact threshold: with W = 2 I every output is exactly 2 a, so a = 32 752 gives 65 504
     (flag 0, split (65 504, 0)) and a = 32 752 + 2^-9 gives 65 504 + 2^-8 (flag 1, split saturated to (65 504, 0),
     fp32 C unsaturated), for one such element on a full tile (one CTA and 2-CTA clusters), on the single-column edge
     store and in the split-K finish pass; gemm_mode 2 and 6 split outputs up to ~1e30 exactly and raise nothing;
  3. split-K deferral: where all of its conditions hold, the raw slices summed in index order, times unscale, plus the
     bias, equal the finished GEMM bit for bit (the sum the consumer kernels' load_split4 / load_split2 perform);
     breaking any one condition makes the GEMM finish the sum itself.

Every case asserts the last_paths bits of the branch it is meant to take, derived from the card's SM count as
gemm.cu's split_k_slices derives the slice count; the fp32 outputs are also held to test_gemm_range_gpu.py's float64
bound (test_bf16_gpu.py's in gemm_mode 6)."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

from test_bf16_host import split3
from test_gemm_range_gpu import FLOOR, REL, ULP, gelu64
from test_gemm_split_out_host import HALF_MAX, split_half, split_tf32

pytestmark = pytest.mark.gpu

GM = GN = 128
# last_paths bits (include/sealdec.h)
DEFERRED, FINISH, FULL_TILE, CLUSTER, TF32, RELU, BF16 = 1 << 10, 1 << 11, 1 << 12, 1 << 13, 1 << 14, 1 << 19, 1 << 24
ACTS = {0: "none", 1: "gelu", 2: "relu"}


@pytest.fixture(scope="module")
def sms():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    return torch.cuda.get_device_properties(0).multi_processor_count


def k_slices(mode, M, N, K, sms):
    """split_k_slices (gemm.cu): a 3xFP16 / 3xBF16 GEMM of few tiles spreads K over up to 8 CTAs"""
    if mode == 2:
        return 1
    tiles, kblocks = -(-M // GM) * -(-N // GN), K // 64
    ks = 1
    if tiles * 2 <= sms and kblocks >= 4:
        ks = min(8, kblocks // 2, sms // tiles)
        while ks > 1 and kblocks % ks:
            ks -= 1
    return ks


def expected_paths(mode, M, N, K, act, sms, deferred=False):
    bits = (RELU if act == 2 else 0) | (BF16 if mode == 6 else 0)
    if k_slices(mode, M, N, K, sms) > 1:
        return bits | (DEFERRED if deferred else FINISH)
    if mode == 2:
        return bits | TF32
    if mode == 5 and M > GM:
        return bits | CLUSTER
    return bits | (FULL_TILE if mode in (3, 5) else 0)


def run(mode, A, W, b, act, outputs, defer_rows=0):
    from seal_b200._lib import check, lib
    M, K = A.shape
    N = W.shape[0]
    out = np.empty((M, N), np.float32)
    piece = {2: np.float32, 3: np.float16, 5: np.float16, 6: np.uint16}[mode]      # bf16 as its bits
    s = [np.empty((M, N), piece) for _ in range(3 if mode == 6 else 2)]
    slices = np.empty((8, M, N), np.float32) if defer_rows else None
    ov, ks, unscale, paths = C.c_int32(-1), C.c_int32(-1), C.c_float(0), C.c_uint32(0)
    check(lib.sealdec_debug_gemm_split(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                       act, outputs, out.ctypes.data, s[0].ctypes.data, s[1].ctypes.data,
                                       s[2].ctypes.data if mode == 6 else None, C.byref(ov), defer_rows,
                                       slices.ctypes.data if slices is not None else None, C.byref(ks), C.byref(unscale),
                                       C.byref(paths)))
    return SimpleNamespace(C=out if outputs & 1 else None, s=s if outputs & 2 else None, overflow=ov.value,
                           paths=paths.value, k_slices=ks.value, unscale=unscale.value,
                           slices=slices[:ks.value] if ks.value > 0 else None)


def split_bits(mode, c):
    """the reference split of float32 c in the mode's format, as bit patterns"""
    if mode == 2:
        return [p.view(np.uint32) for p in split_tf32(c)]
    if mode in (3, 5):
        return [p.view(np.uint16) for p in split_half(c)]
    import torch
    return [(p.numpy().view(np.uint32) >> 16).astype(np.uint16) for p in split3(torch.from_numpy(np.ascontiguousarray(c)))]


def device_bits(mode, s):
    return [p.view(np.uint32 if mode == 2 else np.uint16) for p in s]


def assert_split_of(mode, s, c, label):
    for i, (got, want) in enumerate(zip(device_bits(mode, s), split_bits(mode, c))):
        bad = np.argwhere(got != want)
        assert bad.size == 0, f"{label}: piece {i + 1}: {len(bad)} elements differ, first at {tuple(bad[0])} " \
                              f"(C = {c[tuple(bad[0])]!r}, bits {got[tuple(bad[0])]:#x}, want {want[tuple(bad[0])]:#x})"


def bf16_exact(x):
    """x rounded to bf16 values, so that every mode (gemm_mode 6 rounds W to bf16) multiplies the same matrix"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def inputs(M, N, K, seed, bias=True):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = bf16_exact(rng.standard_normal((N, K)) / np.sqrt(K))
    b = rng.standard_normal(N).astype(np.float32)
    b[::7] -= 40.0              # columns far below zero: GELU gives -0.0 there, ReLU +0
    return A, W, (b if bias else None)


def assert_within_float64(mode, A, W, b, act, got, label):
    """got against float64 within test_gemm_range_gpu.py's per-element bound (test_bf16_gpu.py's in gemm_mode 6)"""
    A64, W64 = A.astype(np.float64), W.astype(np.float64)
    pre = A64 @ W64.T + (b.astype(np.float64) if b is not None else 0.0)
    mag = np.abs(A64) @ np.abs(W64).T
    if mode == 6:
        tol = (48 + A.shape[1] // 256 + 8) * 2.0 ** -23 * mag + 2.0 ** -23 * np.abs(pre)
    else:
        tol = REL * mag + ULP * np.abs(pre) + (FLOOR * np.abs(W64).sum(1)[None, :] if mode != 2 else 0.0)
    exp = pre
    if act == 1:
        exp = gelu64(pre)
        tol = 1.2 * tol + ULP * (np.abs(pre) + np.abs(exp))
    elif act == 2:
        exp = np.maximum(pre, 0.0)
    err = np.abs(got.astype(np.float64) - exp)
    assert np.isfinite(got).all(), label
    worst = np.unravel_index(np.argmax(err / tol), err.shape)
    assert (err <= tol).all(), (label, worst, err[worst], tol[worst])


# ---- 1. the split outputs ----------------------------------------------------------------------------------------------

# K < 256 never splits K: 300 x 1024 x 192 whole tiles (gemm_mode 5: the last cluster's second CTA has no rows),
# 1300 x 1157 x 128 a ragged n tile ending in a single-column store (column 1156), 1 x 3 x 64 one pair and one single
# column; 129 x 129 x 512 and 64 x 1024 x 4096 split K (4 and 8 slices on 132 SMs); 150 x 4096 x 1024 is fc1 of a
# 150-row decoder query slice, which writes only the split (2 slices on 132 SMs, whole tiles on fewer than 128).
SPLIT_SHAPES = [(300, 1024, 192), (1300, 1157, 128), (1, 3, 64), (129, 129, 512), (64, 1024, 4096)]
SPLIT_CASES = [(mode, act, shape) for shape in SPLIT_SHAPES for act in ACTS for mode in (2, 3, 5, 6)]
SPLIT_CASES += [(mode, 1, (150, 4096, 1024)) for mode in (2, 3, 5, 6)]


@pytest.mark.parametrize("mode,act,shape", SPLIT_CASES,
                         ids=[f"mode{m}-{ACTS[a]}-{s[0]}x{s[1]}x{s[2]}" for m, a, s in SPLIT_CASES])
def test_split_is_the_split_of_the_fp32_output(mode, act, shape, sms):
    M, N, K = shape
    A, W, b = inputs(M, N, K, M + N + K)
    label = f"mode {mode} {ACTS[act]} {M}x{N}x{K}"
    want_paths = expected_paths(mode, M, N, K, act, sms)
    both = run(mode, A, W, b, act, 3)
    assert both.paths == want_paths, (label, hex(both.paths), hex(want_paths))
    assert both.overflow == 0 and both.k_slices == 0
    assert_within_float64(mode, A, W, b, act, both.C, label)
    assert_split_of(mode, both.s, both.C, label)
    only = run(mode, A, W, b, act, 2)
    assert only.paths == want_paths, (label, hex(only.paths), hex(want_paths))
    assert_split_of(mode, only.s, both.C, label + " split only")
    if act == 1:
        assert (np.signbit(both.C) & (both.C == 0)).any(), "no -0.0 from GELU: the bias no longer reaches it"
    if act == 2:
        assert (both.C == 0).any() and (both.C >= 0).all()


# ---- 2. the fp16 range flag ---------------------------------------------------------------------------------------------

IN_RANGE = np.float32(32752.0)                 # 2 a = 65 504, fp16's largest value
PAST_RANGE = np.float32(32752.001953125)       # 2 a = 65 504 + 2^-8: the smallest fp32 output past it


def two_eye(N, K):
    W = np.zeros((N, K), np.float32)
    n = min(N, K)
    W[np.arange(n), np.arange(n)] = 2.0
    return W


def eye_inputs(M, K, seed):
    """values on a 2^-6 grid below 16: exact in every mode's operand split, so that C = 2 A exactly"""
    rng = np.random.default_rng(seed)
    return (rng.integers(-1000, 1001, size=(M, K)) / 64.0).astype(np.float32)


def doubled(A, N):
    want = np.zeros((A.shape[0], N), np.float32)
    n = min(N, A.shape[1])
    want[:, :n] = 2.0 * A[:, :n]
    return want


# (label, M, N, K, row, col): n tile 0 of a one-tile-wide GEMM (gemm_mode 5: row 200 is the second CTA of the first
# cluster); column 128 of N = 129, the single-column store of the ragged n tile; the split-K finish pass (2 slices)
FLAG_CASES = [("full_tile", 300, 128, 128, 200, 77), ("edge_column", 300, 129, 192, 5, 128),
              ("splitk_finish", 129, 256, 256, 128, 255)]


@pytest.mark.parametrize("sign", [1.0, -1.0], ids=["pos", "neg"])
@pytest.mark.parametrize("label,M,N,K,row,col", FLAG_CASES, ids=[c[0] for c in FLAG_CASES])
@pytest.mark.parametrize("mode", [3, 5])
def test_fp16_overflow_flag_at_the_threshold(mode, label, M, N, K, row, col, sign, sms):
    W = two_eye(N, K)
    want_paths = expected_paths(mode, M, N, K, 0, sms)
    assert bool(want_paths & FINISH) == (label == "splitk_finish")
    for a, flag in ((IN_RANGE, 0), (PAST_RANGE, 1)):
        A = eye_inputs(M, K, M + N + K)
        A[row, col] = np.float32(sign) * a
        want = doubled(A, N)
        assert float(want[row, col]) == sign * 2.0 * float(a)
        tag = f"mode {mode} {label} a = {sign * float(a)!r}"
        for outputs in (3, 2):
            r = run(mode, A, W, None, 0, outputs)
            assert r.paths == want_paths, (tag, hex(r.paths), hex(want_paths))
            assert r.overflow == flag, (tag, outputs)
            if outputs & 1:
                assert np.array_equal(r.C.view(np.uint32), want.view(np.uint32)), tag
            assert_split_of(mode, r.s, want, tag)
            h1, h2 = r.s[0][row, col], r.s[1][row, col]
            assert h1 == np.float16(sign * HALF_MAX) and h2 == 0, (tag, h1, h2)


# outputs past the fp16 range, up to ~1e30, and a few small ones, on bf16 values (exact in every mode's split)
BIG = np.array([1.5 * 2.0 ** 98, -1.25 * 2.0 ** 60, 66048.0, -40960.0, 98304.0, 3.0 * 2.0 ** -40], np.float32)


@pytest.mark.parametrize("label,M,N,K,row,col", FLAG_CASES, ids=[c[0] for c in FLAG_CASES])
@pytest.mark.parametrize("mode", [2, 6])
def test_wide_range_modes_split_exactly_without_a_flag(mode, label, M, N, K, row, col, sms):
    W = two_eye(N, K)
    A = eye_inputs(M, K, M + N + K)
    A[row, col - len(BIG) + 1:col + 1] = BIG
    A[:M // 2, 0] = BIG[0]
    r = run(mode, A, W, None, 0, 3)
    assert r.paths == expected_paths(mode, M, N, K, 0, sms), hex(r.paths)
    assert r.overflow == 0
    want = doubled(A, N)
    assert np.array_equal(r.C.view(np.uint32), want.view(np.uint32))
    assert_split_of(mode, r.s, want, f"mode {mode} {label}")
    if mode == 2:
        total = r.s[0].astype(np.float64) + r.s[1].astype(np.float64)
    else:
        total = sum((p.astype(np.uint32) << 16).view(np.float32).astype(np.float64) for p in r.s)
    assert np.array_equal(total, want.astype(np.float64))


# ---- 3. split-K deferral ------------------------------------------------------------------------------------------------

# 129 x 1024 x 1024: 16 tiles, K split over 8 CTAs on 132 SMs
DM, DN, DK = 129, 1024, 1024


@pytest.mark.parametrize("mode", [3, 5, 6])
def test_deferred_slices_sum_to_the_finished_output(mode, sms):
    A, W, b = inputs(DM, DN, DK, mode)
    ks = k_slices(mode, DM, DN, DK, sms)
    assert ks > 1
    d = run(mode, A, W, b, 0, 1, defer_rows=DM)
    assert d.paths == expected_paths(mode, DM, DN, DK, 0, sms, deferred=True), hex(d.paths)
    assert d.k_slices == ks
    assert np.isnan(d.C).all()                                 # left for the consumer: nothing wrote C
    assert d.unscale > 0 and np.frexp(np.float32(d.unscale))[0] == 0.5     # a power of two: no FMA can round differently
    f = run(mode, A, W, b, 0, 1, defer_rows=0)
    assert f.paths == expected_paths(mode, DM, DN, DK, 0, sms), hex(f.paths)
    acc = d.slices[0].copy()
    for part in d.slices[1:]:
        acc += part                                            # float32, in index order
    summed = acc * np.float32(d.unscale) + b
    bad = np.argwhere(summed.view(np.uint32) != f.C.view(np.uint32))
    assert bad.size == 0, f"{len(bad)} elements differ, first at {tuple(bad[0])}"
    assert_within_float64(mode, A, W, b, 0, f.C, f"mode {mode} finished")


# each breaks one condition of the deferral, from (no activation, fp32 C only, a bias, N = ldc, M <= defer_rows)
BREAKS = {"gelu": dict(act=1), "relu": dict(act=2), "split_out": dict(outputs=3), "no_bias": dict(bias=False),
          "ldc": dict(N=1022), "rows": dict(defer_rows=DM - 1)}


@pytest.mark.parametrize("broken", list(BREAKS))
@pytest.mark.parametrize("mode", [3, 5, 6])
def test_deferral_needs_every_condition(mode, broken, sms):
    cfg = dict(act=0, outputs=1, bias=True, N=DN, defer_rows=DM)
    cfg.update(BREAKS[broken])
    N, act = cfg["N"], cfg["act"]
    A, W, b = inputs(DM, N, DK, mode + 7, bias=cfg["bias"])
    assert k_slices(mode, DM, N, DK, sms) > 1
    r = run(mode, A, W, b, act, cfg["outputs"], defer_rows=cfg["defer_rows"])
    assert r.paths & FINISH and not r.paths & DEFERRED, hex(r.paths)
    assert r.paths == expected_paths(mode, DM, N, DK, act, sms), hex(r.paths)
    assert r.k_slices == 0
    assert_within_float64(mode, A, W, b, act, r.C, f"mode {mode} {broken}")
    if r.s is not None:
        assert_split_of(mode, r.s, r.C, f"mode {mode} {broken}")
