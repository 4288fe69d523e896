"""CPU: the exact references of the GEMM's split outputs (operand_split.cuh) that test_gemm_split_out_gpu.py compares the
device with bit for bit, and the C signature of the hook it calls.

  - split_half (3xFP16, gemm_mode 3 / 5, split_value for __half): saturate to +-65 504, h1 = rn_half(x), h2 = rn_half(x - h1), numpy's
    round-to-nearest-even conversion.  h1 + h2 == x wherever the pair can hold x: |x| in [2^-14, 65 504] with at most
    22 significant bits on fp16's 2^-24 grid; elsewhere within the documented error max(2^-23 |x|, 2^-25).  Past the
    range the pair is (+-65 504, 0).
  - split_tf32 (3xTF32, gemm_mode 2, split_value for float): hi = x with the 13 low mantissa bits cleared, lo = x - hi; hi + lo == x for every
    finite x.
  - 3xBF16 (gemm_mode 6) uses test_bf16_host.split3, whose exactness that module tests.
  - the ctypes signature of sealdec_debug_gemm_split (seal_b200/_lib.py) matches include/sealdec.h argument by
    argument."""
import ctypes as C
import os
import re

import numpy as np

HALF_MAX = 65504.0


def split_half(x):
    """(h1, h2) float16 arrays of the fp16 split_value (operand_split.cuh) for float32 x"""
    x = np.clip(np.asarray(x, dtype=np.float32), -HALF_MAX, HALF_MAX)
    h1 = x.astype(np.float16)
    return h1, (x - h1.astype(np.float32)).astype(np.float16)


def split_tf32(x):
    """(hi, lo) float32 arrays of the TF32 split_value (operand_split.cuh) for float32 x"""
    x = np.asarray(x, dtype=np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, x - hi


def random_fp32(rng, n, lo_exp, hi_exp):
    """n float32 values with uniform exponents in [lo_exp, hi_exp], random mantissas and signs"""
    e = rng.integers(lo_exp, hi_exp + 1, size=n)
    m = rng.integers(0, 1 << 23, size=n, dtype=np.int64)
    bits = ((e + 127).astype(np.int64) << 23) | m | (rng.integers(0, 2, size=n, dtype=np.int64) << 31)
    return bits.astype(np.uint32).view(np.float32)


def half_sum(x):
    h1, h2 = split_half(x)
    return h1.astype(np.float64) + h2.astype(np.float64)


def test_half_split_is_exact_where_the_pair_holds_x():
    rng = np.random.default_rng(0)
    x = random_fp32(rng, 2_000_000, -14, 15)
    x = x[np.abs(x) <= HALF_MAX]
    # keep 22 significant bits and fp16's subnormal grid: the low half then has at most 11 bits on that grid
    e = np.floor(np.log2(np.abs(x.astype(np.float64))))
    unit = np.maximum(np.exp2(e - 21), 2.0 ** -24)
    x22 = (np.round(x.astype(np.float64) / unit) * unit).astype(np.float32)
    x22 = x22[np.abs(x22) <= HALF_MAX]
    ext = np.array([HALF_MAX, -HALF_MAX, 2.0 ** -14, -(2.0 ** -14), 1.0, 1.0 + 2.0 ** -21, 2.0 ** 15 - 2.0 ** -6,
                    2.0 ** -3 + 2.0 ** -24, 0.0, -0.0], dtype=np.float32)
    for v in (x22, ext):
        assert np.array_equal(half_sum(v), v.astype(np.float64))
    # every other fp32 value of the range: the split's documented error, and not always exact
    err = np.abs(half_sum(x) - x.astype(np.float64))
    assert (err <= np.maximum(2.0 ** -23 * np.abs(x.astype(np.float64)), 2.0 ** -25)).all()
    assert (err > 0).any()


def test_half_split_saturates():
    x = np.array([65504.00390625, 65519.99609375, 65520.0, 1e6, 3.4e38, np.inf], dtype=np.float32)
    for sign in (1.0, -1.0):
        h1, h2 = split_half(sign * x)
        assert (h1 == sign * HALF_MAX).all() and (h2 == 0).all()
        assert (np.signbit(h1) == (sign < 0)).all()
    # at the boundary nothing saturates: 65 504 is fp16's largest value, 65 503.99 rounds up to it
    h1, h2 = split_half(np.array([HALF_MAX, np.nextafter(np.float32(HALF_MAX), np.float32(0))], dtype=np.float32))
    assert (h1 == HALF_MAX).all() and h2[0] == 0 and h2[1] == np.float16(-2.0 ** -8)


def test_tf32_split_is_exact_for_every_finite_value():
    rng = np.random.default_rng(1)
    bits = rng.integers(0, 1 << 32, size=4_000_000, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    x = x[np.isfinite(x)]
    ext = np.array([np.finfo(np.float32).max, -np.finfo(np.float32).max, np.finfo(np.float32).smallest_subnormal,
                    np.finfo(np.float32).tiny, 1.0 + 2.0 ** -23, 0.0, -0.0], dtype=np.float32)
    for v in (x, ext):
        hi, lo = split_tf32(v)
        assert not (hi.view(np.uint32) & 0x1FFF).any()
        assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), v.astype(np.float64))


def header_args(name):
    """the parameter declarations of `name` in include/sealdec.h"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "sealdec.h")).read()
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


def test_split_hook_signature_matches_the_header():
    from seal_b200._lib import lib
    decl = header_args("sealdec_debug_gemm_split")
    types = lib.sealdec_debug_gemm_split.argtypes
    assert len(types) == len(decl), (len(types), decl)
    for d, t in zip(decl, types):
        if "*" in d:
            assert t is C.c_void_p or issubclass(t, C._Pointer), (d, t)
        elif d.startswith("int64_t"):
            assert t is C.c_int64, (d, t)
        else:
            assert d.split()[0] in ("int", "int32_t") and t is C.c_int32, (d, t)
