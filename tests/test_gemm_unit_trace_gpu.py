"""The GEMM's per-unit timeline (sealdec_debug_gemm_units, include/sealdec.h), which tools/gemm_epilogue_probe.py reads;
it is compiled in only by `make GEMM_UNIT_TRACE=1`, so the GPU test skips on a default build:
  - CPU: arguments outside the record are SEALFM_EINVAL before any device work;
  - GPU: in every gemm_mode the stamps of CTA 0 come in program order per work unit (first MMAs committed, K loop
    done, epilogue start, epilogue end, then the next unit's first MMAs), one stamped unit per unit the CTA owns, and
    tracing leaves the output bit-identical."""
import ctypes as C

import numpy as np
import pytest

EINVAL = -1
UNITS = 256


def test_units_arguments_checked():
    from seal_b200._lib import lib
    buf = (C.c_int64 * 8)()
    assert lib.sealdec_debug_gemm_units(None, 8) == EINVAL
    assert lib.sealdec_debug_gemm_units(buf, -1) == EINVAL
    assert lib.sealdec_debug_gemm_units(buf, 4 * UNITS + 1) == EINVAL


def run_gemm(mode, A, W, b, gelu):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    check(lib.sealdec_debug_gemm(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, out.ctypes.data, gelu, 0,
                                 C.byref(C.c_double(0))))
    return out


def units():
    from seal_b200._lib import lib, check
    u = (C.c_int64 * (4 * UNITS))()
    check(lib.sealdec_debug_gemm_units(u, 4 * UNITS))
    return np.array(list(u), dtype=np.int64).reshape(UNITS, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 3, 5, 6])
@pytest.mark.parametrize("M,N,K,gelu", [(1500, 1024, 1024, 0), (1300, 4096, 1024, 1), (1000, 384, 4096, 0)])
def test_unit_stamps_ordered_and_output_unchanged(mode, M, N, K, gelu):
    from seal_b200._lib import lib, check
    if lib.sealdec_debug_gemm_units((C.c_int64 * 1)(), 0) != 0:
        pytest.skip("library built without GEMM_UNIT_TRACE=1")
    rng = np.random.default_rng(M + N + K + mode)
    A = rng.standard_normal((M, K)).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    units()                                                     # clears the record
    ref = run_gemm(mode, A, W, b, gelu)
    assert not units().any(), "stamps written with tracing off"
    check(lib.sealdec_debug_gemm_trace(1, None))
    try:
        got = run_gemm(mode, A, W, b, gelu)
    finally:
        check(lib.sealdec_debug_gemm_trace(0, None))
    assert np.array_equal(ref.view(np.uint32), got.view(np.uint32))
    u = units()
    n = int((u[:, 3] != 0).sum())
    assert n >= 1 and (u[n:] == 0).all() and (u[:n] != 0).all()
    flat = u[:n].reshape(-1)
    assert (np.diff(flat) >= 0).all(), "stamps out of program order"
    assert (u[:n, 1] > u[:n, 0]).all()
