"""Small-M GEMM latency probe: average launch time (CUDA events, hot loop) and the in-kernel timeline of
CTA 0 (sealdec_debug_gemm_trace).  Usage: gemm_trace_probe.py M N K [iters]"""
import ctypes as C, sys, os
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from seal_b200._lib import lib, check
M, N, K = (int(x) for x in sys.argv[1:4])
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 50
rng = np.random.default_rng(0)
A = rng.standard_normal((M, K)).astype(np.float32); W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
b = np.zeros(N, dtype=np.float32); out = np.empty((M, N), dtype=np.float32); us = C.c_double(0)
check(lib.sealdec_debug_gemm_trace(1, None))
check(lib.sealdec_debug_gemm(3, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, out.ctypes.data, 0, iters, C.byref(us)))
t = (C.c_int64 * 20)()
check(lib.sealdec_debug_gemm_trace(0, t))
t = list(t)
cyc = t[6] - t[0]; ns = t[8] - t[7]
f = cyc / ns if ns > 0 else 1.9                      # cycles per ns
names = ["prologue", "first operands", "MMA issue", "last chunk done", "tile stored", "exit"]
d = [(t[i + 1] - t[i]) / f / 1000 for i in range(6)]
print(f"{M}x{N}x{K}: {us.value:.2f} us/launch(+finish); CTA0 total {ns/1000:.2f} us @ {f:.2f} GHz: "
      + ", ".join(f"{n} {x:.2f}" for n, x in zip(names, d)))
sub = [t[4]] + t[9:17]
print("   epilogue passes (staged, stored) us:", " ".join(f"{(sub[i + 1] - sub[i]) / f / 1000:.2f}" for i in range(8)))
