"""Where a GEMM CTA's time goes at the tile boundaries, from the per-unit timeline of CTA 0 (sealdec_debug_gemm_trace +
sealdec_debug_gemm_units) at the shapes bench.py runs (1 000 queries x beam 15 on bart-large: 15 000 rows, and the
7 500-row query slices), in the default gemm_mode 3.  Per work unit the kernel stamps, on consumer warpgroup 1: its
first k-block of MMAs committed (F), its K loop done (L), epilogue start (E0) and end (E1).  Per shape this prints
  - the epilogue's share of CTA 0's traced time: sum(E1 - E0) / (E1[last] - F[0]);
  - the tensor-idle gap at tile boundaries, F[i + 1] - L[i] (this warpgroup has no MMA in flight from the end of one
    unit's K loop to the next unit's first commit: the epilogue plus the wait for the next operands), as a share and
    in microseconds per boundary;
  - the K loop's time per unit, L - F, and the launch's device time (CUDA events over --iters calls).
The lm_head runs twice: through sealdec_debug_gemm_ex without storing (the plain GEMM's tile loop) and through
sealdec_debug_head with the statistics epilogue the decoder uses (HEAD).  Card name, power limit and SM clocks are
sampled in the same run.  Needs a GPU.
--variant no-bias passes no bias to every shape; --variant no-store stores no output at any shape but the HEAD one
(whose sparse logits are its output).  Set against the default, they show what the bias loads and the stores cost.

Needs the library built with the timeline compiled in: make -C seal_b200/csrc GEMM_UNIT_TRACE=1 (after make clean).

Usage: gemm_epilogue_probe.py [--iters 5] [--variant as-is|no-bias|no-store] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from seal_b200._lib import lib, check  # noqa: E402
from head_bench import Sampler  # noqa: E402

D, F, V = 1024, 4096, 50265
UNITS = 256                                # per-unit stamps the kernel keeps (kTraceUnits, wgmma_gemm.cuh)
SHAPES = ([("qkv", m, 3 * D, D, 0) for m in (15000, 7500)] + [("o/cq", m, D, D, 0) for m in (15000, 7500)]
          + [("fc1+gelu", m, F, D, 1) for m in (15000, 7500)] + [("fc2", m, D, F, 0) for m in (15000, 7500)]
          + [("lm_head", 15000, V, D, 0), ("lm_head HEAD", 15000, V, D, 0)])


def traced(call):
    """runs call() with tracing on; returns (20 CTA stamps, [n][4] unit stamps of the last traced launch)"""
    check(lib.sealdec_debug_gemm_units((C.c_int64 * (4 * UNITS))(), 4 * UNITS))       # clear
    check(lib.sealdec_debug_gemm_trace(1, None))
    call()
    t20 = (C.c_int64 * 20)()
    check(lib.sealdec_debug_gemm_trace(0, t20))
    u = (C.c_int64 * (4 * UNITS))()
    check(lib.sealdec_debug_gemm_units(u, 4 * UNITS))
    u = np.array(list(u), dtype=np.int64).reshape(UNITS, 4)
    n = int(np.argmax(u[:, 3] == 0)) if (u[:, 3] == 0).any() else UNITS
    return list(t20), u[:n]


def summarize(t20, u):
    ghz = (t20[6] - t20[0]) / (t20[8] - t20[7]) if t20[8] > t20[7] else 1.98
    us = lambda c: float(c) / ghz / 1e3                                                 # noqa: E731
    span = u[-1, 3] - u[0, 0]
    epi = u[:, 3] - u[:, 2]
    kloop = u[:, 1] - u[:, 0]
    gap = u[1:, 0] - u[:-1, 1]
    return {"units": int(len(u)), "ghz": ghz, "span_us": us(span), "epilogue_share": float(epi.sum() / span),
            "epilogue_us": us(np.median(epi)), "gap_share": float(gap.sum() / span) if len(gap) else 0.0,
            "gap_us": us(np.median(gap)) if len(gap) else 0.0, "kloop_us": us(np.median(kloop))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--variant", default="as-is", choices=["as-is", "no-bias", "no-store"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    rows = []
    with Sampler() as smp:
        for name, M, N, K, gelu in SHAPES:
            A = rng.standard_normal((M, K), dtype=np.float32)
            W = (rng.standard_normal((N, K), dtype=np.float32) * 0.05).astype(np.float32)
            b = rng.standard_normal(N, dtype=np.float32)
            bp = None if args.variant == "no-bias" else b.ctypes.data
            dev_us = C.c_double(0)
            if name == "lm_head HEAD":
                words = (N + 31) // 32
                mask = np.zeros((M, words), dtype=np.uint32)
                mask[np.arange(M)[:, None], rng.integers(0, words, size=(M, 4))] = 1 << 7   # a few allowed tokens per row
                mpad = -(-M // 128) * 128
                out = np.empty((mpad, N), dtype=np.float32)
                stats = np.empty((mpad, -(-N // 128), 2), dtype=np.float32)
                fused = C.c_int32(0)
                call = lambda: check(lib.sealdec_debug_head(M, N, K, A.ctypes.data, W.ctypes.data, bp,  # noqa: E731
                                                            mask.ctypes.data, 2, 1, out.ctypes.data, stats.ctypes.data,
                                                            C.byref(fused)))
                call()
                assert fused.value == 1, "the lm_head took the split-K path"
            else:
                store = 0 if name == "lm_head" or args.variant == "no-store" else 1
                out = np.empty((M, N), dtype=np.float32) if store else None
                call = lambda: check(lib.sealdec_debug_gemm_ex(3, M, N, K, A.ctypes.data, W.ctypes.data, bp,  # noqa: E731
                                                               out.ctypes.data if store else None, gelu, args.iters,
                                                               C.byref(dev_us), -1, store))
                call()                                                                   # warm-up
            t20, u = traced(call)
            r = {"shape": name, "M": M, "N": N, "K": K, "device_us": dev_us.value or None, **summarize(t20, u)}
            rows.append(r)
            del A, W, out
    card = smp.summary()
    print(f"variant {args.variant}: {card['gpu']}, power limit {card['power_limit_w']} W, median SM clock {card['sm_mhz_median']} MHz")
    print(f"{'shape':13s} {'M':>6s} {'N':>6s} {'K':>5s} {'units':>5s} {'call ms':>8s} {'K loop us':>9s} {'epi us':>7s} "
          f"{'epi %':>6s} {'gap us':>7s} {'gap %':>6s}")
    for r in rows:
        ms = f"{r['device_us'] / 1e3:8.3f}" if r["device_us"] else f"{'-':>8s}"
        print(f"{r['shape']:13s} {r['M']:6d} {r['N']:6d} {r['K']:5d} {r['units']:5d} {ms} {r['kloop_us']:9.2f} "
              f"{r['epilogue_us']:7.2f} {r['epilogue_share'] * 100:5.1f}% {r['gap_us']:7.2f} {r['gap_share'] * 100:5.1f}%")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "variant": args.variant, "iters": args.iters, "rows": rows}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
