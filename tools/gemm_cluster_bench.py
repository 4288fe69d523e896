"""The 3xFP16 GEMM at the shapes bench.py runs (1 000 queries x beam 15 on bart-large): the one-CTA-per-tile kernel
(sealdec_debug_gemm_ex mode 3, the default gemm_mode) against the 2-CTA cluster kernel that shares the W tile (mode 5),
alternating the two in one process.  Per shape it prints the device time (CUDA events), the
fp32-equivalent FLOP/s (2 M N K), and the operand bytes each kernel moves from L2 into shared memory per second
(tiles x k-blocks x stage bytes: 64 KB per 64-K block for a one-CTA tile, 96 KB for a cluster's two tiles, which
share 32 KB of W), with the card's name, power limit and SM clocks sampled in the same run.  Outputs of the two
kernels are compared bit for bit at every shape but the lm_head (whose fp32 logits would take 3 GB of host memory
twice; tests/test_gemm_cluster_gpu.py compares it at fewer rows).  Both kernels take the tile order gemm_impl picks
for their mode: the lm_head's L2 bands exist only in mode 3, so its mode-5 time includes re-reading A from HBM once per
n column.  Needs a GPU.

Usage: gemm_cluster_bench.py [--iters 20] [--reps 3] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from seal_b200._lib import lib, check  # noqa: E402
from head_bench import Sampler  # noqa: E402

GM = GN = 128
KB = 64                                  # K per 64-K block: 128 B of fp16 per row
ONE_CTA_STAGE = 4 * GM * KB * 2          # A h1 / h2 and W h1 / h2 of one tile
PAIR_STAGE = 2 * (2 * GM * KB * 2) + 2 * GN * KB * 2   # A halves of both tiles, W halves once

D, F, V = 1024, 4096, 50265
DECODER = [(n, k) for n, k in ((3 * D, D), (D, D), (F, D), (D, F))]
SHAPES = ([("decoder", m, n, k) for m in (15000, 7500) for n, k in DECODER]
          + [("lm_head", 15000, V, D)]
          + [("encoder", 20000, n, k) for n, k in DECODER])


def gemm(mode, A, W, b, store, iters):
    M, K = A.shape
    N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32) if store else None
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm_ex(mode, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data,
                                    out.ctypes.data if store else None, 0, iters, C.byref(us), -1, store))
    return out, us.value


def l2_bytes(mode, M, N, K):
    m_tiles, n_tiles, kb = -(-M // GM), -(-N // GN), K // KB
    if mode == 3:
        return m_tiles * n_tiles * kb * ONE_CTA_STAGE
    return -(-m_tiles // 2) * n_tiles * kb * PAIR_STAGE


def card_limits():
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm,clocks_event_reasons.sw_power_cap",
                        "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True).stdout.strip()
    parts = [x.strip() for x in q.split(",")]
    return {"sm_mhz_max": parts[0] if parts else None, "sw_power_cap_now": parts[1] if len(parts) > 1 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3, help="alternating repetitions of both kernels per shape")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    rows, all_identical = [], True
    with Sampler() as smp:
        for name, M, N, K in SHAPES:
            A = rng.standard_normal((M, K), dtype=np.float32)
            W = (rng.standard_normal((N, K), dtype=np.float32) * 0.05).astype(np.float32)
            b = rng.standard_normal(N, dtype=np.float32)
            store = 0 if name == "lm_head" else 1
            identical = None
            if store:
                ref, _ = gemm(3, A, W, b, 1, 0)
                got, _ = gemm(5, A, W, b, 1, 0)
                identical = bool(np.array_equal(ref.view(np.uint32), got.view(np.uint32)))
                all_identical &= identical
                del ref, got
            t = {3: [], 5: []}
            gemm(3, A, W, b, store, 2); gemm(5, A, W, b, store, 2)       # warm-up
            for _ in range(args.reps):
                for mode in (3, 5):
                    t[mode].append(gemm(mode, A, W, b, store, args.iters)[1])
            rows.append({"shape": name, "M": M, "N": N, "K": K, "store": store, "bit_identical": identical,
                         "us_one_cta": t[3], "us_cluster": t[5],
                         "l2_bytes_one_cta": l2_bytes(3, M, N, K), "l2_bytes_cluster": l2_bytes(5, M, N, K)})
    card = smp.summary()
    card.update(card_limits())
    print(f"{card['gpu']}, power limit {card['power_limit_w']} W, median SM clock {card['sm_mhz_median']} of "
          f"{card['sm_mhz_max']} MHz, median draw {card['power_draw_w_median']} W ({card['samples']} samples), "
          f"sw_power_cap at the end: {card['sw_power_cap_now']}")
    print(f"{args.iters} calls per timing, {args.reps} alternating repetitions; one-CTA = mode 3, cluster = mode 5")
    print(f"{'shape':8s} {'M':>6s} {'N':>6s} {'K':>5s} {'one-CTA ms':>11s} {'cluster ms':>11s} {'gain':>6s} {'spread':>7s} "
          f"{'TFLOP/s':>15s} {'L2->SM TB/s':>13s} {'bits':>5s}")
    for r in rows:
        a, c = float(np.median(r["us_one_cta"])), float(np.median(r["us_cluster"]))
        spread = max((max(v) - min(v)) / np.median(v) for v in (r["us_one_cta"], r["us_cluster"]))
        fl = 2.0 * r["M"] * r["N"] * r["K"]
        r.update(median_ms_one_cta=a / 1e3, median_ms_cluster=c / 1e3)
        same = "-" if r["bit_identical"] is None else ("same" if r["bit_identical"] else "DIFF")
        print(f"{r['shape']:8s} {r['M']:6d} {r['N']:6d} {r['K']:5d} {a / 1e3:11.3f} {c / 1e3:11.3f} "
              f"{(a - c) / a * 100:5.1f}% {spread * 100:6.1f}% {fl / a / 1e6:7.1f}/{fl / c / 1e6:7.1f} "
              f"{r['l2_bytes_one_cta'] / a / 1e6:6.2f}/{r['l2_bytes_cluster'] / c / 1e6:6.2f} {same:>5s}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "iters": args.iters, "reps": args.reps, "rows": rows}, f, indent=1)
    return 0 if all_identical else 1


if __name__ == "__main__":
    sys.exit(main())
