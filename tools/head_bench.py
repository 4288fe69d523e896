"""lm_head cost at the benchmarked shape (1 000 queries x beam 15 = 15 000 rows, bart-large: K = 1 024, V = 50 265):
the 3xFP16 GEMM in each tile order, with and without the dense fp32 logits store, and the per-row statistics /
top-2*beam kernel (topk_rows_kernel<256, 4096>) that streams those logits back.  Prints, per variant, the device time
(CUDA events, after a warm-up) next to the HBM bytes that the tile order implies, computed from the shapes, and the
card's name, power limit and median SM clock sampled during the run.  Needs a GPU.

Usage: head_bench.py [--rows 15000] [--iters 30] [--reps 3] [--out FILE.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from seal_b200._lib import lib, check  # noqa: E402

GM = GN = 128
L2_BAND_BYTES = 8 << 20           # gemm_impl: bands of m tiles whose A halves take <= 8 MB


class Sampler:
    """nvidia-smi (name, power limit, SM clock, power draw) every 100 ms while the variants run."""

    def __init__(self):
        self.rows, self.proc = [], None

    def __enter__(self):
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,power.draw",
                                      "--format=csv,noheader,nounits", "-lms", "100", "-i", "0"],
                                     stdout=subprocess.PIPE, text=True)
        threading.Thread(target=lambda: [self.rows.append([x.strip() for x in ln.split(",")]) for ln in self.proc.stdout],
                         daemon=True).start()
        return self

    def __exit__(self, *exc):
        self.proc.terminate()
        self.proc.wait()

    def summary(self):
        ok = [r for r in self.rows if len(r) == 4]
        num = lambda i: [float(r[i]) for r in ok if r[i].replace(".", "").isdigit()]   # noqa: E731
        sm, lim, pw = num(2), num(1), num(3)
        return {"gpu": ok[0][0] if ok else None, "power_limit_w": max(lim) if lim else None,
                "sm_mhz_median": float(np.median(sm)) if sm else None,
                "power_draw_w_median": float(np.median(pw)) if pw else None, "samples": len(ok)}


def gemm(A, W, b, band, store, iters):
    M, K = A.shape
    N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32) if store else None
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm_ex(3, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data,
                                    out.ctypes.data if store else None, 0, iters, C.byref(us), band, store))
    return out, us.value


def head_bytes(M, N, K, band, store):
    """HBM bytes of one lm_head call when A is larger than the L2: A and W halves (4 B per element) as often as the
    tile order re-reads them from HBM (m fastest over all rows: A once per n column, W once; bands: A once, W once per
    band), the bias, and the fp32 logits if stored."""
    m_tiles, n_tiles = -(-M // GM), -(-N // GN)
    a, w = M * K * 4, N * K * 4
    traffic = a * n_tiles + w if band <= 0 or band >= m_tiles else a + w * -(-m_tiles // band)
    return traffic + N * 4 + (M * ((N + 3) // 4 * 4) * 4 if store else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=15000)
    ap.add_argument("--vocab", type=int, default=50265)
    ap.add_argument("--d-model", type=int, default=1024)
    ap.add_argument("--beams", type=int, default=15)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3, help="alternating repetitions of every variant")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    M, N, K = args.rows, args.vocab, args.d_model
    rng = np.random.default_rng(0)
    A = rng.standard_normal((M, K), dtype=np.float32)
    W = (rng.standard_normal((N, K), dtype=np.float32) * 0.05).astype(np.float32)
    b = rng.standard_normal(N, dtype=np.float32)
    m_tiles = -(-M // GM)
    auto = max(1, L2_BAND_BYTES // (GM * K * 4)) if M * K * 4 > L2_BAND_BYTES else 0
    variants = [("current order (m fastest), dense store", 0, 1),
                (f"banded ({auto} m tiles, decoder default), dense store", -1, 1),
                ("current order, no store", 0, 0),
                (f"banded ({auto} m tiles), no store", -1, 0)]
    for bsz in (8, 16, 32, 64):
        if bsz != auto and bsz < m_tiles:
            variants.append((f"banded ({bsz} m tiles), dense store", bsz, 1))
    times = {v[0]: [] for v in variants}
    times["topk_rows_kernel<256, 4096>"] = []
    with Sampler() as smp:
        ref, _ = gemm(A, W, b, 0, 1, 0)
        got, _ = gemm(A, W, b, -1, 1, 0)
        identical = bool(np.array_equal(ref.view(np.uint32), got.view(np.uint32)))
        del ref, got
        for _ in range(args.reps):
            for name, band, store in variants:
                times[name].append(gemm(A, W, b, band, store, args.iters)[1])
            us = C.c_double(0)
            check(lib.sealdec_debug_topk_rows(M, N, args.beams, 8, args.iters, C.byref(us)))
            times["topk_rows_kernel<256, 4096>"].append(us.value)
    card = smp.summary()
    ld = (N + 3) // 4 * 4
    rows = []
    for name, band, store in variants:
        eff = (auto if band < 0 else band)
        rows.append({"variant": name, "us": times[name], "bytes": head_bytes(M, N, K, eff, store), "flop": 2.0 * M * N * K})
    rows.append({"variant": "topk_rows_kernel<256, 4096>", "us": times["topk_rows_kernel<256, 4096>"],
                 "bytes": M * ld * 4 + M * ((N + 31) // 32) * 4, "flop": 0.0})
    print(f"{card['gpu']}, power limit {card['power_limit_w']} W, median SM clock {card['sm_mhz_median']} MHz, "
          f"median draw {card['power_draw_w_median']} W ({card['samples']} samples)")
    print(f"M = {M}, N = {N}, K = {K}; {args.iters} calls per timing, {args.reps} alternating repetitions; "
          f"banded logits bit-identical to the current order: {identical}")
    print(f"{'variant':58s} {'median us':>10s} {'min..max us':>18s} {'HBM GB':>8s} {'GB/s':>7s} {'TFLOP/s':>8s}")
    for r in rows:
        med = float(np.median(r["us"]))
        fl = r["flop"] / med / 1e6
        print(f"{r['variant']:58s} {med:10.1f} {min(r['us']):8.1f}..{max(r['us']):8.1f} {r['bytes'] / 1e9:8.2f} "
              f"{r['bytes'] / med / 1e3:7.0f} {fl:8.1f}")
    print("the statistics epilogue (HeadEpi) needs a decode step's masks: bench.py's phases_us_last_step times it")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "shape": [M, N, K], "bit_identical": identical, "rows": rows}, f, indent=1)
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())
