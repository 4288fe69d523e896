"""The top-k logits warp at the mT5 vocabulary (V = 250 112), where each logits row's threshold runs on one cluster of
five CTAs (topk_threshold_cluster_kernel).

* The cluster kernel alone through sealdec_debug_topk_threshold_cluster on 300 and 15 000 rows of random fp32 logits
  at top_k 10 and 1 000: its device time from torch.profiler (CUDA activities; the hook's host-to-device copy is not
  counted) and the achieved bytes/s of its one read of V * 4 bytes per row, against the 3.35 TB/s of the H100 SXM data
  sheet.  The 15 000-row case needs a 15 GB host array (300 random rows repeated) and is reported as not measured when
  the host has less than 40 GB available.
* Whole generates of a random-init t5-base-shaped model (tools/t5_bench.py's shape) with the mT5 vocabulary on
  bench.py's corpus (10 M-token index) and queries, beam 15, body n-grams of 10, at top_k 0 / 10 / 100: ms per generate
  (CUDA events around `--steps` calls on the decode stream after `--warmup` calls; at Q = 20 these replay the call's
  CUDA graph, at Q = 300 they run eagerly), the phase split of one more, eager call, and the decode steps that ran the
  cluster kernel (sealbart_get_stat "topk_cluster_steps").
The GPU's name and power limit, and the median SM clock during the timed calls, are read in the same run.  One JSON
line per configuration on stdout.

    python tools/topk_large_bench.py [--steps 3] [--warmup 2] [--queries 20,300] [--topk 0,10,100]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import BEAM, LP, MAX_LEN, MIN_LEN, ClockSampler, build_inputs  # noqa: E402
from diverse_bench import gpu_info  # noqa: E402
from t5_bench import make_t5  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
V_MT5 = 250112


def host_available_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def cluster_kernel_time(rows, k, reps):
    """mean device time of topk_threshold_cluster_kernel over `reps` hook calls, from the profiler's kernel records"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from seal_b200._lib import check, lib
    rng = np.random.default_rng(0)
    base = (rng.standard_normal((min(rows, 300), V_MT5), dtype=np.float32) * 3.0).astype(np.float32)
    X = np.empty((rows, V_MT5), np.float32)
    for r0 in range(0, rows, len(base)):
        X[r0:r0 + len(base)] = base[:rows - r0]
    thr = np.empty(rows, np.float32); mx = np.empty(rows, np.float32); ls = np.empty(rows, np.float32)
    call = lambda: check(lib.sealdec_debug_topk_threshold_cluster(rows, V_MT5, V_MT5, X.ctypes.data, k, thr.ctypes.data,
                                                                  mx.ctypes.data, ls.ctypes.data))
    call()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "topk_threshold_cluster_kernel" in e.name]
    assert len(times) == reps, (len(times), reps)
    us = float(np.mean(times))
    return us, rows * V_MT5 * 4 / (us * 1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--queries", default="20,300")
    ap.add_argument("--topk", default="0,10,100")
    args = ap.parse_args()
    import torch
    from seal_b200.beam_search import DeviceRecords, SealBartEngine, generate_records_device
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.sharding import RecordLayout
    from seal_b200.synthetic import corpus_symbols

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info(0)
    qs = [int(x) for x in args.queries.split(",")]
    ks = [int(x) for x in args.topk.split(",")]
    print(json.dumps({"setup": info, "V": V_MT5, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup}), flush=True)
    for rows in (300, 15000):
        for k in (10, 1000):
            if rows * V_MT5 * 4 * 2.5 > host_available_bytes():
                print(json.dumps({"kernel": "topk_threshold_cluster_kernel", "rows": rows, "V": V_MT5, "top_k": k,
                                  "us": "not measured (host memory)", **info}), flush=True)
                continue
            us, bps = cluster_kernel_time(rows, k, reps=3)
            print(json.dumps({"kernel": "topk_threshold_cluster_kernel", "rows": rows, "V": V_MT5, "top_k": k, "us": us,
                              "bytes_per_s": bps, "share_of_3.35TBps": bps / HBM_BYTES_PER_S, **info}), flush=True)
    docs, ids_all, mask_all = build_inputs(max(qs), seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    model = make_t5("t5-base", V_MT5)
    eng = SealBartEngine.from_hf(model, device=0)
    del model
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM)
    H = (MAX_LEN - 1) * 2 * BEAM + BEAM
    stream = torch.cuda.Stream(device=dev)
    for Q in qs:
        ids_np = np.ascontiguousarray(ids_all[:Q]); mask_np = np.ascontiguousarray(mask_all[:Q])
        ids = torch.from_numpy(ids_np).to(dev); mask = torch.from_numpy(mask_np).to(dev)
        rec = DeviceRecords(RecordLayout(Q, H, MAX_LEN), dev)
        src_tokens = int(mask_np.sum())
        for k in ks:
            call = lambda: generate_records_device(eng, index, ids, mask, out=rec, src_tokens=src_tokens, stream=stream,
                                                   top_k=k, **kw)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            sampler = ClockSampler(0)
            sampler.start()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                call()
            e1.record(stream)
            torch.cuda.synchronize()
            clocks = sampler.stop()
            ms = e0.elapsed_time(e1) / args.steps
            graph = eng.stat("last_used_graph")
            errs = rec.host()["errors"]
            eng.set_option("cuda_graph", 0)                     # phase events need an eager call
            call()
            torch.cuda.synchronize()
            phases = eng.last_phase_us()
            cluster_steps = eng.stat("topk_cluster_steps")
            eng.set_option("cuda_graph", -1)
            print(json.dumps({"model": "t5-base", "V": V_MT5, "queries": Q, "top_k": k, "ms_per_generate": ms,
                              "queries_per_s": Q / (ms * 1e-3), "cuda_graph": graph, "topk_cluster_steps": cluster_steps,
                              "last_phase_us": phases, "error_flags": errs.tolist(), "sm_clock_mhz": clocks["sm_mhz"],
                              "clock_reasons": clocks["reasons"], **info}), flush=True)


if __name__ == "__main__":
    main()
