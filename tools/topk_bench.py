"""The top-k logits warp (fm_index_generate's topk) on the benchmark workload: bench.py's corpus (10 M-token index),
queries and BART-large at beam 15, body n-grams of 10, with top_k in {0, 10, 100, 1000}.

* Per (queries, top_k): ms per generate (CUDA events around `--steps` calls on the decode stream, after `--warmup`
  calls), the phase split of one more, eager call (sealdec_last_phase_us), the kernel launches and the number of decode
  steps whose lm_head used the statistics epilogue (a top-k step needs every logit, so it stores them densely).
* The threshold kernel alone (topk_threshold_kernel through sealdec_debug_topk_threshold) on R rows of V = 50 265
  random fp32 logits: its device time from torch.profiler (CUDA activities; the host-to-device copy of the hook is
  not counted) and the achieved bytes/s of its one read of V * 4 bytes per row, against the 3.35 TB/s of the H100 SXM
  data sheet.
The GPU's name and power limit, and the median SM clock during the timed calls, are read in the same run.  One JSON
line per configuration on stdout.

    python tools/topk_bench.py [--steps 5] [--warmup 2] [--queries 20,1000] [--topk 0,10,100,1000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BEAM, LP, MAX_LEN, MIN_LEN, ClockSampler, build_inputs, make_model  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, power, smax = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_max_clock": smax}


def threshold_kernel_time(rows, V, k, reps):
    """mean device time of topk_threshold_kernel over `reps` hook calls, from the profiler's kernel records"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from seal_b200._lib import check, lib
    rng = np.random.default_rng(0)
    X = np.ascontiguousarray((rng.standard_normal((rows, V)) * 3.0).astype(np.float32))
    thr = np.empty(rows, np.float32); mx = np.empty(rows, np.float32); ls = np.empty(rows, np.float32)
    call = lambda: check(lib.sealdec_debug_topk_threshold(rows, V, V, X.ctypes.data, k, thr.ctypes.data, mx.ctypes.data,
                                                          ls.ctypes.data))
    call()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "topk_threshold_kernel" in e.name]
    assert len(times) == reps, (len(times), reps)
    us = float(np.mean(times))
    return us, rows * V * 4 / (us * 1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--queries", default="20,1000")
    ap.add_argument("--topk", default="0,10,100,1000")
    args = ap.parse_args()
    import torch
    from seal_b200._lib import lib
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
    print(json.dumps({"setup": info, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup}), flush=True)
    for rows in (300, 15000):
        for k in (10, 1000):
            us, bps = threshold_kernel_time(rows, 50265, k, reps=5)
            print(json.dumps({"kernel": "topk_threshold_kernel", "rows": rows, "V": 50265, "top_k": k, "us": us,
                              "bytes_per_s": bps, "share_of_3.35TBps": bps / HBM_BYTES_PER_S, **info}), flush=True)
    docs, ids_all, mask_all = build_inputs(max(qs), seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    eng = SealBartEngine.from_hf(make_model(), device=0)
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM, forced_bos_token_id=None)
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
            graph = int(lib.sealbart_get_stat(eng._h, b"last_used_graph"))
            errs = rec.host()["errors"]
            lib.sealbart_set_option(eng._h, b"cuda_graph", 0)          # phase events need an eager call
            call()
            torch.cuda.synchronize()
            phases = eng.last_phase_us()
            fused = eng.stat("fused_head_steps")
            lib.sealbart_set_option(eng._h, b"cuda_graph", -1)
            print(json.dumps({"queries": Q, "top_k": k, "ms_per_generate": ms, "cuda_graph": graph,
                              "eager_launch_count": eng.last_launch_count(), "fused_head_steps": fused,
                              "last_phase_us": phases, "sm_clock_mhz": clocks["sm_mhz"], "clock_reasons": clocks["reasons"],
                              "error_flags": errs.tolist(), **info}), flush=True)


if __name__ == "__main__":
    main()
