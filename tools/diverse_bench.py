"""Diverse beam groups on the benchmark workload: bench.py's corpus (10 M-token index), queries and BART-large at beam 15,
body n-grams of 10, for Q in {20, 1 000}, groups G in {1, 3, 5} and penalty in {0, 0.5} (G = 1 has no penalty).

Per configuration: ms per generate (CUDA events around `--steps` calls on the decode stream, after `--warmup` calls;
at Q = 20 these replay the call's CUDA graph), the phase split of one more, eager call (sealdec_last_phase_us) and the
kernel launches per generate.  The GPU's name and power limit, and the median SM clock during the timed calls, are
read in the same run.  One JSON line per configuration on stdout.

    python tools/diverse_bench.py [--steps 5] [--warmup 2] [--queries 20,1000]
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


def gpu_info(index):
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, power, smax = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "sm_max_clock": smax}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--queries", default="20,1000")
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
    qs = [int(x) for x in args.queries.split(",")]
    docs, ids_all, mask_all = build_inputs(max(qs), seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    eng = SealBartEngine.from_hf(make_model(), device=0)
    info = gpu_info(0)
    print(json.dumps({"setup": info, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup}), flush=True)
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM, forced_bos_token_id=None)
    H = (MAX_LEN - 1) * 2 * BEAM + BEAM
    stream = torch.cuda.Stream(device=dev)
    for Q in qs:
        ids_np = np.ascontiguousarray(ids_all[:Q]); mask_np = np.ascontiguousarray(mask_all[:Q])
        ids = torch.from_numpy(ids_np).to(dev); mask = torch.from_numpy(mask_np).to(dev)
        rec = DeviceRecords(RecordLayout(Q, H, MAX_LEN), dev)
        src_tokens = int(mask_np.sum())
        for G, pen in ((1, 0.0), (3, 0.0), (3, 0.5), (5, 0.0), (5, 0.5)):
            call = lambda: generate_records_device(eng, index, ids, mask, out=rec, src_tokens=src_tokens, stream=stream,
                                                   num_beam_groups=G, diversity_penalty=pen, **kw)
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
            launches = eng.last_launch_count()
            errs = rec.host()["errors"]
            lib.sealbart_set_option(eng._h, b"cuda_graph", 0)          # phase events need an eager call
            call()
            torch.cuda.synchronize()
            phases = eng.last_phase_us()
            lib.sealbart_set_option(eng._h, b"cuda_graph", -1)
            print(json.dumps({"queries": Q, "groups": G, "penalty": pen, "ms_per_generate": ms, "cuda_graph": graph,
                              "last_launch_count": launches, "eager_launch_count": eng.last_launch_count(),
                              "last_phase_us": phases, "sm_clock_mhz": clocks["sm_mhz"], "clock_reasons": clocks["reasons"],
                              "error_flags": errs.tolist(), **info}), flush=True)


if __name__ == "__main__":
    main()
