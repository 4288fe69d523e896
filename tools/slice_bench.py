"""Query slices at bench.py's workload (1 000 queries, beam 15, bart-large, the synthetic 10 M-token index): one
generate with the batch run whole and one with it run as two query slices on two streams (include/sealdec.h,
"query_slices"), alternating in one process.  Prints ms per generate for each (device events around every call, after
a warm-up), whether the records of the two are bit-identical, and the card's name, power limit and median SM clock
sampled during the timings.  --profile DIR also traces one generate of each with torch.profiler and reports how much
of the add+LN / cross-attention kernel time of one slice runs while a GEMM of the other is on the GPU.  Needs a GPU.

Usage: slice_bench.py [--queries 1000] [--reps 3] [--profile DIR]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from head_bench import Sampler  # noqa: E402

SIDE_KERNELS = ("add_ln_kernel", "cross_attn_small_kernel", "dec_self_attn")


def overlap_report(trace_events):
    """Per side-kernel family: total time, and the part of it during which a wgmma_gemm_x3_kernel of ANOTHER stream
    runs."""
    ev = [e for e in trace_events if e.get("cat") == "kernel" and "dur" in e]
    gemms = {}
    for e in ev:
        if "wgmma_gemm_x3_kernel" in e["name"]:
            gemms.setdefault(e.get("tid"), []).append((e["ts"], e["ts"] + e["dur"]))
    out = {}
    for fam in SIDE_KERNELS:
        tot = ovl = 0.0
        for e in ev:
            if fam not in e["name"]:
                continue
            a, b = e["ts"], e["ts"] + e["dur"]
            tot += b - a
            cover = []
            for tid, iv in gemms.items():
                if tid == e.get("tid"):
                    continue
                cover += [(max(a, x), min(b, y)) for x, y in iv if x < b and y > a]
            cover.sort()
            end = a
            for x, y in cover:                      # union of the covering intervals
                if y > end:
                    ovl += y - max(x, end)
                    end = y
        out[fam] = {"us": tot, "us_beside_other_gemm": ovl}
    out["wgmma_gemm_x3_kernel_us"] = sum(y - x for iv in gemms.values() for x, y in iv)
    out["streams_with_gemms"] = len(gemms)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3, help="timings of each setting, alternating")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", metavar="DIR", default=None)
    args = ap.parse_args()

    import torch
    import bench
    from seal_b200._lib import lib, check
    from seal_b200.beam_search import SealBartEngine, DeviceRecords, generate_records_device
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.sharding import RecordLayout
    from seal_b200.synthetic import corpus_symbols

    dev = torch.device("cuda", 0)
    docs, ids_np, mask_np = bench.build_inputs(args.queries, seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    eng = SealBartEngine.from_hf(bench.make_model(), device=0)
    kw = dict(min_length=bench.MIN_LEN, max_length=bench.MAX_LEN, length_penalty=bench.LP, num_beams=bench.BEAM,
              forced_bos_token_id=None)
    H = (bench.MAX_LEN - 1) * 2 * bench.BEAM + bench.BEAM
    recs = {s: DeviceRecords(RecordLayout(args.queries, H, bench.MAX_LEN), dev) for s in (0, 1)}
    ids = torch.from_numpy(ids_np).to(dev); mask = torch.from_numpy(mask_np).to(dev)
    src_tokens = int(mask_np.sum())
    stream = torch.cuda.Stream(device=dev)

    def generate(slices):
        check(lib.sealbart_set_option(eng._h, b"query_slices", slices))
        with torch.cuda.stream(stream):
            generate_records_device(eng, index, ids, mask, out=recs[slices], src_tokens=src_tokens, stream=stream, **kw)
        paths = int(lib.sealbart_get_stat(eng._h, b"last_paths"))
        assert bool(paths & (1 << 15)) == bool(slices), (slices, hex(paths))

    def timed(slices):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        generate(slices)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(args.warmup):
        for s in (0, 1):
            generate(s)
    torch.cuda.synchronize()
    times = {0: [], 1: []}
    with Sampler() as smp:
        for _ in range(args.reps):
            for s in (0, 1):
                times[s].append(timed(s))
    card = smp.summary()
    a, b = recs[0].host(), recs[1].host()
    identical = all(a[k].tobytes() == b[k].tobytes() for k in ("scores", "lens", "tokens", "valid", "lo", "hi", "errors"))
    res = {"card": card, "queries": args.queries, "beam": bench.BEAM,
           "ms_per_generate": {"whole": times[0], "two_slices": times[1]}, "records_bit_identical": identical}
    print(f"{card['gpu']}, power limit {card['power_limit_w']} W, median SM clock {card['sm_mhz_median']} MHz, "
          f"median draw {card['power_draw_w_median']} W ({card['samples']} samples)")
    for s, name in ((0, "whole batch"), (1, "two query slices")):
        print(f"{name:18s} ms per generate: median {np.median(times[s]):8.2f}   all {', '.join(f'{t:.2f}' for t in times[s])}")
    print(f"records bit-identical: {identical}")

    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        os.makedirs(args.profile, exist_ok=True)
        res["profile"] = {}
        for s in (0, 1):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                generate(s)
                torch.cuda.synchronize()
            path = os.path.join(args.profile, f"slices{s}.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                rep = overlap_report(json.load(f)["traceEvents"])
            res["profile"]["two_slices" if s else "whole"] = rep
            print(("two query slices" if s else "whole batch") + ": " + json.dumps(rep))
        with open(os.path.join(args.profile, "slice_bench.json"), "w") as f:
            json.dump(res, f, indent=1)
    check(lib.sealbart_set_option(eng._h, b"query_slices", -1))
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())
