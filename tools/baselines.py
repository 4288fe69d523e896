"""The reference-side baselines SURVEY.md section 8(d) plans, measured on the GPU box beside our path:

 1. FM-index micro-baseline: the decode's own trace (LF triples, per-step beam ranges) replayed through the compiled,
    unmodified reference (oracle/_ref: seal/cpp_modules/fm_index.cpp + sdsl-lite) -- backward_search_step on one
    thread, distinct_count_multi on all host cores (one std::async per range, fm_index.cpp:111-131), for the build with
    the reference's flags (-O3 -DNDEBUG, SWAR popcount) and the -msse4.2 -mpopcnt build; our kernels on the same trace.
 2. End-to-end baseline at the reference's operating point (README.md:76-83: batch 20, beam 15): the reference
    algorithm (oracle decode loop: per-step .tolist(), from-scratch get_range, per-row masks) with eager fp32 HF BART
    ON THE SAME GPU (KV cache, like the reference) + sdsl on the host cores; our path at the same batch size.

    python tools/baselines.py [--queries 1000] [--e2e-batches 5] [--out baselines.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--e2e-batches", type=int, default=5)
    ap.add_argument("--out", default="baselines.json")
    args = ap.parse_args()
    from bench import build_inputs, make_model, decode_trace, BEAM, MIN_LEN, MAX_LEN, LP
    from oracle.decode_oracle import fm_index_generate_oracle
    from oracle.fm_oracle import OracleIndex, RefFM, ref_available
    from seal_b200.beam_search import SealBartEngine, generate_records, fm_index_generate
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import corpus_symbols
    # the oracle loop does its score arithmetic with torch on the host: one thread per hardware thread is far too many for
    # it (128 threads: 6.6 s per batch of 20; 16 threads: 0.5 s) -- same calibration as bench.py's baseline leg
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {"cpu_count": os.cpu_count(), "torch_threads": torch.get_num_threads()}
    docs, ids, mask = build_inputs(args.queries, 4321)
    sym = corpus_symbols(docs)
    index = FMIndex(); RawFM.initialize(index, sym)
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1])); index._sync_beginnings(); index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    model = make_model()
    eng = SealBartEngine.from_hf(model, device=0)
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM)
    rec = generate_records(eng, index, ids, mask, forced_bos_token_id=None, **kw)

    # ---- the decode's trace ----------------------------------------------------------------------------------------
    s_np, l_np, h_np = decode_trace(rec)
    # ranges the reference expands: the beams entering each step = first BEAM non-EOS candidates of the previous step
    K = 2 * BEAM
    lows, highs = [], []
    for st in range(MAX_LEN - 2):
        for q in range(args.queries):
            nb = 0
            for k in range(K):
                h = st * K + k
                if rec["tokens"][q, h, st + 1] != 2 and nb < BEAM:
                    nb += 1
                    if rec["valid"][q, h] == 1:
                        lows.append(int(rec["lo"][q, h])); highs.append(int(rec["hi"][q, h]))
    lows = np.asarray(lows, dtype=np.uint64); highs = np.asarray(highs, dtype=np.uint64)
    out["trace"] = {"lf_triples": int(len(s_np)), "expand_ranges": int(len(lows)), "mean_range_width": float((highs - lows).mean())}

    # ---- ours on the trace -----------------------------------------------------------------------------------------
    dev = torch.device("cuda", 0)
    ts, tl, th = (torch.from_numpy(a).to(dev) for a in (s_np, l_np, h_np))
    def ctime(fn, iters=20):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters): fn()
        b.record(); torch.cuda.synchronize()
        return a.elapsed_time(b) / iters * 1e-3
    t_lf = ctime(lambda: index.lf_step_tensors(ts, tl, th))
    tlo = torch.from_numpy(lows.astype(np.int64)).to(dev); thi = torch.from_numpy(highs.astype(np.int64)).to(dev)
    m_out = index.expand_mask_tensors(tlo, thi, 50265)
    t_ex = ctime(lambda: index.expand_mask_tensors(tlo, thi, 50265, out=m_out), iters=10)
    out["ours"] = {"lf_steps_per_s": len(s_np) / t_lf, "lf_us": t_lf * 1e6, "expand_ranges_per_s": len(lows) / t_ex, "expand_us": t_ex * 1e6}

    # ---- the reference's FM-index on the trace ---------------------------------------------------------------------
    if ref_available():
        path = "/tmp/baseline_ref.fmi"
        t0 = time.perf_counter(); ref = RefFM(sym); out["ref_build_s"] = time.perf_counter() - t0
        ref.save(path)
        for name, fm in (("O3_swar", ref), ("O3_popcnt", RefFM(path=path, popcnt=True) if ref_available(popcnt=True) else None)):
            if fm is None:
                continue
            n1 = min(len(s_np), 200_000)
            t0 = time.perf_counter(); a, b = fm.backward_search_step_batch(s_np[:n1].astype(np.uint64), l_np[:n1].astype(np.uint64), h_np[:n1].astype(np.uint64)); t1 = time.perf_counter() - t0
            n2 = min(len(lows), 30_000)
            t0 = time.perf_counter(); fm.distinct_count_multi(lows[:n2], highs[:n2], want_output=False); t2 = time.perf_counter() - t0
            out[f"reference_{name}"] = {"lf_steps_per_s_1thread": n1 / t1, "lf_sample": n1, "expand_ranges_per_s_all_cores_async": n2 / t2,
                                       "expand_sample": n2, "cores": os.cpu_count()}
        ora = OracleIndex(_raw=ref)
        ora.beginnings = list(index.beginnings)
        ora.occurring_distinct, ora.occurring_counts = ora.get_distinct_count(0, len(ora))
        # ---- end to end at batch 20 ------------------------------------------------------------------------------
        model_gpu = model.to("cuda")
        ids_t = torch.from_numpy(ids); mask_t = torch.from_numpy(mask)
        nb = args.e2e_batches
        fm_index_generate_oracle(model_gpu, ora, ids_t[:20].cuda(), mask_t[:20].cuda(), use_cache=True, **kw)      # warm-up
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for b in range(nb):
            fm_index_generate_oracle(model_gpu, ora, ids_t[20 * b:20 * b + 20].cuda(), mask_t[20 * b:20 * b + 20].cuda(), use_cache=True, **kw)
        torch.cuda.synchronize(); t_ref = time.perf_counter() - t0
        out["e2e_batch20_reference_algorithm_eager_gpu_bart"] = {"queries_per_s": 20 * nb / t_ref, "ms_per_batch": t_ref / nb * 1e3,
                                                                 "what": "oracle decode loop (seal/beam_search.py restated) + HF BART eager fp32 with KV cache on this GPU + sdsl-lite on host cores"}
        del model_gpu
    for b in range(3):
        fm_index_generate(eng, index, ids[:20], mask[:20], keep_history=True, **kw)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    nb = max(args.e2e_batches, 20)
    for b in range(nb):
        o = (20 * b) % (args.queries - 20)
        fm_index_generate(eng, index, ids[o:o + 20], mask[o:o + 20], keep_history=True, **kw)
    torch.cuda.synchronize(); t_ours = time.perf_counter() - t0
    out["e2e_batch20_ours"] = {"queries_per_s": 20 * nb / t_ours, "ms_per_batch": t_ours / nb * 1e3,
                               "what": "seal_b200.fm_index_generate (host arrays in, python list of hypotheses out)"}
    # single-call latency of the drop-in API (seal/retrieval.py:91 filters keys with one get_count per key)
    keys = [docs[i % len(docs), 3:3 + 1 + i % 4].tolist() for i in range(2000)]
    for k in keys[:50]:
        index.get_count(k)
    t0 = time.perf_counter()
    for k in keys:
        index.get_count(k)
    out["get_count_us_per_call"] = (time.perf_counter() - t0) / len(keys) * 1e6
    t0 = time.perf_counter()
    lo_b, hi_b = index.get_range_batch(keys)
    out["get_range_batch_us_per_key"] = (time.perf_counter() - t0) / len(keys) * 1e6
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
