"""Evidence aggregation at SEALSearcher's defaults: the per-query aggregate_evidence loop against
batch_aggregate_evidence, on keys from real constrained decodes.

Corpus: bench.py's synthetic 100 000 x 100-token corpus (10 M tokens).  Keys: generate_records at SEALSearcher's
decode defaults (beam 15, length 10) with bench.py's BART-large model, one key per distinct decoded hypothesis
(tokens > 2, best score), plus compute_unigram_scores of the same queries.  Aggregation at SEALSearcher's defaults
(max_hits 1 500, fully_score 1 500, use_top_k_ngrams 5 000, add_best_unigrams_to_ngrams).  At each batch size the
loop and the batched call alternate in the same run, their outputs are compared for equality every time, and one
extra batched run reports the phase breakdown.  Also: queries/s of the decode alone and of decode + batched
aggregation.  Prints the card's name and power limit; writes JSON to --out.

    python tools/evidence_bench.py --batches 20 1000 --out evidence_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

AGG = dict(max_occurrences_1=1500, n_docs_complete_score=1500, alpha=2.0, beta=0.8, length_penalty=0.0,
           use_fm_index_frequency=True, add_best_unigrams_to_ngrams=True, use_top_k_unigrams=5000, sort_by_length=False,
           sort_by_freq=False, smoothing=5.0, allow_overlaps=False, single_key=0.0, unigrams_ignore_free_places=False)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        pl = f"unknown ({e})"
    return name, pl


def keys_from_records(rec):
    keys = []
    for q in range(rec["valid"].shape[0]):
        best = {}
        for h in np.flatnonzero(rec["valid"][q]):
            k = tuple(int(t) for t in rec["tokens"][q, h, :rec["lens"][q, h]] if t > 2)
            if k:
                best[k] = max(best.get(k, -np.inf), float(rec["scores"][q, h]))
        keys.append([(list(k), s) for k, s in best.items()])
    return keys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[20, 1000])
    ap.add_argument("--reps", type=int, default=2, help="alternations of loop and batched call per batch size")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from bench import build_inputs, make_model, BEAM, MIN_LEN, MAX_LEN, LP
    from seal_b200.beam_search import generate_records
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.keys import aggregate_evidence, batch_aggregate_evidence, compute_unigram_scores, _batch_evidence, _AGG_DEFAULTS
    from seal_b200.synthetic import corpus_symbols
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    n_max = max(args.batches)
    docs, ids, mask = build_inputs(n_max, seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    model = make_model()
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM, forced_bos_token_id=None)
    generate_records(model, index, ids[:8], mask[:8], **kw)                       # warm-up (engine upload)
    t = time.perf_counter(); rec = generate_records(model, index, ids, mask, **kw); t_dec = time.perf_counter() - t
    keys = keys_from_records(rec)
    unis = list(compute_unigram_scores(model, ids, tolist=False).astype(np.float64))
    print(f"decode: {n_max} queries in {t_dec:.3f} s ({n_max / t_dec:.0f} q/s); keys/query: mean "
          f"{np.mean([len(k) for k in keys]):.1f}", flush=True)
    report = dict(card=name, power_limit=pl, corpus_tokens=int(docs.size), decode_s=t_dec, decode_qps=n_max / t_dec,
                  keys_per_query=float(np.mean([len(k) for k in keys])), batches={})
    batch_aggregate_evidence(keys[:4], unis[:4], index, **AGG)                    # warm-up (allocator, module load)
    for B in args.batches:
        kq, uq = keys[:B], unis[:B]
        loop_s, batch_s = [], []
        for r in range(args.reps):
            t = time.perf_counter(); exp = [aggregate_evidence(k, u, index, **AGG) for k, u in zip(kq, uq)]
            loop_s.append(time.perf_counter() - t)
            print(f"  batch {B} rep {r}: loop {loop_s[-1]:.3f} s", flush=True)
            t = time.perf_counter(); got = batch_aggregate_evidence(kq, uq, index, **AGG); batch_s.append(time.perf_counter() - t)
            print(f"  batch {B} rep {r}: batched {batch_s[-1]:.3f} s", flush=True)
            assert len(got) == len(exp) and all(list(g[0].items()) == list(e[0].items()) and list(g[1].items()) == list(e[1].items())
                                                for g, e in zip(got, exp)), f"batched != per-query at batch {B}"
        phases = {}
        _batch_evidence(kq, uq, index, {**_AGG_DEFAULTS, **AGG}, phases)
        docs_per_q = float(np.mean([len(g[0]) for g in got]))
        row = dict(loop_s=loop_s, batched_s=batch_s, loop_ms_per_query=1e3 * min(loop_s) / B,
                   batched_ms_per_query=1e3 * min(batch_s) / B, speedup=min(loop_s) / min(batch_s),
                   phases_ms={k: 1e3 * v for k, v in phases.items()}, docs_per_query=docs_per_q, equal=True)
        report["batches"][str(B)] = row
        print(f"batch {B}: loop {min(loop_s):.3f} s ({row['loop_ms_per_query']:.2f} ms/query), batched {min(batch_s):.3f} s "
              f"({row['batched_ms_per_query']:.2f} ms/query), x{row['speedup']:.1f}; equal", flush=True)
        print("  phases (ms): " + ", ".join(f"{k} {v:.1f}" for k, v in row["phases_ms"].items()), flush=True)
    B = n_max
    agg = min(report["batches"][str(B)]["batched_s"])
    loop = min(report["batches"][str(B)]["loop_s"])
    report["end_to_end_qps"] = dict(decode_only=B / t_dec, decode_plus_batched=B / (t_dec + agg),
                                    decode_plus_loop=B / (t_dec + loop))
    print("end to end (q/s): " + ", ".join(f"{k} {v:.0f}" for k, v in report["end_to_end_qps"].items()), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
