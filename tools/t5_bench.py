"""T5 backbones on the benchmark workload: bench.py's corpus (10 M-token index) and queries, beam 15, body n-grams of 10
(9 decode steps), on random-init T5 models of the t5-base and t5-large shapes (relu feed-forward, tied lm_head with
the d_model^-0.5 output scale) and of the T5 v1.1 / Flan-T5 XL shape (`--models t5-xl`: d_model 2 048, gated-gelu,
untied lm_head); vocabulary = the corpus's 50 265 ids so that every query and index token is in range.  The
fp16-overflow count reflects random weights only.

Per model and batch: queries/s and ms per generate (CUDA events around `--steps` calls on the decode stream, after
`--warmup` calls; at Q = 20 these replay the call's CUDA graph), the phase split of one more, eager call
(sealdec_last_phase_us), the fp16-overflow fallback count of the host-buffer entry point on the same batch, and the
GPU's name, power limit and the median SM clock during the timed calls.  One JSON line per configuration on stdout.

    python tools/t5_bench.py [--steps 3] [--warmup 1] [--queries 20,1000] [--models t5-base,t5-large]
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

SHAPES = {"t5-base": dict(d_model=768, num_heads=12, d_ff=3072, num_layers=12, num_decoder_layers=12),
          "t5-large": dict(d_model=1024, num_heads=16, d_ff=4096, num_layers=24, num_decoder_layers=24),
          # the XL member of T5 v1.1 / Flan-T5: ~2.9e9 parameters with this vocabulary, ~23 GB of device weights
          "t5-xl": dict(d_model=2048, num_heads=32, d_ff=5120, num_layers=24, num_decoder_layers=24,
                        feed_forward_proj="gated-gelu", tie_word_embeddings=False)}


def make_t5(name, vocab):
    import torch
    from transformers import T5Config, T5ForConditionalGeneration
    shape = dict(dict(feed_forward_proj="relu", tie_word_embeddings=True), **SHAPES[name])
    cfg = T5Config(vocab_size=vocab, d_kv=64, dropout_rate=0.0, **shape)
    torch.manual_seed(0)
    return T5ForConditionalGeneration(cfg).eval().float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--queries", default="20,1000")
    ap.add_argument("--models", default="t5-base,t5-large")
    args = ap.parse_args()
    import torch
    from seal_b200.beam_search import DeviceRecords, SealBartEngine, generate_records, generate_records_device
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.sharding import RecordLayout
    from seal_b200.synthetic import VOCAB, corpus_symbols

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
    info = gpu_info(0)
    print(json.dumps({"setup": info, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup}), flush=True)
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM)
    H = (MAX_LEN - 1) * 2 * BEAM + BEAM
    stream = torch.cuda.Stream(device=dev)
    for name in args.models.split(","):
        model = make_t5(name, VOCAB)
        eng = SealBartEngine.from_hf(model, device=0)
        del model
        for Q in qs:
            ids_np = np.ascontiguousarray(ids_all[:Q]); mask_np = np.ascontiguousarray(mask_all[:Q])
            ids = torch.from_numpy(ids_np).to(dev); mask = torch.from_numpy(mask_np).to(dev)
            rec = DeviceRecords(RecordLayout(Q, H, MAX_LEN), dev)
            src_tokens = int(mask_np.sum())
            call = lambda: generate_records_device(eng, index, ids, mask, out=rec, src_tokens=src_tokens, stream=stream, **kw)
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
            eng.set_option("cuda_graph", -1)
            before = eng.stat("overflow_fallbacks")
            generate_records(eng, index, ids_np, mask_np, want_ranges=False, **kw)
            print(json.dumps({"model": name, "queries": Q, "queries_per_s": Q / (ms * 1e-3), "ms_per_generate": ms,
                              "cuda_graph": graph, "last_phase_us": phases, "error_flags": errs.tolist(),
                              "overflow_fallbacks": eng.stat("overflow_fallbacks") - before,
                              "sm_clock_mhz": clocks["sm_mhz"], "clock_reasons": clocks["reasons"], **info}), flush=True)
        del eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
