"""bf16 weights (gemm_mode 6, the 3xBF16 GEMM) on the benchmark workload: bench.py's corpus (10 M-token index) and
queries, beam 15, body n-grams of 10 (9 decode steps), random weights.

  bart-large   bench.py's model in fp32 (gemm_mode 3) and the same model `.to(torch.bfloat16)` (gemm_mode 6, chosen by
               the dtype rule), both resident, timed alternately in rounds at each batch size
  t5-xxl       the t5-v1_1-xxl layers (d 4 096, 64 heads, d_ff 10 240, 24 + 24, gated-gelu, untied lm_head) with the
               corpus's 50 265-id vocabulary, built from bf16 tensors generated one at a time (never a whole model in
               memory); the batches of --xxl-queries in ascending order up to the first whose workspace does not
               fit (a failed allocation leaves the buffers allocated before it, so a smaller batch is not tried after)

Per configuration: ms per generate (CUDA events around --steps calls after --warmup; Q = 20 replays the call's CUDA
graph), device_bytes, the error flags, and the GPU's name, power limit and median SM clock during the timed calls.
One JSON line per configuration.

    python tools/bf16_bench.py [--steps 3] [--warmup 1] [--rounds 3] [--queries 20,1000] [--xxl-queries 20,100,200,300,400,500]
                               [--models bart-large,t5-xxl]
"""
import argparse
import json
import math
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import BEAM, LP, MAX_LEN, MIN_LEN, ClockSampler, build_inputs, make_model  # noqa: E402
from diverse_bench import gpu_info  # noqa: E402

XXL = dict(d_model=4096, num_heads=64, d_kv=64, d_ff=10240, num_layers=24, num_decoder_layers=24,
           feed_forward_proj="gated-gelu", tie_word_embeddings=False)


def xxl_engine(vocab):
    """a SealT5Engine of the XXL shape from seeded bf16 tensors made on the GPU one at a time"""
    import torch
    from transformers import T5Config
    from seal_b200.beam_search import SealT5Engine
    d, f, H = XXL["d_model"], XXL["d_ff"], XXL["num_heads"]
    shapes = {"shared.weight": (vocab, d), "lm_head.weight": (vocab, d), "encoder.final_layer_norm.weight": (d,),
              "decoder.final_layer_norm.weight": (d,),
              "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (32, H),
              "decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (32, H)}
    for stack, subs in (("encoder", ["SelfAttention"]), ("decoder", ["SelfAttention", "EncDecAttention"])):
        for i in range(24):
            p = f"{stack}.block.{i}.layer."
            for j, a in enumerate(subs):
                shapes.update({f"{p}{j}.{a}.{w}.weight": (d, d) for w in "qkvo"})
                shapes[f"{p}{j}.layer_norm.weight"] = (d,)
            j = len(subs)
            shapes.update({f"{p}{j}.DenseReluDense.wi_0.weight": (f, d), f"{p}{j}.DenseReluDense.wi_1.weight": (f, d),
                           f"{p}{j}.DenseReluDense.wo.weight": (d, f), f"{p}{j}.layer_norm.weight": (d,)})

    class Lazy:
        def items(self):
            for i, (k, s) in enumerate(shapes.items()):
                if len(s) == 1:
                    yield k, torch.full(s, 0.02 if k.startswith("decoder.final") else 1.0, dtype=torch.bfloat16, device="cuda")
                    continue
                g = torch.Generator(device="cuda").manual_seed(i)
                std = 1.0 if k == "lm_head.weight" else 0.1 if "relative" in k else 1.0 / math.sqrt(s[1])
                yield k, (torch.randn(s, generator=g, device="cuda") * std).to(torch.bfloat16)

        def get(self, k, default=None):
            return default

    cfg = T5Config(vocab_size=vocab, dropout_rate=0.0, pad_token_id=0, eos_token_id=1, decoder_start_token_id=0, **XXL)
    cfg.forced_bos_token_id = None; cfg.forced_eos_token_id = None
    eng = SealT5Engine(Lazy(), cfg, device=0, gemm_mode=6)
    torch.cuda.empty_cache()
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--queries", default="20,1000")
    ap.add_argument("--xxl-queries", default="20,100,200,300,400,500")
    ap.add_argument("--models", default="bart-large,t5-xxl")
    args = ap.parse_args()
    import torch
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import DeviceRecords, SealBartEngine, generate_records_device
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.sharding import RecordLayout
    from seal_b200.synthetic import VOCAB, corpus_symbols

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    qs = [int(x) for x in args.queries.split(",")]
    xqs = [int(x) for x in args.xxl_queries.split(",")]
    docs, ids_all, mask_all = build_inputs(max(qs + xqs), seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    info = gpu_info(0)
    print(json.dumps({"setup": info, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds}), flush=True)
    kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM)
    H = (MAX_LEN - 1) * 2 * BEAM + BEAM
    stream = torch.cuda.Stream(device=dev)

    def timed(eng, Q):
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
        return {"ms_per_generate": e0.elapsed_time(e1) / args.steps, "cuda_graph": eng.stat("last_used_graph"),
                "error_flags": rec.host()["errors"].tolist(), "sm_clock_mhz": clocks["sm_mhz"]}

    models = args.models.split(",")
    if "bart-large" in models:
        fp = make_model()
        bf = make_model().to(torch.bfloat16)
        engs = {"fp32": SealBartEngine.from_hf(fp, device=0), "bf16": SealBartEngine.from_hf(bf, device=0)}
        del fp, bf
        assert engs["fp32"].gemm_mode == 3 and engs["bf16"].gemm_mode == 6
        for Q in qs:
            runs = {k: [] for k in engs}
            for _ in range(args.rounds):
                for k, eng in engs.items():
                    runs[k].append(timed(eng, Q))
            for k, eng in engs.items():
                ms = [r["ms_per_generate"] for r in runs[k]]
                print(json.dumps({"model": "bart-large", "weights": k, "gemm_mode": eng.gemm_mode, "queries": Q,
                                  "ms_per_generate_median": statistics.median(ms), "ms_per_generate": ms,
                                  "device_gb": eng.device_bytes() / 1e9, "runs": runs[k], **info}), flush=True)
        del engs
        torch.cuda.empty_cache()
    if "t5-xxl" in models:
        eng = xxl_engine(VOCAB)
        for Q in sorted(xqs):
            try:
                r = timed(eng, Q)
            except (SealB200Error, RuntimeError) as e:          # the workspace of this batch does not fit
                print(json.dumps({"model": "t5-xxl", "queries": Q, "does_not_fit": str(e)[:200]}), flush=True)
                break
            print(json.dumps({"model": "t5-xxl", "weights": "bf16", "gemm_mode": 6, "queries": Q,
                              "device_gb": eng.device_bytes() / 1e9, **r, **info}), flush=True)


if __name__ == "__main__":
    main()
