"""Pre-LayerNorm BART-family backbones (Pegasus, mBART) on the benchmark workload, with random weights: the synthetic
10 M-token corpus and queries of seal_b200.synthetic, beam 15, body n-grams of 10 (9 decode steps), against bart-large
under the same conditions.  Shapes:

  pegasus-large  d 1 024, 16 + 16 layers, ffn 4 096, relu, 96 103 ids, scaled embedding, sinusoidal positions
  mbart-large    d 1 024, 12 + 12 layers, ffn 4 096, gelu, 250 027 ids, scaled embedding, layernorm_embedding
  bart-large     BartConfig() defaults (50 265 ids)

Per model, batch and top_k: queries/s and ms per generate (CUDA events around `--steps` calls after `--warmup`; Q = 20
replays the call's CUDA graph, Q = 1 000 runs eagerly), the top-k cluster steps, the fp16-overflow fallback count of
the host-buffer entry point on the same batch, and the GPU's name and power limit.  One JSON line per configuration.

    python tools/preln_bench.py [--steps 3] [--warmup 1] [--queries 20,1000] [--topk 0,10]
                                [--models pegasus-large,mbart-large,bart-large]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BEAM, MIN_LEN, MAX_LEN, LP = 15, 10, 10, 0.0              # SEALSearcher's body n-grams

SHAPES = {
    "pegasus-large": ("pegasus", dict(vocab_size=96103, d_model=1024, encoder_layers=16, decoder_layers=16,
                                      encoder_attention_heads=16, decoder_attention_heads=16, encoder_ffn_dim=4096,
                                      decoder_ffn_dim=4096, activation_function="relu", scale_embedding=True,
                                      max_position_embeddings=1024, pad_token_id=0, eos_token_id=1,
                                      decoder_start_token_id=0, forced_eos_token_id=1)),
    "mbart-large": ("mbart", dict(vocab_size=250027, d_model=1024, encoder_layers=12, decoder_layers=12,
                                  encoder_attention_heads=16, decoder_attention_heads=16, encoder_ffn_dim=4096,
                                  decoder_ffn_dim=4096, activation_function="gelu", scale_embedding=True,
                                  max_position_embeddings=1024)),
    "bart-large": ("bart", dict()),
}


def gpu_info(index):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(index)],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, power = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power}


def make_model(name):
    import torch
    from transformers import BartConfig, BartForConditionalGeneration, MBartConfig, MBartForConditionalGeneration
    from transformers import PegasusConfig, PegasusForConditionalGeneration
    mt, kw = SHAPES[name]
    cfg_cls, model_cls = {"pegasus": (PegasusConfig, PegasusForConditionalGeneration),
                          "mbart": (MBartConfig, MBartForConditionalGeneration),
                          "bart": (BartConfig, BartForConditionalGeneration)}[mt]
    cfg = cfg_cls(**kw)
    cfg.forced_bos_token_id = None
    if mt == "mbart":
        cfg.decoder_start_token_id = cfg.eos_token_id
    torch.manual_seed(0)
    return model_cls(cfg).eval().float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--queries", default="20,1000")
    ap.add_argument("--topk", default="0,10")
    ap.add_argument("--models", default="pegasus-large,mbart-large,bart-large")
    args = ap.parse_args()
    import torch
    from seal_b200.beam_search import DeviceRecords, SealBartEngine, generate_records, generate_records_device
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.sharding import RecordLayout
    from seal_b200.synthetic import corpus_symbols, make_corpus, make_queries

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    qs = [int(x) for x in args.queries.split(",")]
    docs = make_corpus()
    ids_all, mask_all = make_queries(max(qs), seed=4321)
    index = FMIndex()
    RawFM.initialize(index, corpus_symbols(docs))
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1]))
    index._sync_beginnings()
    index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    info = gpu_info(0)
    print(json.dumps({"setup": info, "beam": BEAM, "min_length": MIN_LEN, "max_length": MAX_LEN,
                      "steps": args.steps, "warmup": args.warmup}), flush=True)
    H = (MAX_LEN - 1) * 2 * BEAM + BEAM
    stream = torch.cuda.Stream(device=dev)
    for name in args.models.split(","):
        model = make_model(name)
        eng = SealBartEngine.from_hf(model, device=0)
        del model
        for Q in qs:
            ids_np = np.ascontiguousarray(ids_all[:Q]); mask_np = np.ascontiguousarray(mask_all[:Q])
            ids = torch.from_numpy(ids_np).to(dev); mask = torch.from_numpy(mask_np).to(dev)
            rec = DeviceRecords(RecordLayout(Q, H, MAX_LEN), dev)
            src_tokens = int(mask_np.sum())
            for k in [int(x) for x in args.topk.split(",")]:
                kw = dict(min_length=MIN_LEN, max_length=MAX_LEN, length_penalty=LP, num_beams=BEAM, top_k=k)
                call = lambda: generate_records_device(eng, index, ids, mask, out=rec, src_tokens=src_tokens, stream=stream, **kw)
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(args.steps):
                    call()
                e1.record(stream)
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                graph, cl = eng.stat("last_used_graph"), eng.stat("topk_cluster_steps")
                errs = rec.host()["errors"]
                before = eng.stat("overflow_fallbacks")
                generate_records(eng, index, ids_np, mask_np, want_ranges=False, **kw)
                print(json.dumps({"model": name, "queries": Q, "top_k": k, "queries_per_s": Q / (ms * 1e-3),
                                  "ms_per_generate": ms, "cuda_graph": graph, "topk_cluster_steps": cl,
                                  "error_flags": errs.tolist(), "overflow_fallbacks": eng.stat("overflow_fallbacks") - before,
                                  "device_gb": eng.device_bytes() / 1e9, **info}), flush=True)
            del rec
        del eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
