"""Beyond-L2 index (BASELINE.json configs[2], "Natural Questions index ... batch=20"): a >= 1e9-token synthetic index
built on the GPU, the LF / expansion kernels measured where the metric's "HBM GB/s" exists, and batch-20 / 1 000-query
decodes on it.  No oracle can be built at this size (sdsl needs hours), so parity is checked through size-independent
properties: for sampled corpus n-grams the SA range width equals a brute-force occurrence count over the text, every
located row is an occurrence, and backward_search_multi == the fold of backward_search_step.

    python tools/big_index_bench.py [--tokens 1000000000] [--out big_index.json]

Corpus = R replicas of the 10 M-token phrase corpus (seal_b200.synthetic, seed 1234), each pushed through its own
random permutation of the token ids: same statistics as the benchmark corpus, no n-gram shared between replicas.
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
from seal_b200.synthetic import make_corpus, make_queries, VOCAB  # noqa: E402

TITLE_EOS = 49314          # '@@' in BART's vocabulary: SEALSearcher.title_eos_token_id


def cuda_time(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=1_000_000_000)
    ap.add_argument("--out", default="big_index.json")
    ap.add_argument("--no-decode", action="store_true")
    args = ap.parse_args()
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    out = {"tokens_requested": args.tokens}
    t = time.time()
    base = make_corpus()                                      # [100 000, 100] int32
    reps = max(1, args.tokens // base.size)
    rng = np.random.Generator(np.random.PCG64(2024))
    # documents in SEAL's title form (scripts/build_fm_index.py:132): title tokens, the title separator, body, </s> --
    # the first 6 tokens of every synthetic document act as its title
    docs = np.empty((reps * base.shape[0], base.shape[1] + 1), dtype=np.int32)
    for r in range(reps):
        perm = np.arange(VOCAB, dtype=np.int32)
        if r:
            perm[4:] = rng.permutation(VOCAB - 4).astype(np.int32) + 4      # specials (0..3) stay
        blk = perm[base]
        blk[blk == TITLE_EOS] = TITLE_EOS - 1                           # the separator only ever separates
        d = docs[r * base.shape[0]:(r + 1) * base.shape[0]]
        d[:, :6] = blk[:, :6]; d[:, 6] = TITLE_EOS; d[:, 7:] = blk[:, 6:]
    out["corpus_s"] = time.time() - t
    n = docs.size
    out["tokens"] = int(n)
    t = time.time()
    sym = (docs[:, ::-1].astype(np.uint64) + np.uint64(10)).reshape(-1)     # seal/index.py:50-53
    index = FMIndex(); RawFM.initialize(index, sym)
    out["build_s"] = time.time() - t
    del sym
    t = time.time()
    index.beginnings = list(range(0, n + 1, docs.shape[1])); index._sync_beginnings(); index.to_device(0)
    out["upload_s"] = time.time() - t
    out["device_MB"] = index.device_bytes() / 1e6
    m = index.size()
    dev = torch.device("cuda", 0)
    with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
        hbm = float(json.load(f)["hbm_gbs"])

    # ---- properties instead of an oracle -----------------------------------------------------------------------
    flat = docs.reshape(-1)
    DL = docs.shape[1]
    checks = []
    prng = np.random.default_rng(5)
    for _ in range(6):
        d = int(prng.integers(0, docs.shape[0])); a = int(prng.integers(7, 90)); L = int(prng.integers(1, 5))
        gram = docs[d, a:a + L]
        lo, hi = index.get_range(gram.tolist())
        # brute force over the text: occurrences inside one document (the index text is per-document reversed, so an
        # n-gram cannot span a document boundary except through </s>, which the sampled positions exclude)
        hit = np.ones(n - L + 1, dtype=bool)
        for k in range(L):
            hit &= flat[k:n - L + 1 + k] == gram[k]
        starts = np.nonzero(hit)[0]
        starts = starts[(starts % DL) + L <= DL]
        ok_count = (hi - lo) == len(starts)
        # fold of single steps == multi
        l, r = 0, m
        for tkn in gram.tolist():
            l, r = index.backward_search_step(tkn + 10, l, r)
        ok_fold = (l, r + 1) == (lo, hi)
        # located rows are occurrences: positions are in reversed-text coordinates -> document id must hold the n-gram
        rows = np.arange(lo, min(hi, lo + 64), dtype=np.uint64)
        pos, doc_ids = index.locate_rows(rows)
        ok_loc = all(any((docs[int(di), j:j + L] == gram).all() for j in range(0, DL - L + 1)) for di in doc_ids.tolist())
        checks.append({"len": L, "count": int(hi - lo), "brute": int(len(starts)), "count_ok": bool(ok_count), "fold_ok": bool(ok_fold), "locate_ok": bool(ok_loc)})
    out["property_checks"] = checks
    out["properties_ok"] = all(c["count_ok"] and c["fold_ok"] and c["locate_ok"] for c in checks)

    # ---- LF kernel where HBM is the bound ---------------------------------------------------------------------
    g = torch.Generator(device=dev); g.manual_seed(1)
    Nlf = 1 << 22
    sy = torch.randint(14, 50275, (Nlf,), device=dev, generator=g)
    lo2 = torch.randint(0, m // 2, (Nlf,), device=dev, generator=g)
    hi2 = lo2 + torch.randint(1, m // 2, (Nlf,), device=dev, generator=g)
    s = cuda_time(lambda: index.lf_step_tensors(sy, lo2, hi2))
    import ctypes as C
    from seal_b200._lib import lib as _l, check as _c
    us = C.c_double(0)
    _c(_l.sealfm_debug_sector_probe(int(index.device_bytes()), Nlf * 32, 5, C.byref(us)))
    ceil_gbps = Nlf * 32 * 32 / (us.value * 1e-6) / 1e9
    out["lf_random"] = {"triples": Nlf, "us": s * 1e6, "algorithmic_GBps": Nlf * 768 / s / 1e9, "frac_of_hbm_peak": Nlf * 768 / s / 1e9 / hbm, "hbm_peak_GBps": hbm,
                        "sector_GBps": Nlf * 32 * 32 / s / 1e9, "uniform_random_sector_GBps": ceil_gbps, "ratio_to_uniform_random_sector_rate": (Nlf * 32 * 32 / s / 1e9) / ceil_gbps}
    # count-proportional walk (what a trained model does): ranges from sampled corpus n-grams, expansion of their successor sets
    for R in (15000, 300):
        toks = torch.tensor(flat[prng.integers(0, n, size=R)].astype(np.int64) + 10, device=dev)
        lo = torch.zeros(R, dtype=torch.int64, device=dev); hi = torch.full((R,), m - 1, dtype=torch.int64, device=dev)
        res = {}
        for depth in range(1, 5):
            lo, hi = index.lf_step_tensors(toks, lo, hi)
            width = hi + 1 - lo
            t_lf = cuda_time(lambda: index.lf_step_tensors(toks, lo, hi))
            mask = index.expand_mask_tensors(lo, hi + 1, VOCAB)
            t_ex = cuda_time(lambda: index.expand_mask_tensors(lo, hi + 1, VOCAB, out=mask), iters=5)
            res[depth] = {"lf_us": t_lf * 1e6, "expand_us": t_ex * 1e6, "mean_width": float(width.float().mean()), "max_width": int(width.max())}
            u = torch.rand(R, device=dev)
            row = (lo + (u * width.float()).long()).clamp_(max=m - 1)
            # symbol of a random row of each range = count-proportional next token (distinct of [row, row+1))
            dc = index.distinct_count_multi(row.tolist(), (row + 1).tolist())
            toks = torch.tensor([d[0] if d else 12 for d in dc], dtype=torch.int64, device=dev)
        out[f"walk_R{R}"] = res

    # ---- decode on the big index -------------------------------------------------------------------------------
    if not args.no_decode:
        from bench import make_model
        from seal_b200._lib import lib
        from seal_b200.beam_search import SealBartEngine, generate_records
        index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
        model = make_model()
        eng = SealBartEngine.from_hf(model, device=0)
        del model
        # BASELINE.json configs[4] shape: batch 64, beam 15, title pass (seal/retrieval.py:161-175: min 1 / max 15, decoding
        # forced to start after a </s>, own end-of-title token) followed by the body pass -- 14 + 9 decode steps
        ids64, am64 = make_queries(64, seed=99)
        title_kw = dict(min_length=1, max_length=15, length_penalty=0.0, num_beams=15, forced_bos_token_id=None,
                        force_decoding_from=[2], eos_token_id=TITLE_EOS)
        body_kw = dict(min_length=10, max_length=10, length_penalty=0.0, num_beams=15, forced_bos_token_id=None)
        for _ in range(3):
            generate_records(eng, index, ids64, am64, **title_kw); generate_records(eng, index, ids64, am64, **body_kw)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(5):
            rt = generate_records(eng, index, ids64, am64, **title_kw); rb = generate_records(eng, index, ids64, am64, **body_kw)
        dt = (time.perf_counter() - t0) / 5
        n_titles = int(((rt["valid"] == 1) & (rt["tokens"][np.arange(64)[:, None], np.arange(rt["lens"].shape[1])[None, :], np.maximum(rt["lens"] - 1, 0)] == TITLE_EOS)).sum())
        out["decode_title_plus_body_Q64"] = {"ms_per_batch": dt * 1e3, "queries_per_s": 64 / dt, "complete_titles_found": n_titles,
                                             "used_cuda_graph": int(lib.sealbart_get_stat(eng._h, b"last_used_graph"))}
        for Q in (20, 1000):
            ids, am = make_queries(Q, seed=4321)
            kw = dict(min_length=10, max_length=10, length_penalty=0.0, num_beams=15, forced_bos_token_id=None)
            for _ in range(3):
                rec = generate_records(eng, index, ids, am, **kw)
            torch.cuda.synchronize(); t0 = time.perf_counter()
            it = 5 if Q == 20 else 2
            for _ in range(it):
                rec = generate_records(eng, index, ids, am, **kw)
            dt = (time.perf_counter() - t0) / it
            # every valid record's range is the fold of its tokens
            bad = 0; checked = 0
            for q in range(min(Q, 4)):
                for h in range(rec["scores"].shape[1]):
                    if rec["valid"][q, h] == 1:
                        tk = rec["tokens"][q, h, :rec["lens"][q, h]].tolist()
                        checked += 1
                        bad += (int(rec["lo"][q, h]), int(rec["hi"][q, h])) != tuple(index.get_range(tk[1:]))
            out[f"decode_Q{Q}"] = {"ms_per_generate": dt * 1e3, "queries_per_s": Q / dt, "phases_us": eng.last_phase_us() if Q == 1000 else None,
                                   "ranges_checked": checked, "ranges_bad": int(bad)}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
