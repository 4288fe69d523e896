"""Micro-benchmark of the FM-index kernels on the 10 M-token synthetic index (BASELINE.json
configs[1]) with the reference's CPU path timed beside it on a bounded sample.
Writes fm_microbench.json in the current directory.  Not the headline bench (bench.py)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seal_b200.synthetic import make_corpus, corpus_symbols  # noqa: E402
from seal_b200.cpp_modules.fm_index import FMIndex  # noqa: E402


def cuda_time(fn, iters=20, warmup=3):
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
    n_docs = int(os.environ.get("FMB_DOCS", "100000"))
    out = {"n_docs": n_docs}
    t = time.time(); docs = make_corpus(n_docs=n_docs); text = corpus_symbols(docs); out["corpus_s"] = time.time() - t
    t = time.time(); fm = FMIndex(); fm.initialize(text); out["build_s"] = time.time() - t
    t = time.time(); fm.to_device(0); out["upload_s"] = time.time() - t
    m = fm.size(); L = 16
    out["size"] = m
    dev = "cuda"
    rng = np.random.default_rng(0)
    V = 50265
    # walks: R rows, choose next token proportional to corpus counts (trained-model-like) by
    # sampling a random BWT row inside the current range and reading its symbol via distinct on [r,r+1)
    for R in (15000, 300):
        lo = torch.zeros(R, dtype=torch.int64, device=dev); hi = torch.full((R,), m, dtype=torch.int64, device=dev)
        # first token: sample corpus positions
        toks = torch.tensor(text[rng.integers(0, len(text), size=R)].astype(np.int64), device=dev)
        res = {}
        for depth in range(1, 9):
            lo, hi = fm.lf_step_tensors(toks, lo, hi)          # hi inclusive
            width = (hi + 1 - lo)
            t_lf = cuda_time(lambda: fm.lf_step_tensors(toks, lo, hi))
            mask = fm.expand_mask_tensors(lo, hi + 1, V)
            t_ex = cuda_time(lambda: fm.expand_mask_tensors(lo, hi + 1, V, out=mask))
            kb = torch.tensor([bin(int(x) & 0xffffffff).count("1") for x in mask[:64].flatten().tolist()]).view(64, -1).sum(1)
            res[depth] = {"lf_us": t_lf * 1e6, "expand_us": t_ex * 1e6, "mean_width": float(width.float().mean()),
                          "max_width": int(width.max()), "mean_kb_first64": float(kb.float().mean()),
                          "lf_alg_GBps": R * 48 * L / t_lf / 1e9}
            # next token: the symbol of a random row of each range (count-proportional choice)
            u = torch.rand(R, device=dev)
            row = lo + (u * width.float()).long().clamp_(min=0)
            row = torch.minimum(row, hi)
            # symbol at BWT[row]: expand [row,row+1) and find the set bit
            mk = fm.expand_mask_tensors(row, row + 1, V)
            nz = mk != 0
            word = nz.float().argmax(dim=1)
            w = mk.gather(1, word[:, None]).squeeze(1)
            bit = torch.log2((w & -w).abs().float()).long()
            nxt = word * 32 + bit
            has = nz.any(dim=1)
            toks = torch.where(has, nxt + 10, torch.full_like(nxt, 14))
        out[f"walk_R{R}"] = res
    # big LF batch: throughput regime
    N = 1 << 20
    sym = torch.tensor(text[rng.integers(0, len(text), size=N)].astype(np.int64), device=dev)
    lo = torch.randint(0, m // 2, (N,), device=dev); hi = lo + torch.randint(1, m // 2, (N,), device=dev)
    t_lf = cuda_time(lambda: fm.lf_step_tensors(sym, lo, hi), iters=10)
    out["lf_1M"] = {"us": t_lf * 1e6, "steps_per_s": N / t_lf, "alg_GBps": N * 48 * L / t_lf / 1e9}
    rows = rng.integers(0, m, size=1 << 16).astype(np.uint64)
    t = time.time(); fm.locate_batch(rows); out["locate_64k_host_call_s"] = time.time() - t
    # reference on host cores, bounded sample
    try:
        from oracle.fm_oracle import RefFM, ref_available
        if ref_available():
            t = time.time(); ref = RefFM(text); out["ref_build_s"] = time.time() - t
            n = 200000
            s = sym[:n].cpu().numpy().astype(np.uint64); l = lo[:n].cpu().numpy().astype(np.uint64); h = hi[:n].cpu().numpy().astype(np.uint64)
            t = time.time(); rl, rh = ref.backward_search_step_batch(s, l, h); dt = time.time() - t
            out["ref_lf"] = {"steps_per_s_1thread": n / dt}
            gl, gh = fm.lf_step_tensors(sym[:n].contiguous(), lo[:n].contiguous(), hi[:n].contiguous())
            out["ref_lf"]["bit_exact_vs_gpu"] = bool(np.array_equal(gl.cpu().numpy().astype(np.uint64), rl) and np.array_equal(gh.cpu().numpy().astype(np.uint64), rh))
            out["cpu_count"] = os.cpu_count()
    except Exception as ex:  # pragma: no cover
        out["ref_error"] = repr(ex)
    # ---- beyond-L2 index: the metric's "rank-kernel HBM GB/s" needs the tree in DRAM, not in L2 ----
    big = int(os.environ.get("FMB_BIG", "0"))
    if big:
        del fm
        torch.cuda.empty_cache()
        rng2 = np.random.default_rng(1)
        p = 1.0 / (np.arange(50000) + 1.0); cdf = np.cumsum(p / p.sum())
        t = time.time()
        btext = (np.minimum(np.searchsorted(cdf, rng2.random(big)), 49999) + 14).astype(np.uint64)
        out["big_corpus_s"] = time.time() - t
        t = time.time(); bfm = FMIndex(); bfm.initialize(btext); out["big_build_s"] = time.time() - t
        bfm.to_device(0)
        bm = bfm.size()
        from seal_b200._lib import lib
        out["big_index_device_MB"] = lib.sealfm_device_bytes(bfm._h) / 1e6
        res = {}
        for N in (15000, 1 << 18, 1 << 22):
            sym = torch.tensor(btext[rng2.integers(0, big, size=N)].astype(np.int64), device=dev)
            lo = torch.randint(0, bm // 2, (N,), device=dev); hi = lo + torch.randint(1, bm // 2, (N,), device=dev)
            t_lf = cuda_time(lambda: bfm.lf_step_tensors(sym, lo, hi), iters=10)
            res[N] = {"us": t_lf * 1e6, "steps_per_s": N / t_lf, "alg_GBps": N * 48 * L / t_lf / 1e9,
                      "sector_GBps": N * (64 + 16) * L / t_lf / 1e9}
        out["big_lf"] = res
        # expansion of narrow ranges (typical decode rows): width 1..64
        R = 1 << 16
        lo = torch.randint(0, bm - 100, (R,), device=dev); hi = lo + torch.randint(1, 64, (R,), device=dev)
        mask = bfm.expand_mask_tensors(lo, hi, V)
        t_ex = cuda_time(lambda: bfm.expand_mask_tensors(lo, hi, V, out=mask), iters=5)
        out["big_expand_narrow"] = {"R": R, "us": t_ex * 1e6}
    with open("fm_microbench.json", "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out)[:3000])


if __name__ == "__main__":
    main()
