"""NQ-sized index construction on the GPU through sealfm_build_gpu_ex (the suffix array in pinned host memory):
wall time per phase and per sorting round, peak device and pinned host memory, and size-independent property checks
(no oracle can be built at this size).

    python tools/build_large_bench.py [--tokens 3200000000] [--out build_large.json]

The text is R permuted replicas of the 10 M-token benchmark corpus, built the way tools/big_index_bench.py builds its
corpus (title separator included), here as the u32 symbol stream passed to the builder without widening.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from seal_b200.synthetic import make_corpus, VOCAB  # noqa: E402

TITLE_EOS = 49314


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=3_200_000_000)
    ap.add_argument("--out", default="build_large.json")
    ap.add_argument("--ngrams", type=int, default=10, help="brute-force n-gram counts (each one scans the whole text)")
    args = ap.parse_args()
    import torch
    from seal_b200._lib import lib, BuildStats, check
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    out = {"tokens_requested": args.tokens,
           "host_ram_bytes": os.sysconf("SC_PHYS_PAGES") * os.sysconf("SC_PAGE_SIZE"),
           "gpu": torch.cuda.get_device_name(0)}
    t = time.time()
    base = make_corpus()
    reps = max(1, args.tokens // (base.shape[0] * (base.shape[1] + 1)))
    rng = np.random.Generator(np.random.PCG64(2024))
    DL = base.shape[1] + 1
    text = np.empty(reps * base.shape[0] * DL, dtype=np.uint32)
    blkn = base.shape[0] * DL
    for r in range(reps):
        perm = np.arange(VOCAB, dtype=np.int32)
        if r:
            perm[4:] = rng.permutation(VOCAB - 4).astype(np.int32) + 4
        blk = perm[base]
        blk[blk == TITLE_EOS] = TITLE_EOS - 1
        d = np.empty((base.shape[0], DL), dtype=np.int32)
        d[:, :6] = blk[:, :6]; d[:, 6] = TITLE_EOS; d[:, 7:] = blk[:, 6:]
        text[r * blkn:(r + 1) * blkn] = (d[:, ::-1].astype(np.uint32) + 10).reshape(-1)     # seal/index.py:50-53
    n = len(text)
    out["tokens"] = n
    out["corpus_s"] = time.time() - t
    print(f"corpus: {n} tokens in {out['corpus_s']:.0f} s", flush=True)
    torch.cuda.synchronize()
    t = time.time()
    h = C.c_void_p()
    check(lib.sealfm_build_gpu_ex(text.ctypes.data, n, 4, 0, None, C.byref(h)))
    out["build_s"] = time.time() - t
    print(f"built in {out['build_s']:.1f} s", flush=True)
    st = BuildStats()
    check(lib.sealfm_build_gpu_ex_stats(C.byref(st)))
    fm = RawFM(); fm._adopt(h.value)
    out["phases_s"] = dict(zip(["round0_bucketing", "doubling_rounds", "bwt_and_samples", "wavelet_tree"], list(st.phase_s)))
    out["rounds"] = [{"round": r, "s": st.round_s[r], "unsorted_rows": int(st.round_unsorted[r]),
                      "unsorted_fraction": st.round_unsorted[r] / (n + 1)} for r in range(st.rounds)]
    out["chunk_elems"] = int(st.chunk_elems)
    out["windows"] = int(st.windows)
    out["giant_groups"] = int(st.giant_groups)
    out["key_partitions"] = int(st.key_partitions)
    out["wide"] = int(st.wide)
    out["device_peak_GB"] = st.device_peak_bytes / 1e9
    out["pinned_host_GB"] = st.host_pinned_bytes / 1e9
    t = time.time()
    fm.to_device(0)
    from test_fm_build_large_gpu import check_properties
    check_properties(fm, text, np.random.default_rng(5), n_grams=args.ngrams)
    out["properties_ok"] = True
    out["properties_s"] = time.time() - t
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
