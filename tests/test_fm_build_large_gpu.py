"""sealfm_build_gpu_ex (fm_build_large.cu: prefix doubling with the suffix array in pinned host memory) against
sealfm_build (host SA-IS), whose sections are pinned against sdsl's own .fmi files: tree bits, alphabet, C, SA samples
and ISA samples must be identical words.  Small windows force every streaming path, and the build statistics prove
that each one ran."""
import ctypes as C
import os
import tempfile
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SECTIONS = ["tree", "alphabet", "C", "sa_samples", "isa_samples"]
EINVAL, ENOMEM = -1, -3


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


def build_host(text):
    from seal_b200._lib import lib, check
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    a = np.ascontiguousarray(np.asarray(text, dtype=np.uint64))
    out = C.c_void_p()
    check(lib.sealfm_build(a.ctypes.data, len(a), C.byref(out)))
    fm = RawFM(); fm._adopt(out.value)
    return fm


def build_ex(text, width=8, chunk=0, wide=0, budget=0):
    """-> (status, index or None, stats or None)"""
    from seal_b200._lib import lib, BuildOpts, BuildStats
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    a = np.ascontiguousarray(np.asarray(text, dtype=np.uint64 if width == 8 else np.uint32))
    opts = BuildOpts(device_budget_bytes=budget, chunk_elems=chunk, force_wide=wide)
    out = C.c_void_p(12345)
    rc = lib.sealfm_build_gpu_ex(a.ctypes.data, len(a), width, 0, C.byref(opts), C.byref(out))
    if rc != 0:
        assert out.value is None, "a failed build must leave *out null"
        return rc, None, None
    st = BuildStats()
    assert lib.sealfm_build_gpu_ex_stats(C.byref(st)) == 0
    fm = RawFM(); fm._adopt(out.value)
    return rc, fm, st


def assert_same(h, g, label):
    assert g.size() == h.size(), label
    for w, nm in enumerate(SECTIONS):
        a, b = h.section(w), g.section(w)
        assert a.shape == b.shape and np.array_equal(a, b), f"{label}: section {nm} differs"


def _texts():
    from seal_b200.synthetic import make_corpus, corpus_symbols
    rng = np.random.default_rng(17)
    yield "one symbol", [5]
    yield "two symbols", [9, 9]
    for n in (31, 32, 33, 63, 64, 65, 127, 128, 129, 1000):
        yield f"random n={n}", rng.integers(1, 40, size=n)
    yield "single run 7^5000", np.full(5000, 7)
    yield "period-3 text", np.tile([3, 1, 2], 3000)
    yield "all distinct", rng.permutation(4000) + 1
    yield "wide alphabet", rng.integers(1, 2 ** 31, size=3000)
    yield "max symbol 2^32-1", np.array([2 ** 32 - 1, 1, 2 ** 32 - 1, 7, 1], dtype=np.uint64)
    docs = make_corpus(n_docs=2000, doc_len=100, n_phrases=1500, seed=8)      # verbatim repeats, duplicate phrases
    yield "phrase corpus 200k", corpus_symbols(docs)
    yield "duplicated documents", np.concatenate([corpus_symbols(docs[:50])] * 6)


@pytest.mark.parametrize("chunk,wide", [(64, 1), (257, 1), (257, 0), (4096, 1), (0, 1), (0, 0)])
def test_sections_match_host_builder(chunk, wide):
    seen = {"spanning": 0, "giant": 0, "partitions": 0, "single_key": 0, "multi_window_rounds": 0, "text_bytes": set()}
    for label, text in _texts():
        rc, g, st = build_ex(text, chunk=chunk, wide=wide)
        assert rc == 0, label
        assert_same(build_host(text), g, f"{label} (chunk {chunk}, wide {wide})")
        assert st.wide == (1 if wide else 0)
        if chunk:
            assert st.chunk_elems == min(chunk, len(text) + 1)
        seen["spanning"] += st.spanning_groups
        seen["giant"] += st.giant_groups
        seen["partitions"] += st.key_partitions
        seen["single_key"] += st.single_key_buckets
        seen["multi_window_rounds"] += st.max_windows_per_round > 1
        seen["text_bytes"].add(st.text_bytes)
    assert seen["text_bytes"] == {2, 4}                   # u16 and u32 text on the device
    if chunk and chunk <= 4096:
        assert seen["spanning"] > 0, "no group crossed a window edge"
        assert seen["giant"] > 0 and seen["partitions"] > 0, "no group larger than a window went through the key split"
        assert seen["single_key"] > 0, "no single-key bucket larger than a window"
        assert seen["multi_window_rounds"] > 0, "no round needed more than one window"


def test_input_widths_and_errors():
    from seal_b200.synthetic import make_corpus, corpus_symbols
    text = corpus_symbols(make_corpus(n_docs=500, doc_len=60, n_phrases=400, seed=3))
    _, g8, _ = build_ex(text, width=8, chunk=1000)
    _, g4, _ = build_ex(text, width=4, chunk=1000)
    assert_same(g8, g4, "u32 vs u64 input")
    assert_same(build_host(text), g4, "u32 input vs host")
    assert build_ex([3, 0, 4])[0] == EINVAL                               # 0 is the sentinel
    assert build_ex([3, 0, 4], width=4)[0] == EINVAL
    assert build_ex(np.array([3, 2 ** 32, 4], dtype=np.uint64))[0] == EINVAL
    from seal_b200._lib import lib
    a = np.arange(1, 100, dtype=np.uint32)
    out = C.c_void_p(12345)
    assert lib.sealfm_build_gpu_ex(a.ctypes.data, len(a), 3, 0, None, C.byref(out)) == EINVAL and out.value is None
    # a budget below the ISA alone is refused before anything large is allocated
    assert build_ex(np.full(1_000_000, 5), budget=1 << 20)[0] == ENOMEM


def test_benchmark_corpus_with_a_sixteenth_window():
    """The benchmark's 10 M-token corpus through windows of ~m/16 rows; prints both build times."""
    from seal_b200.synthetic import make_corpus, corpus_symbols
    text = corpus_symbols(make_corpus())
    t0 = time.perf_counter(); rc, g, st = build_ex(text, chunk=(len(text) + 1) // 16 + 1); tg = time.perf_counter() - t0
    assert rc == 0
    t0 = time.perf_counter(); h = build_host(text); th = time.perf_counter() - t0
    print(f"index build, 10 M tokens: GPU streamed {tg:.3f} s ({st.rounds} rounds, {st.windows} windows, phases "
          f"{[round(x, 3) for x in st.phase_s]} s, device peak {st.device_peak_bytes / 1e9:.2f} GB), host SA-IS {th:.3f} s")
    assert_same(h, g, "benchmark corpus")
    assert st.max_windows_per_round > 1


def test_fmindex_gpu_large_switch_matches_host(monkeypatch):
    """SEALB200_BUILD=gpu_large through seal_b200.index.FMIndex (both the in-memory and the file path) == host."""
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    seqs = [d.tolist() for d in make_corpus(n_docs=2000, doc_len=100, n_phrases=1500, seed=8)]
    monkeypatch.setenv("SEALB200_BUILD", "host")
    ref = FMIndex(); ref.initialize(seqs, in_memory=True)
    monkeypatch.setenv("SEALB200_BUILD", "gpu_large")
    with tempfile.TemporaryDirectory() as d:
        ref.save(os.path.join(d, "host"))
        for in_memory in (True, False):
            ix = FMIndex(); ix.initialize(seqs, in_memory=in_memory)
            for w in range(5):
                assert np.array_equal(ix.section(w), ref.section(w)), (in_memory, SECTIONS[w])
            assert ix.occurring_distinct == ref.occurring_distinct and ix.occurring_counts == ref.occurring_counts
            ix.save(os.path.join(d, "gpu"))
            with open(os.path.join(d, "host.fmi"), "rb") as a, open(os.path.join(d, "gpu.fmi"), "rb") as b:
                assert a.read() == b.read(), "saved .fmi differs"


def test_run_longer_than_the_window_splits_in_few_partitions():
    """a^n $ with a window far smaller than the run: the giant group's split reads a snapshot of its keys, so each
    round peels the rows whose keys point outside the run in one partition (plus a balanced split of those when they
    outnumber the window) instead of one block of rows per partition."""
    n = 200_000
    text = np.full(n, 1, dtype=np.uint64)
    rc, g, st = build_ex(text, chunk=257, wide=1)
    assert rc == 0
    assert_same(build_host(text), g, "a^200000, window 257")
    assert st.giant_groups > 0
    # cutting c distinct keys into windows takes ~c / W partitions, so at most ~2 n / W per round over all rounds
    # together here (c doubles each round); peeling one block per partition took ~n of them
    assert st.key_partitions <= st.rounds + 2 * n // 257, st.key_partitions


# ---- beyond 2^32 rows --------------------------------------------------------------------------------------------
BIG_N = (1 << 32) + 4999
# host RAM: the u32 text (~17 GB) + the pinned 64-bit suffix array (~34 GB) + the built index and the test's own
# arrays; an estimate, not a measurement
BIG_HOST_BYTES = 64 << 30


def _host_ram():
    return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")


def _need_big_host():
    if _host_ram() < BIG_HOST_BYTES:
        pytest.skip(f"needs ~{BIG_HOST_BYTES >> 30} GiB of available host RAM, {_host_ram() >> 30} GiB available")


def test_run_beyond_2_pow_32_closed_form():
    """a^n $ with n = 2^32 + 4 999: one giant group every round.  SA[i] = n - i, BWT = a^n $, so every section is
    known in closed form (as in test_fm_gpu.test_rows_beyond_2_pow_32)."""
    _need_big_host()
    n = BIG_N; m = n + 1
    rc, g, st = build_ex(np.ones(n, dtype=np.uint32), width=4)
    assert rc == 0
    print(f"a^n, n = {n}: {st.rounds} rounds, phases {[round(x, 1) for x in st.phase_s]} s, "
          f"device peak {st.device_peak_bytes / 1e9:.1f} GB, pinned {st.host_pinned_bytes / 1e9:.1f} GB")
    assert st.wide == 1 and st.giant_groups > 0
    words = (m + 63) // 64
    tree = np.full(words, np.uint64(0xFFFFFFFFFFFFFFFF), dtype=np.uint64)
    tree[n >> 6] = np.uint64((1 << (n & 63)) - 1)
    tree[(n >> 6) + 1:] = 0
    assert g.size() == m
    assert np.array_equal(g.section(0), tree)
    del tree
    assert g.section(1).tolist() == [0, 1] and g.section(2).tolist() == [0, 1, m]
    assert np.array_equal(g.section(3), np.uint64(n) - np.arange((m + 31) // 32, dtype=np.uint64) * np.uint64(32))
    assert np.array_equal(g.section(4), np.uint64(n) - np.arange(n // 64 + 1, dtype=np.uint64) * np.uint64(64))


def test_iid_text_beyond_2_pow_32_properties():
    """An i.i.d. text over 50 265 symbols with n = 2^32 + 4 999: no oracle at this size, so size-independent
    properties (as tools/big_index_bench.py checks them)."""
    _need_big_host()
    n = BIG_N
    rng = np.random.default_rng(11)
    text = np.empty(n, dtype=np.uint32)
    step = 1 << 28
    for a in range(0, n, step):
        text[a:a + step] = rng.integers(10, 10 + 50265, size=min(step, n - a), dtype=np.uint32)
    rc, g, st = build_ex(text, width=4)
    assert rc == 0
    print(f"i.i.d. text, n = {n}: {st.rounds} rounds, phases {[round(x, 1) for x in st.phase_s]} s")
    check_properties(g, text, rng, n_grams=20)       # each brute-force count scans the 4.3e9-symbol text


def check_properties(g, text, rng, n_grams=200):
    """locate(ISA sample row) == its position; suffixes at consecutive SA samples ascend; n-gram counts equal a
    brute-force count; extract_text of sampled rows matches the text."""
    n = len(text); m = n + 1
    isa = g.section(4); sas = g.section(3)
    ks = rng.integers(0, len(isa), size=10_000)
    assert np.array_equal(g.locate_batch(isa[ks]), (ks * 64).astype(np.uint64))
    for i in rng.integers(0, len(sas) - 1, size=2000):
        p, q = int(sas[i]), int(sas[i + 1])
        L = 64
        while True:
            a = text[p:p + L]; b = text[q:q + L]
            k = min(len(a), len(b))
            d = np.nonzero(a[:k] != b[:k])[0]
            if len(d):
                assert a[d[0]] < b[d[0]], (i, p, q)
                break
            if k < L:                                       # one ran into the sentinel: the shorter suffix is smaller
                assert len(a) < len(b), (i, p, q)
                break
            L *= 4
    for _ in range(n_grams):
        p = int(rng.integers(0, n - 4)); k = int(rng.integers(1, 5))
        gram = text[p:p + k]
        hit = np.ones(n - k + 1, dtype=bool)
        for j in range(k):
            hit &= text[j:n - k + 1 + j] == gram[j]
        lo, hi = g.backward_search_multi(gram[::-1].tolist())      # the last query symbol is the first of the match
        assert hi - lo == int(hit.sum()), (p, k)
    for i in rng.integers(0, len(sas), size=50):
        p = int(sas[i])
        e = min(p + 40, n)
        assert g.extract_text(p, e) == text[p:e][::-1].tolist()     # extract_text walks backwards from e
