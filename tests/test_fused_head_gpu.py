"""GPU: the lm_head statistics epilogue (HeadEpi).  Where the select kernels read only a row's allowed tokens, the
lm_head writes per-tile log-softmax statistics and stores the logits only at the row's read set.  Checked against the
dense path (every logit stored, statistics streamed by topk_rows_kernel): the logits buffer is filled with NaN before
every statistics-epilogue head, so a read outside the read set would change the records; the log-sum-exp is summed in
another order, so scores may differ in the last bits."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def tiny_setup(vocab=2000, n_docs=300, doc_len=30, seed=3):
    from oracle.decode_oracle import make_bart
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    docs = make_corpus(n_docs=n_docs, doc_len=doc_len, n_phrases=2 * n_docs, seed=seed, vocab=vocab)
    idx = FMIndex(); idx.initialize([d.tolist() for d in docs], in_memory=True)
    return idx, make_bart(seed=0, layers=2, vocab=vocab, d_model=128)


def make_inputs(rng, Q, S, vocab):
    ids = rng.integers(4, vocab, size=(Q, S)).astype(np.int64)
    am = np.ones_like(ids)
    ids[:, 0] = 0
    for q in range(Q):
        n = int(rng.integers(max(3, S // 2), S + 1))
        ids[q, n - 1] = 2
        ids[q, n:] = 1
        am[q, n:] = 0
    return ids, am


def run_both(eng, idx, ids, am, **kw):
    from seal_b200._lib import lib, check
    from seal_b200.beam_search import generate_records
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 0))
    check(lib.sealbart_set_option(eng._h, b"fused_head", 0))
    check(lib.sealbart_set_option(eng._h, b"poison_logits", 0))
    dense = generate_records(eng, idx, ids, am, **kw)
    assert lib.sealbart_get_stat(eng._h, b"fused_head_steps") == 0
    check(lib.sealbart_set_option(eng._h, b"fused_head", 1))
    check(lib.sealbart_set_option(eng._h, b"poison_logits", 1))
    try:
        fused = generate_records(eng, idx, ids, am, **kw)
        steps = lib.sealbart_get_stat(eng._h, b"fused_head_steps")
    finally:
        check(lib.sealbart_set_option(eng._h, b"poison_logits", 0))
        check(lib.sealbart_set_option(eng._h, b"fused_head", -1))
    return dense, fused, steps


def assert_same_records(dense, fused, tol=1e-5):
    for k in ("lens", "tokens", "valid", "lo", "hi"):
        assert np.array_equal(dense[k], fused[k]), k
    a, b = dense["scores"], fused["scores"]
    fin = np.isfinite(a)
    assert np.array_equal(fin, np.isfinite(b))
    assert np.array_equal(a[~fin], b[~fin])
    d = np.abs(a[fin].astype(np.float64) - b[fin]).max(initial=0.0)
    assert d <= tol, d
    return d


# (name, generate arguments, statistics-epilogue steps expected): the body shape, the index rules (stop_at_count,
# always_allow_eos), forced BOS (its first full step reads the occurring mask and stays dense), a live EOS
TINY_CASES = [
    ("beam15", dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0), 6),
    ("stop_at_count", dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0, stop_at_count=3), 6),
    ("always_allow_eos", dict(num_beams=15, min_length=3, max_length=8, length_penalty=1.0, always_allow_eos=True), 6),
    ("forced_bos", dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0, forced_bos_token_id=0), 5),
    ("eos_live", dict(num_beams=15, min_length=3, max_length=8, length_penalty=1.0), 6),
]


@pytest.fixture(scope="module")
def tiny():
    from seal_b200.beam_search import SealBartEngine
    idx, model = tiny_setup()
    return idx, SealBartEngine.from_hf(model, device=0)


@pytest.mark.parametrize("name,kw,steps", TINY_CASES, ids=[c[0] for c in TINY_CASES])
def test_fused_head_matches_dense_with_poisoned_logits(tiny, name, kw, steps):
    idx, eng = tiny
    kw = dict(kw)
    kw.setdefault("forced_bos_token_id", None)
    # 40 queries x 15 beams = 600 rows: 5 x 16 GEMM tiles, the persistent (not split-K) lm_head
    ids, am = make_inputs(np.random.default_rng(5), Q=40, S=12, vocab=2000)
    dense, fused, used = run_both(eng, idx, ids, am, **kw)
    # max_length 8: steps at cur_len 2..6 (7 is the dead ForcedEOS step, 1 the compact first step)
    assert used >= steps - 1, used
    d = assert_same_records(dense, fused)
    print(f"{name}: {used} statistics-epilogue steps, worst |dscore| {d:.2e}")


def test_fused_head_diverse_groups_stay_dense(tiny):
    idx, eng = tiny
    ids, am = make_inputs(np.random.default_rng(6), Q=40, S=12, vocab=2000)
    kw = dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0, forced_bos_token_id=None,
              num_beam_groups=3, diversity_penalty=0.5)
    dense, fused, used = run_both(eng, idx, ids, am, **kw)
    assert used == 0
    assert_same_records(dense, fused, tol=0.0)


def test_fused_head_bart_large():
    """bart-large shapes (V = 50 265: 393 tiles of statistics per row, K = 1 024)."""
    from oracle.decode_oracle import make_bart
    from seal_b200.beam_search import SealBartEngine
    idx, _ = tiny_setup()
    eng = SealBartEngine.from_hf(make_bart(seed=0), device=0)
    ids, am = make_inputs(np.random.default_rng(7), Q=12, S=16, vocab=2000)
    kw = dict(num_beams=15, min_length=3, max_length=10, length_penalty=1.0, forced_bos_token_id=None)
    dense, fused, used = run_both(eng, idx, ids, am, **kw)
    assert used >= 7, used
    d = assert_same_records(dense, fused)
    print(f"bart-large: {used} statistics-epilogue steps, worst |dscore| {d:.2e}")
