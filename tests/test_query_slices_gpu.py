"""GPU: query slices.  After the first decode step a generate whose two halves of the batch have more than 2 048 rows
each runs the halves on two streams (include/sealdec.h, "query_slices").  Every kernel then computes each row exactly
as on the whole batch, so the records must be bit-identical with slicing on and off -- on uneven halves, through a
captured CUDA graph, with either lm_head, with diverse groups, without the FM index, with a forced BOS and after the
fp16-range fallback to 3xTF32.  Below the threshold the call stays whole."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PATH_QUERY_SLICES = 1 << 15                    # "last_paths" bit of a sliced generate


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


def make_index(vocab=2000, n_docs=300, doc_len=30, seed=3):
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    docs = make_corpus(n_docs=n_docs, doc_len=doc_len, n_phrases=2 * n_docs, seed=seed, vocab=vocab)
    idx = FMIndex(); idx.initialize([d.tolist() for d in docs], in_memory=True)
    return idx


@pytest.fixture(scope="module")
def setup():
    # d_model 1 024 (bart-large widths, two layers): at > 2 048 rows per slice no decoder GEMM takes split-K
    from oracle.decode_oracle import make_bart
    from seal_b200.beam_search import SealBartEngine
    return make_index(), SealBartEngine.from_hf(make_bart(seed=0, layers=2, vocab=2000), device=0)


def run(eng, idx, ids, am, slices, **kw):
    from seal_b200._lib import lib, check
    from seal_b200.beam_search import generate_records
    check(lib.sealbart_set_option(eng._h, b"query_slices", slices))
    try:
        rec = generate_records(eng, idx, ids, am, **kw)
    finally:
        check(lib.sealbart_set_option(eng._h, b"query_slices", -1))
    return rec, int(lib.sealbart_get_stat(eng._h, b"last_paths"))


def assert_identical(a, b):
    for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
        x, y = a[k], b[k]
        if x is None:
            assert y is None, k
            continue
        assert x.shape == y.shape and x.dtype == y.dtype, k
        assert x.tobytes() == y.tobytes(), k                      # bit for bit, -inf / NaN scores included


BASE = dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0, forced_bos_token_id=None)
CASES = [
    ("q300", 300, {}, -1),
    ("q301_uneven", 301, {}, -1),
    ("dense_head", 300, {}, 0),
    ("fused_head", 300, {}, 1),
    ("eos_live", 300, dict(min_length=3, length_penalty=1.0, always_allow_eos=True), -1),
    ("diverse_groups", 300, dict(num_beam_groups=3, diversity_penalty=0.5), -1),
    ("disable_fm_index", 300, dict(disable_fm_index=True), -1),
    ("forced_bos", 300, dict(forced_bos_token_id=0), -1),
]


@pytest.mark.parametrize("name,Q,extra,fused", CASES, ids=[c[0] for c in CASES])
def test_slices_bit_identical(setup, name, Q, extra, fused):
    from seal_b200._lib import lib, check
    idx, eng = setup
    kw = dict(BASE, **extra)
    ids, am = make_inputs(np.random.default_rng(11), Q=Q, S=12, vocab=2000)
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 0))
    check(lib.sealbart_set_option(eng._h, b"fused_head", fused))
    try:
        whole, p0 = run(eng, idx, ids, am, 0, **kw)
        steps0 = int(lib.sealbart_get_stat(eng._h, b"fused_head_steps"))
        sliced, p1 = run(eng, idx, ids, am, 1, **kw)
        steps1 = int(lib.sealbart_get_stat(eng._h, b"fused_head_steps"))
    finally:
        check(lib.sealbart_set_option(eng._h, b"fused_head", -1))
    assert not p0 & PATH_QUERY_SLICES
    assert p1 & PATH_QUERY_SLICES, hex(p1)
    assert steps0 == steps1
    if fused == 1:
        assert steps1 > 0
    assert_identical(whole, sliced)


def test_slices_through_cuda_graph(setup):
    """First call eager, second captured (both streams join the capture), third a replay: all equal the whole call."""
    from seal_b200._lib import lib, check
    idx, eng = setup
    ids, am = make_inputs(np.random.default_rng(12), Q=301, S=12, vocab=2000)
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 0))
    whole, _ = run(eng, idx, ids, am, 0, **BASE)
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 1))
    try:
        used = []
        for it in range(3):
            got, paths = run(eng, idx, ids, am, 1, **BASE)
            used.append(int(lib.sealbart_get_stat(eng._h, b"last_used_graph")))
            assert paths & PATH_QUERY_SLICES, (it, hex(paths))
            assert_identical(whole, got)
    finally:
        check(lib.sealbart_set_option(eng._h, b"cuda_graph", -1))
    assert used == [0, 1, 1], used


def test_slices_after_fp16_overflow_fallback():
    """Activations beyond the fp16 range: the host-buffer call repeats the pass with the 3xTF32 kernels, sliced too."""
    import torch
    from oracle.decode_oracle import make_bart
    from seal_b200._lib import lib, check
    from seal_b200.beam_search import SealBartEngine
    model = make_bart(seed=0, layers=2, vocab=2000)
    with torch.no_grad():
        model.model.decoder.layers[0].fc1.weight.mul_(2e6)
    eng = SealBartEngine.from_hf(model, device=0)
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 0))
    idx = make_index()
    ids, am = make_inputs(np.random.default_rng(13), Q=300, S=12, vocab=2000)
    whole, _ = run(eng, idx, ids, am, 0, **BASE)
    n0 = int(lib.sealbart_get_stat(eng._h, b"overflow_fallbacks"))
    sliced, paths = run(eng, idx, ids, am, 1, **BASE)
    assert int(lib.sealbart_get_stat(eng._h, b"overflow_fallbacks")) == n0 + 1 >= 2
    assert paths & PATH_QUERY_SLICES and paths & (1 << 14), hex(paths)    # sliced, on the 3xTF32 kernels
    assert_identical(whole, sliced)


def test_small_batch_stays_whole(setup):
    """Q = 200 x 15 beams: 1 500 rows per half, below the threshold -- the call is not split."""
    idx, eng = setup
    ids, am = make_inputs(np.random.default_rng(14), Q=200, S=12, vocab=2000)
    from seal_b200._lib import lib, check
    check(lib.sealbart_set_option(eng._h, b"cuda_graph", 0))
    _, paths = run(eng, idx, ids, am, 1, **BASE)
    assert not paths & PATH_QUERY_SLICES, hex(paths)
