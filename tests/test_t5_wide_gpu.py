"""GPU: T5 models of the XL / XXL widths (d_model 2 048, 3 072, 4 096: the wide t5_rms_row_kernel instantiation) against
transformers' T5ForConditionalGeneration, with the methods of test_t5_gpu.py on seeded, random-init, shallow models:

  - last-position logits against a float64 forward: packed, unpacked, holed and left-padded sources up to 150
    positions, B = 1 .. 16, decoder positions up to 60 with ancestry, gemm_mode 3 and 2, a small batch whose GEMMs
    split K (the RMSNorm kernel sums the pending slices) and more than 2 048 rows; last_paths names t5_rms_wide, never
    the d <= 1 024 kernel;
  - fm_index_generate against the decode oracle, CUDA-graph replay and query slices bit-identical to the eager call,
    rescore_keys / compute_unigram_scores against float64, and the 3xTF32 re-run after an fp16-range overflow.

Full-depth XL / XXL models are not loaded here: the widths are what these kernels see differently."""
import numpy as np
import pytest

from t5_models import EOS, PAD, t5_sources, title_corpus
from test_t5_gpu import ABS_LOGPROB, assert_identical, beam_inputs, check_bounds, compare_generate, hf_logits, log_softmax

pytestmark = pytest.mark.gpu

BITS = ["enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
        "cross_grouped", "add_ln_row", "add_ln_warp", "splitk_deferred", "splitk_finish", "gemm_full_tile",
        "gemm_cluster", "gemm_tf32", "query_slices", "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate",
        "t5_rms_wide"]
SHAPE_BITS = {"enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
              "cross_grouped", "add_ln_row", "add_ln_warp", "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate",
              "t5_rms_wide"}
VOCAB = 2000

# name -> T5Config arguments (the XL members of T5 v1.1 / Flan-T5 / mT5 have d 2 048, 32 heads, gated-gelu, untied)
SHAPES = {
    "W2048": dict(d_model=2048, num_heads=32, d_ff=1280, num_layers=2, num_decoder_layers=2,
                  feed_forward_proj="gated-gelu", tie_word_embeddings=False),
    "W3072": dict(d_model=3072, num_heads=48, d_ff=512, num_layers=1, num_decoder_layers=2,
                  feed_forward_proj="gated-gelu", tie_word_embeddings=False),
    "W4096": dict(d_model=4096, num_heads=64, d_ff=256, num_layers=1, num_decoder_layers=1,
                  feed_forward_proj="relu", tie_word_embeddings=True),
}


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32


def make_wide(name, seed=0):
    """As tests/t5_models.py:make_t5: the generation attributes of a released config and an untied lm_head of unit
    standard deviation.  The decoder's final_layer_norm weight sets the logits' standard deviation to ~ 2 rather than
    make_t5's ~ 4: at d_model 2 048 the fp32 rounding of a 10-step beam score grows with the logits' scale, and at ~ 4
    both fp32 HF and these kernels reach the 1e-4 score bound against float64"""
    import torch
    from transformers import T5Config, T5ForConditionalGeneration
    cfg = T5Config(vocab_size=VOCAB, d_kv=64, dropout_rate=0.0, pad_token_id=PAD, eos_token_id=EOS, **SHAPES[name])
    cfg.decoder_start_token_id = PAD
    cfg.forced_bos_token_id = None
    cfg.forced_eos_token_id = None
    torch.manual_seed(seed)
    model = T5ForConditionalGeneration(cfg).eval().float()
    d = cfg.d_model
    untied = not SHAPES[name]["tie_word_embeddings"]
    with torch.no_grad():
        if untied:
            g = torch.Generator().manual_seed(seed + 1)
            model.lm_head.weight = torch.nn.Parameter(torch.randn(VOCAB, d, generator=g))
        model.decoder.final_layer_norm.weight.fill_(2.0 / d ** 0.5 if untied else 2.0)
    return model


_MODELS = {}


def get_model(name):
    """(fp64 HF on the GPU, fp32 HF on the GPU, fp32 HF on the CPU, our engine); one width at a time stays loaded"""
    if name not in _MODELS:
        import copy
        import torch
        from seal_b200.beam_search import SealBartEngine, SealT5Engine
        _MODELS.clear()
        torch.cuda.empty_cache()
        cpu = make_wide(name)
        eng = SealBartEngine.from_hf(cpu, device=0, gemm_mode=3)
        assert isinstance(eng, SealT5Engine)
        _MODELS[name] = (copy.deepcopy(cpu).double().cuda().eval(), copy.deepcopy(cpu).cuda().eval(), cpu, eng)
    return _MODELS[name]


def paths(eng):
    v = eng.stat("last_paths")
    assert v >= 0 and v >> len(BITS) == 0, f"undocumented path bit in {v:#x}"
    return {n for i, n in enumerate(BITS) if v >> i & 1}


def expected_bits(model, S, am, src_tokens):
    right = all(list(row) == sorted(row, reverse=True) for row in am.tolist())
    gated = SHAPES[model]["feed_forward_proj"] == "gated-gelu"
    return {"enc_packed" if right and src_tokens != -2 else "enc_unpacked", "cross_small" if S <= 32 else "cross_grouped",
            "t5_enc_attn", "t5_dec_attn", "t5_rms_wide", "t5_gate" if gated else "t5_relu"}


# (name, model, Q, S, B, P, kwargs); "splitk": every GEMM of the decoder step has few enough tiles to split K, and the
# o / co / wo slices reach the RMSNorm kernel unsummed
CASES = [
    ("w2048_splitk", "W2048", 3, 24, 4, 6, dict(share=True, splitk=True)),
    ("w2048_B1_P1", "W2048", 2, 12, 1, 1, dict()),
    ("w2048_unpacked", "W2048", 3, 20, 3, 4, dict(src_tokens=-2, share=True)),
    ("w2048_holes", "W2048", 3, 60, 3, 5, dict(kind="holes", share=True)),
    ("w2048_left_S150", "W2048", 2, 150, 2, 3, dict(kind="left", share=True)),
    ("w2048_P60", "W2048", 2, 16, 4, 60, dict(share=True)),
    ("w2048_B16", "W2048", 2, 12, 16, 8, dict(share=True)),
    ("w2048_mode2", "W2048", 2, 33, 4, 5, dict(gemm_mode=2, share=True)),
    ("w2048_R2100", "W2048", 140, 10, 15, 3, dict(share=True)),
    ("w3072_holes", "W3072", 3, 50, 5, 9, dict(kind="holes", share=True)),
    ("w3072_mode2", "W3072", 2, 24, 4, 6, dict(gemm_mode=2, share=True, kind="left")),
    ("w3072_S150_P40", "W3072", 2, 150, 3, 40, dict(share=True)),
    ("w4096_packed", "W4096", 2, 30, 3, 5, dict(share=True)),
    ("w4096_unpacked", "W4096", 2, 20, 2, 4, dict(src_tokens=-2, share=True)),
    ("w4096_B1", "W4096", 2, 12, 1, 1, dict()),
    ("w4096_mode2", "W4096", 2, 40, 4, 7, dict(gemm_mode=2, share=True, kind="holes")),
]


@pytest.mark.parametrize("name,model,Q,S,B,P,kw", CASES, ids=[c[0] for c in CASES])
def test_wide_forward_vs_float64(name, model, Q, S, B, P, kw):
    m64, m32, cpu, eng = get_model(model)
    rng = np.random.default_rng(sum(map(ord, name)))
    kind, src_tokens, mode = kw.get("kind", "right"), kw.get("src_tokens", -1), kw.get("gemm_mode", 3)
    ids, am = t5_sources(rng, Q, S, VOCAB, kind)
    dec, anc = beam_inputs(rng, Q, B, P, VOCAB, kw.get("share", False) and B > 1 and P > 1)
    if mode != 3:
        eng.set_option("gemm_mode", mode)
    try:
        outs = []
        for a in ([anc, None] if anc is not None else [None]):
            outs.append(eng.debug_step_logits(ids, am, B, dec, anc=a, src_tokens=src_tokens))
            got = paths(eng)
            assert got & SHAPE_BITS == expected_bits(model, S, am, src_tokens), sorted(got)
            if mode == 2:
                assert "gemm_tf32" in got and "gemm_full_tile" not in got
            if kw.get("splitk"):
                assert "splitk_deferred" in got, sorted(got)
    finally:
        if mode != 3:
            eng.set_option("gemm_mode", 3)
    ref64, ref32 = hf_logits(m64, ids, am, B, dec), hf_logits(m32, ids, am, B, dec)
    check_bounds(f"{name} anc", outs[0], ref64, ref32)
    if anc is not None:
        check_bounds(f"{name} identity", outs[1], ref64, ref32)


# ---- decode ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def corpus():
    from oracle.fm_oracle import OracleIndex
    from seal_b200.index import FMIndex
    docs, teos = title_corpus()
    idx = FMIndex(); idx.initialize(docs, in_memory=True)
    return OracleIndex(docs), idx, teos


def torch_sources(rng, Q, S):
    import torch
    ids, am = t5_sources(rng, Q, S, VOCAB)
    return torch.from_numpy(ids), torch.from_numpy(am)


@pytest.mark.parametrize("style", ["body", "title"])
def test_w2048_fm_index_generate_vs_oracle(style, corpus):
    """keep_history=True against the oracle that orders equal scores by flat index, as the kernels do; queries whose
    beams depend on the order of equal finite scores are left out, as in test_t5_gpu.py"""
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import _engine_for, fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, _ = get_model("W2048")
    ids, am = torch_sources(np.random.default_rng(21), 6, 14)
    if style == "body":
        kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0)
    else:
        kw = dict(num_beams=5, min_length=1, max_length=15, length_penalty=0.0, force_decoding_from=[1], eos_token_id=teos)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, info=info, flat_ties=True, **kw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=True, **kw)
    assert all(t[0] == PAD for q in got for _, t in q)
    worst, n = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"),
                                keep_q=[not t for t in info["tie_sensitive"]])
    print(f"W2048 {style}: worst |dscore| {worst:.2e} over {n} queries, {sum(len(q) for q in got)} hypotheses")
    got_paths = paths(_engine_for(cpu))                 # the engine fm_index_generate ran on
    assert "t5_rms_wide" in got_paths and "t5_rms" not in got_paths
    assert n >= len(got) // 2 + 1


def test_w2048_topk_groups_and_stock_scorer(corpus):
    """topk, diverse beam groups and the stock scorer (keep_history=False) on the XL width"""
    from group_oracle import fm_index_generate_groups_oracle
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("W2048")
    ids, am = torch_sources(np.random.default_rng(33), 8, 12)
    kw = dict(num_beams=5, min_length=0, max_length=8, length_penalty=0.0)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=40, info=info, flat_ties=True, **kw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=True, topk=40, **kw)
    worst, n = compare_generate(got, exp, ora, keep_q=[g >= 1e-4 for g in info["min_gap"]])
    print(f"topk=40: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    gkw = dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0)
    info = {}
    exp = fm_index_generate_groups_oracle(cpu, ora, ids, am, info=info, **gkw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=True, **gkw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"diverse groups: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    # with the stock scorer most of these queries have beams that depend on the order of tied scores (equal fill-in
    # candidates where the index allows few continuations): 16 queries, of which the seeded batch leaves 3 to compare
    ids, am = torch_sources(np.random.default_rng(34), 16, 12)
    skw = dict(num_beams=4, min_length=0, max_length=8, length_penalty=1.0, always_allow_eos=True)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, info=info, flat_ties=True, keep_history=False, **skw)
    got = fm_index_generate(cpu, idx, ids, am, **skw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"keep_history=False: worst {worst:.2e} over {n} queries")
    assert n >= 3


def test_w2048_graph_replay_and_query_slices_bit_identical(corpus):
    """300 queries x beam 15 (4 500 rows): the query-sliced call and CUDA-graph replays give the records of the eager,
    unsliced call byte for byte"""
    import torch
    from seal_b200.beam_search import generate_records, generate_records_device
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("W2048")
    ids, am = t5_sources(np.random.default_rng(9), 300, 12, VOCAB)
    kw = dict(num_beams=15, min_length=4, max_length=4, length_penalty=0.0)
    eng.set_option("cuda_graph", 0)
    try:
        eng.set_option("query_slices", 0)
        ref = generate_records(eng, idx, ids, am, **kw)
        assert "query_slices" not in paths(eng)
        eng.set_option("query_slices", 1)
        assert_identical(generate_records(eng, idx, ids, am, **kw), ref)
        assert "query_slices" in paths(eng)
        eng.set_option("cuda_graph", 1)
        ids_d, am_d = torch.from_numpy(ids).cuda(), torch.from_numpy(am).cuda()
        out, used = None, []
        for _ in range(3):
            out = generate_records_device(eng, idx, ids_d, am_d, out=out, src_tokens=int(am.sum()), **kw)
            torch.cuda.synchronize()
            used.append(eng.stat("last_used_graph"))
            got = out.host()
            assert not got["errors"].any()
            assert_identical(got, ref)
        assert used[-1] == 1, used
    finally:
        eng.set_option("query_slices", -1)
        eng.set_option("cuda_graph", -1)


# ---- teacher-forced scoring ---------------------------------------------------------------------------------------

def test_w2048_rescore_keys_and_unigram_scores_vs_float64():
    from seal_b200.keys import compute_unigram_scores, rescore_keys
    m64, m32, cpu, eng = get_model("W2048")
    rng = np.random.default_rng(12)
    inputs = [rng.integers(4, VOCAB, size=int(rng.integers(3, 40))).tolist() + [EOS] for _ in range(5)]
    keys = [[rng.integers(2, VOCAB, size=int(rng.integers(1, 9))).tolist() + ([EOS] if rng.random() < 0.5 else [])
             for _ in range(int(rng.integers(1, 6)))] for _ in range(5)]
    got = rescore_keys(cpu, inputs, keys)
    S = max(len(i) for i in inputs)
    ids = np.zeros((5, S), dtype=np.int64); am = np.zeros_like(ids)
    for q, i in enumerate(inputs):
        ids[q, :len(i)] = i; am[q, :len(i)] = 1
    worst = 0.0
    for q in range(5):
        for (score, k) in got[q]:
            dec = np.array([[PAD] + list(k)], dtype=np.int64)
            want = 0.0
            for p in range(len(k)):
                lp = log_softmax(hf_logits(m64, ids[q:q + 1], am[q:q + 1], 1, dec[:, :p + 1]))[0, k[p]]
                want += lp if k[p] >= 2 else 0.0
            worst = max(worst, abs(score - want))
    print(f"rescore_keys: worst |d| {worst:.2e}")
    assert worst < 1e-4
    full = compute_unigram_scores(cpu, inputs, tolist=False)
    ref = log_softmax(hf_logits(m64, ids, am, 1, np.full((5, 1), PAD, dtype=np.int64)))
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(full), fin)
    e = np.abs(full[fin] - ref[fin]).max()
    print(f"compute_unigram_scores: worst |d| {e:.2e}")
    assert e < ABS_LOGPROB


# ---- fp16 overflow --------------------------------------------------------------------------------------------------

def test_w2048_fp16_overflow_falls_back_to_tf32(corpus):
    """A scaled wi_1 pushes wo's input past 65 504: sealdec_generate re-runs in 3xTF32 and returns the records of a
    gemm_mode 2 run exactly, and that run's logits meet the float64 bounds"""
    import copy
    import torch
    from seal_b200.beam_search import SealT5Engine, generate_records
    ora, idx, teos = corpus
    _MODELS.clear()
    torch.cuda.empty_cache()
    model = make_wide("W2048")
    with torch.no_grad():
        model.decoder.block[0].layer[2].DenseReluDense.wi_1.weight.mul_(1e5)
    eng = SealT5Engine.from_hf(model, device=0, gemm_mode=3)
    ref = SealT5Engine.from_hf(model, device=0, gemm_mode=2)
    rng = np.random.default_rng(5)
    ids, am = t5_sources(rng, 3, 10, VOCAB)
    kw = dict(num_beams=4, min_length=5, max_length=5, length_penalty=0.0)
    before = eng.stat("overflow_fallbacks")
    got = generate_records(eng, idx, ids, am, **kw)
    assert eng.stat("overflow_fallbacks") == before + 1
    assert_identical(got, generate_records(ref, idx, ids, am, **kw))
    dec, anc = beam_inputs(rng, 3, 4, 4, VOCAB, True)
    logits = ref.debug_step_logits(ids, am, 4, dec, anc=anc)
    assert {"gemm_tf32", "t5_rms_wide"} <= paths(ref)
    m64, m32 = copy.deepcopy(model).double().cuda().eval(), copy.deepcopy(model).cuda().eval()
    check_bounds("W2048 fp16 overflow, 3xTF32", logits, hf_logits(m64, ids, am, 4, dec), hf_logits(m32, ids, am, 4, dec))
