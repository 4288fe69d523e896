"""GPU: the pre-LayerNorm BART-family forward (sealbart_create with a variant: preln_kernels.cuh + BART's attention,
GEMM and decode kernels) against transformers' Pegasus and mBART, and every entry point SEALSearcher reaches with such a
backbone.

  - last-position logits (sealdec_debug_step_logits) against a float64 forward of the same seeded model, with
    test_t5_gpu.py's method: the finiteness pattern, |dlog-prob| <= 1e-4, |dlogit| <= 8 x fp32 HF's own error + 1e-6,
    and the last_paths bits restated from the shapes;
  - fm_index_generate against the decode oracles (flat_ties) on the fp32 HF models, the top-k warp on 96 103 and
    250 027 ids (cluster kernel), diverse groups, the stock scorer, and the README's paraphrase call on a 60-row table;
  - CUDA-graph replay and query slices bit-identical to the eager call; rescore_keys / compute_unigram_scores against
    float64; the fp16-overflow fallback."""
import numpy as np
import pytest

from preln_models import EOS, PAD, make_preln, preln_sources
from t5_models import title_corpus
from test_t5_gpu import assert_identical, beam_inputs, check_bounds, compare_generate, hf_logits, log_softmax

pytestmark = pytest.mark.gpu

BITS = ["enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
        "cross_grouped", "add_ln_row", "add_ln_warp", "splitk_deferred", "splitk_finish", "gemm_full_tile",
        "gemm_cluster", "gemm_tf32", "query_slices", "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate",
        "t5_rms_wide", "preln_norm", "preln_embed_ln"]
SHAPE_BITS = set(BITS[:10]) | {"t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate", "t5_rms_wide", "preln_norm",
                               "preln_embed_ln"}
TOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32


_MODELS = {}


def get_model(name):
    """(fp64 HF on the GPU, fp32 HF on the GPU, fp32 HF on the CPU, our engine)"""
    if name not in _MODELS:
        import copy
        from seal_b200.beam_search import SealBartEngine, SealPreLnEngine
        cpu = make_preln(name)
        eng = SealBartEngine.from_hf(cpu, device=0, gemm_mode=3)
        assert isinstance(eng, SealPreLnEngine)
        _MODELS[name] = (copy.deepcopy(cpu).double().cuda().eval(), copy.deepcopy(cpu).cuda().eval(), cpu, eng)
    return _MODELS[name]


def paths(eng):
    v = eng.stat("last_paths")
    assert v >= 0 and v >> len(BITS) == 0, f"undocumented path bit in {v:#x}"
    return {n for i, n in enumerate(BITS) if v >> i & 1}


def expected_bits(model, Q, S, B, t, am, src_tokens):
    """the shape-determined branches of one debug step call (forward.cu, gemm.cu), restated"""
    cfg = get_model(model)[2].config
    right = all(list(row) == sorted(row, reverse=True) for row in am.tolist())
    bits = {"enc_packed" if right and src_tokens != -2 else "enc_unpacked", "cross_small" if S <= 32 else "cross_grouped",
            "preln_norm"}
    if cfg.model_type == "mbart":
        bits.add("preln_embed_ln")
    if cfg.activation_function == "relu":
        bits.add("t5_relu")
    for pos in range(t):
        P = pos + 1
        saq = 2 * P * B * 64 * 4 + 2 * P * 32 * 4 + 128 * 4
        if pos >= 1 and 2 <= B <= 32 and P <= 128 and saq <= 112 * 1024:
            bits.add("self_query")
        else:
            bits.add("self_rounds3" if P <= 12 else "self_rounds8" if P <= 32 else "self_long")
    return bits


# (name, model, Q, S, B, P, kwargs): packed, unpacked, holed and left-padded sources; positions up to 59 on the 60-row
# Pegasus table and up to 127 on the 128-row ones, with ancestry; B = 1 .. 32; gemm_mode 3 and 2; split-K (the small
# cases) and more than 2 048 rows
CASES = [
    ("peg_S1", "pegasus_relu", 3, 1, 2, 2, dict(share=True)),
    ("peg_B1_P1", "pegasus_relu", 2, 12, 1, 1, dict()),
    ("peg_P60", "pegasus_relu", 2, 12, 2, 60, dict(share=True)),
    ("peg_S60_B1_P40", "pegasus_relu", 2, 60, 1, 40, dict()),
    ("peg_holes", "pegasus_relu", 3, 40, 3, 4, dict(kind="holes", share=True)),
    ("peg_left", "pegasus_relu", 3, 40, 2, 3, dict(kind="left", share=True)),
    ("peg_unpacked", "pegasus_relu", 3, 20, 4, 3, dict(src_tokens=-2, share=True)),
    ("peg_B32", "pegasus_relu", 2, 16, 32, 6, dict(share=True)),
    ("peg_mode2", "pegasus_relu", 3, 33, 4, 3, dict(gemm_mode=2, share=True)),
    ("peg_R4000", "pegasus_relu", 250, 12, 16, 3, dict(share=True)),
    ("pgelu_B15", "pegasus_gelu", 2, 20, 15, 15, dict(share=True)),
    ("pgelu_P128", "pegasus_gelu", 2, 12, 2, 128, dict(share=True)),
    ("pgelu_holes", "pegasus_gelu", 3, 70, 5, 9, dict(kind="holes", share=True)),
    ("pgelu_mode2", "pegasus_gelu", 2, 24, 4, 8, dict(gemm_mode=2, share=True, kind="left")),
    ("mbart_B1_P33", "mbart", 2, 40, 1, 33, dict()),
    ("mbart_B4", "mbart", 2, 20, 4, 10, dict(share=True)),
    ("mbart_S128_P128", "mbart", 2, 128, 2, 128, dict(share=True)),
    ("mbart_mode2", "mbart", 2, 24, 3, 5, dict(gemm_mode=2, share=True, kind="holes")),
    ("mrelu_B24", "mbart_relu", 2, 16, 24, 20, dict(share=True)),
    ("mrelu_left", "mbart_relu", 3, 33, 5, 10, dict(kind="left", share=True)),
    ("mrelu_R2100", "mbart_relu", 140, 10, 15, 2, dict()),
]


@pytest.mark.parametrize("name,model,Q,S,B,P,kw", CASES, ids=[c[0] for c in CASES])
def test_forward_vs_float64(name, model, Q, S, B, P, kw):
    m64, m32, cpu, eng = get_model(model)
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(sum(map(ord, name)))
    kind, src_tokens, mode = kw.get("kind", "right"), kw.get("src_tokens", -1), kw.get("gemm_mode", 3)
    ids, am = preln_sources(rng, Q, S, V, kind)
    dec, anc = beam_inputs(rng, Q, B, P, V, kw.get("share", False) and B > 1 and P > 1)
    if mode != 3:
        eng.set_option("gemm_mode", mode)
    try:
        outs = []
        for a in ([anc, None] if anc is not None else [None]):
            outs.append(eng.debug_step_logits(ids, am, B, dec, anc=a, src_tokens=src_tokens))
            got = paths(eng)
            assert got & SHAPE_BITS == expected_bits(model, Q, S, B, P, am, src_tokens), sorted(got)
            if mode == 2:
                assert "gemm_tf32" in got and "gemm_full_tile" not in got
    finally:
        if mode != 3:
            eng.set_option("gemm_mode", 3)
    ref64, ref32 = hf_logits(m64, ids, am, B, dec), hf_logits(m32, ids, am, B, dec)
    check_bounds(f"{name} anc", outs[0], ref64, ref32)
    if anc is not None:
        check_bounds(f"{name} identity", outs[1], ref64, ref32)


def test_position_table_and_state_dict_keys():
    """Decoder inputs longer than the table and sources longer than max_positions are refused; the other variant's
    keys (layernorm_embedding on Pegasus), stray keys and wrong sizes are rejected; a missing final layer_norm fails
    finalize; unsupported variants fail before any allocation."""
    import ctypes as C
    from seal_b200._lib import BartVariant, SealB200Error, check, lib
    from seal_b200.beam_search import preln_native_config
    _, _, cpu, eng = get_model("pegasus_relu")
    ids, am = preln_sources(np.random.default_rng(1), 2, 8, 2000)
    dec = np.zeros((2, 61), dtype=np.int64)
    with pytest.raises(SealB200Error, match="longer than the position table"):
        eng.debug_step_logits(ids, am, 1, dec)
    from seal_b200.keys import _teacher_forced
    with pytest.raises(SealB200Error, match="longer than the position table"):
        _teacher_forced(eng, ids, am, dec, np.arange(2, dtype=np.int32))
    long_ids, long_am = preln_sources(np.random.default_rng(1), 1, 61, 2000)
    with pytest.raises(SealB200Error, match="source longer than max_positions"):
        eng.debug_step_logits(long_ids, long_am, 1, dec[:1, :2])
    for name, bad_keys in (("pegasus_relu", ["model.encoder.layernorm_embedding.weight", "model.decoder.layers.2.fc1.weight"]),
                           ("mbart_relu", ["model.encoder.layers.3.fc1.weight", "model.encoder.final_layer_norm.weight"])):
        model = make_preln(name)
        sd = model.state_dict()
        cfg, var = preln_native_config(model.config, 3)
        h = C.c_void_p()
        check(lib.sealbart_create(C.byref(cfg), C.byref(var), 0, C.byref(h)))
        try:
            w = np.zeros(128 * 320, dtype=np.float32)
            for bad in bad_keys:
                assert lib.sealbart_set_tensor(h, bad.encode(), w.ctypes.data, 128) != 0, bad
            assert lib.sealbart_set_tensor(h, b"model.decoder.layer_norm.weight", w.ctypes.data, 127) != 0
            for k, v in sd.items():
                if k != "model.decoder.layer_norm.bias":
                    a = np.ascontiguousarray(v.float().numpy())
                    check(lib.sealbart_set_tensor(h, k.encode(), a.ctypes.data, a.size))
            assert lib.sealbart_finalize(h) != 0
        finally:
            lib.sealbart_free(h)
    cfg, _ = preln_native_config(make_preln("pegasus_relu").config, 3)
    for v in ((1, 1, 0, 0), (1, 0, 2, 0), (1, 0, 0, 2), (2, 0, 0, 0), (0, 0, 0, 0), (0, 2, 1, 1)):
        h = C.c_void_p()
        assert lib.sealbart_create(C.byref(cfg), C.byref(BartVariant(*v)), 0, C.byref(h)) != 0 and not h.value, v


# ---- decode ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def corpus():
    from oracle.fm_oracle import OracleIndex
    from seal_b200.index import FMIndex
    docs, teos = title_corpus()
    idx = FMIndex(); idx.initialize(docs, in_memory=True)
    return OracleIndex(docs), idx, teos


def torch_sources(rng, Q, S, V=2000):
    import torch
    ids, am = preln_sources(rng, Q, S, V)
    return torch.from_numpy(ids), torch.from_numpy(am)


def run_vs_oracle(model_name, corpus, seed, Q, S, topk=0, keep_history=True, min_q=None, **kw):
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model(model_name)
    ids, am = torch_sources(np.random.default_rng(seed), Q, S)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=topk, info=info, flat_ties=True, keep_history=keep_history, **kw)
    got = fm_index_generate(eng, idx, ids, am, keep_history=keep_history, topk=topk, **kw)
    # with the warp, as in the T5 and BART top-k tests: queries whose k-th / (k+1)-th logit gap falls below 1e-4 (the
    # oracle breaks ties by flat index, as the kernels do); without it, queries whose beams depend on tied scores
    keep = [g >= 1e-4 for g in info["min_gap"]] if topk > 0 else [not t for t in info["tie_sensitive"]]
    worst, n = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"), keep_q=keep)
    print(f"{model_name} topk={topk} keep_history={keep_history}: worst |dscore| {worst:.2e} over {n} of {Q} queries")
    assert n >= (min_q if min_q is not None else Q // 2 + 1)
    return eng


@pytest.mark.parametrize("model", ["pegasus_relu", "mbart_relu", "pegasus_gelu"])
@pytest.mark.parametrize("style", ["body", "title", "stock"])
def test_fm_index_generate_vs_oracle(model, style, corpus):
    teos = corpus[2]
    if style == "body":
        kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0, stop_at_count=2)
    elif style == "title":
        kw = dict(num_beams=5, min_length=1, max_length=15, length_penalty=0.0, force_decoding_from=[EOS], eos_token_id=teos)
    else:
        kw = dict(num_beams=4, min_length=0, max_length=8, length_penalty=1.0, always_allow_eos=True, keep_history=False)
    run_vs_oracle(model, corpus, 21, 6, 14, **kw)


@pytest.mark.parametrize("model,topk", [("pegasus_relu", 1), ("pegasus_relu", 10), ("pegasus_relu", 100),
                                        ("pegasus_96k", 0), ("pegasus_96k", 10), ("pegasus_96k", 100),
                                        ("mbart_250k", 0), ("mbart_250k", 1), ("mbart_250k", 10)])
def test_topk_vs_oracle(model, topk, corpus):
    """top-k at 96 103 ids runs the cluster threshold kernel with 2 CTAs per row, at 250 027 with 5"""
    eng = run_vs_oracle(model, corpus, 33, 6, 12, topk=topk, num_beams=4, min_length=0, max_length=7, length_penalty=0.0,
                        min_q=2 if topk == 1 else None)
    V = int(eng.config.vocab_size)
    assert (eng.stat("topk_cluster_steps") > 0) == (topk > 0 and V > 53248)


def test_diverse_groups_and_transformers_output(corpus):
    import torch
    from group_oracle import fm_index_generate_groups_oracle
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("pegasus_relu")
    ids, am = torch_sources(np.random.default_rng(5), 6, 12)
    gkw = dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0)
    info = {}
    exp = fm_index_generate_groups_oracle(cpu, ora, ids, am, info=info, **gkw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=True, **gkw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"diverse groups: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    kw = dict(num_beams=4, min_length=2, max_length=9, length_penalty=1.0, always_allow_eos=True)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, info=info, flat_ties=True, keep_history=False,
                                        transformers_output=True, **kw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=False, transformers_output=True, **kw)
    if not any(info["tie_sensitive"]):
        assert torch.equal(got.cpu(), exp)
    # keep_history=True with transformers_output: the reference's uninitialised [Q * num_beams, 3] tensor (zeros here)
    z = fm_index_generate(cpu, idx, ids, am, keep_history=True, transformers_output=True, **kw)
    assert tuple(z.shape) == (6 * 4, 3)


def _readme_call(fmg, model, idx, ids, am, **over):
    kw = dict(keep_history=False, transformers_output=True, always_allow_eos=True, max_length=100)
    kw.update(over)
    return fmg(model, idx, ids, am, **kw)


def test_readme_paraphrase_call_on_a_60_row_table(corpus):
    """The README's paraphrase-mining call (keep_history=False, transformers_output=True, always_allow_eos=True,
    max_length=100) through seal_b200.compat.install()'s seal.beam_search.fm_index_generate on the 60-row Pegasus:
    a batch whose stock scorer finishes before position 60 equals the oracle; one that does not raises the oracle's
    IndexError, and so does keep_history=True at that max_length."""
    import copy
    import sys
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200 import compat
    ora, idx, teos = corpus
    saved = {k: sys.modules.get(k) for k in ("seal", "seal.index", "seal.beam_search", "seal.cpp_modules", "seal.cpp_modules.fm_index")}
    try:
        seal = compat.install()
        fmg = sys.modules["seal.beam_search"].fm_index_generate
        assert seal.fm_index_generate is fmg
        # EOS favoured by its bias: every beam ends within a few steps, the scorer is done long before position 60
        early = make_preln("pegasus_relu")
        with torch.no_grad():
            early.final_logits_bias[0, EOS] = 6.0
        ids, am = torch_sources(np.random.default_rng(40), 4, 12)
        exp = fm_index_generate_topk_oracle(early, ora, ids, am, topk=0, flat_ties=True, keep_history=False,
                                            transformers_output=True, always_allow_eos=True, max_length=100)
        got = _readme_call(fmg, early, idx, ids, am)
        assert torch.equal(got.cpu(), exp), (got, exp)
        # min_length 70 forbids EOS until step 69: the reference's forward reaches position 60 and raises
        _, _, cpu, eng = get_model("pegasus_relu")
        with pytest.raises(IndexError) as e_ref:
            fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, flat_ties=True, keep_history=False,
                                          transformers_output=True, always_allow_eos=True, max_length=100, min_length=70)
        with pytest.raises(IndexError) as e_got:
            _readme_call(fmg, cpu, idx, ids, am, min_length=70)
        assert str(e_got.value) == str(e_ref.value)
        with pytest.raises(IndexError):
            _readme_call(fmg, cpu, idx, ids, am, keep_history=True)
        # max_length 61: keep_history=True reaches position 59, the last row, and runs
        _readme_call(fmg, cpu, idx, ids, am, keep_history=True, transformers_output=False, max_length=61)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_graph_replay_and_query_slices_bit_identical(corpus):
    import torch
    from seal_b200._lib import check, lib
    from seal_b200.beam_search import generate_records, generate_records_device
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("mbart_relu")
    rng = np.random.default_rng(8)
    ids, am = preln_sources(rng, 5, 12, 2000)
    kw = dict(num_beams=4, min_length=6, max_length=6, length_penalty=0.0)
    host = generate_records(eng, idx, ids, am, **kw)
    ids_d, am_d = torch.from_numpy(ids).cuda(), torch.from_numpy(am).cuda()
    out, used = None, []
    for it in range(4):
        out = generate_records_device(eng, idx, ids_d, am_d, out=out, src_tokens=int(am.sum()), **kw)
        torch.cuda.synchronize()
        used.append(eng.stat("last_used_graph"))
        got = out.host()
        assert not got["errors"].any()
        assert_identical(got, host)
    assert used[0] == 0 and used[-1] == 1, used
    # query slices at 300 queries x beam 15: > 2 048 rows per half, enough tiles at d = 512 that no GEMM splits K
    _, _, cpu_m, eng_m = get_model("pegasus_gelu")
    ids, am = preln_sources(np.random.default_rng(9), 300, 12, 2000)
    kw = dict(num_beams=15, min_length=4, max_length=4, length_penalty=0.0)
    recs = []
    for sl in (0, 1):
        check(lib.sealbart_set_option(eng_m._h, b"query_slices", sl))
        try:
            recs.append(generate_records(eng_m, idx, ids, am, **kw))
        finally:
            check(lib.sealbart_set_option(eng_m._h, b"query_slices", -1))
        assert ("query_slices" in paths(eng_m)) == bool(sl)
    assert_identical(recs[0], recs[1])


# ---- teacher-forced scoring ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("model", ["pegasus_relu", "mbart_relu"])
def test_rescore_keys_and_unigram_scores_vs_float64(model):
    from seal_b200.keys import compute_unigram_scores, rescore_keys
    m64, m32, cpu, eng = get_model(model)
    rng = np.random.default_rng(12)
    inputs = [rng.integers(4, 2000, size=int(rng.integers(3, 40))).tolist() + [EOS] for _ in range(5)]
    keys = [[rng.integers(2, 2000, size=int(rng.integers(1, 9))).tolist() + ([EOS] if rng.random() < 0.5 else [])
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
    print(f"{model} rescore_keys: worst |d| {worst:.2e}")
    assert worst < 1e-4
    full = compute_unigram_scores(cpu, inputs, tolist=False)
    ref = log_softmax(hf_logits(m64, ids, am, 1, np.full((5, 1), PAD, dtype=np.int64)))
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(full), fin)
    e = np.abs(full[fin] - ref[fin]).max()
    print(f"{model} compute_unigram_scores: worst |d| {e:.2e}")
    assert e < 1e-4


# ---- fp16 overflow --------------------------------------------------------------------------------------------------

def test_fp16_overflow_falls_back_to_tf32(corpus):
    """A scaled fc1 pushes a feed-forward activation past 65 504: sealdec_generate re-runs in 3xTF32 and returns the
    records of a gemm_mode 2 run exactly, and they match the oracle"""
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import SealPreLnEngine, fm_index_generate, generate_records
    ora, idx, teos = corpus
    model = make_preln("pegasus_relu")
    with torch.no_grad():
        model.model.decoder.layers[0].fc1.weight.mul_(3e5)
    eng = SealPreLnEngine.from_hf(model, device=0, gemm_mode=3)
    ref = SealPreLnEngine.from_hf(model, device=0, gemm_mode=2)
    rng = np.random.default_rng(5)
    ids, am = preln_sources(rng, 3, 10, 2000)
    kw = dict(num_beams=4, min_length=5, max_length=5, length_penalty=0.0)
    before = eng.stat("overflow_fallbacks")
    got = generate_records(eng, idx, ids, am, **kw)
    assert eng.stat("overflow_fallbacks") == before + 1
    assert_identical(got, generate_records(ref, idx, ids, am, **kw))
    ti, ta = torch.from_numpy(ids), torch.from_numpy(am)
    info = {}
    exp = fm_index_generate_topk_oracle(model, ora, ti, ta, topk=0, info=info, flat_ties=True, **kw)
    out = fm_index_generate(eng, idx, ti, ta, keep_history=True, **kw)
    worst, n = compare_generate(out, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"overflow fallback vs oracle: worst {worst:.2e} over {n} queries")
    assert n >= 1
