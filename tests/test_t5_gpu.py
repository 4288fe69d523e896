"""GPU: the T5 forward (sealt5_create: t5_kernels.cuh + the shared GEMM, cross-attention and decode kernels) against
transformers' T5ForConditionalGeneration, and every entry point SEALSearcher reaches with a T5 backbone.

  - last-position logits (sealdec_debug_step_logits) against a float64 forward of the same seeded model, with the
    method of test_bart_paths_gpu.py: the finiteness pattern, an absolute bound on the log-probs, a bound relative to
    fp32 HF's own error against float64, and the last_paths bits restated from the shapes;
  - fm_index_generate against the decode oracle (oracle/decode_oracle.py and the top-k / group oracles) on the fp32 HF
    model with SEAL's T5 token conventions (tests/t5_models.py);
  - CUDA-graph replay and query slices bit-identical to the eager call; rescore_keys / compute_unigram_scores against
    float64; the fp16-overflow fallback of sealdec_generate and the documented error of sealdec_teacher_forced."""
import numpy as np
import pytest

from t5_models import EOS, PAD, make_t5, t5_sources, title_corpus

pytestmark = pytest.mark.gpu

BITS = ["enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
        "cross_grouped", "add_ln_row", "add_ln_warp", "splitk_deferred", "splitk_finish", "gemm_full_tile",
        "gemm_cluster", "gemm_tf32", "query_slices", "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate"]
SHAPE_BITS = {"enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
              "cross_grouped", "add_ln_row", "add_ln_warp", "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_relu", "t5_gate"}
CAL_C = 8.0
CAL_FLOOR = 1e-6
ABS_LOGPROB = 1e-4
TOL = 1e-4                      # |dscore| of a recorded hypothesis, the project's decode bound


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
        from seal_b200.beam_search import SealBartEngine, SealT5Engine
        cpu = make_t5(name)
        eng = SealBartEngine.from_hf(cpu, device=0, gemm_mode=3)
        assert isinstance(eng, SealT5Engine)
        _MODELS[name] = (copy.deepcopy(cpu).double().cuda().eval(), copy.deepcopy(cpu).cuda().eval(), cpu, eng)
    return _MODELS[name]


def hf_logits(model, ids, am, B, dec, rows=None):
    import torch
    from transformers.modeling_outputs import BaseModelOutput
    dev = next(model.parameters()).device
    with torch.inference_mode():
        ids_t = torch.as_tensor(ids, device=dev); am_t = torch.as_tensor(am, device=dev)
        enc = model.get_encoder()(input_ids=ids_t, attention_mask=am_t).last_hidden_state
        sel = torch.as_tensor(rows, device=dev) if rows is not None else torch.arange(len(ids), device=dev).repeat_interleave(B)
        out = []
        for r0 in range(0, len(dec), 512):
            s = sel[r0:r0 + 512]
            o = model(encoder_outputs=BaseModelOutput(last_hidden_state=enc[s]), attention_mask=am_t[s],
                      decoder_input_ids=torch.as_tensor(dec[r0:r0 + 512], device=dev), use_cache=False)
            out.append(o.logits[:, -1, :].double().cpu())
    return torch.cat(out).numpy()


def log_softmax(x):
    import torch
    return torch.log_softmax(torch.from_numpy(np.asarray(x, dtype=np.float64)), -1).numpy()


def beam_inputs(rng, Q, B, t, vocab, share):
    """decoder inputs [Q*B, t] starting with decoder_start (0); with `share`, beams copy prefixes of earlier beams of
    their query and anc[r][s] names the lowest row with the same prefix (as a beam search leaves the cache)"""
    dec = rng.integers(2, vocab, size=(Q * B, t)).astype(np.int64)
    dec[:, 0] = PAD
    if not share:
        return dec, None
    for q in range(Q):
        for b in range(1, B):
            p = int(rng.integers(0, b)); k = int(rng.integers(1, t + 1))
            dec[q * B + b, :k] = dec[q * B + p, :k]
    anc = np.empty((Q * B, t), dtype=np.int32)
    for r in range(Q * B):
        q0 = (r // B) * B
        for s in range(t):
            anc[r, s] = next(r2 for r2 in range(q0, r + 1) if np.array_equal(dec[r2, :s + 1], dec[r, :s + 1]))
    return dec, anc


def paths(eng):
    v = eng.stat("last_paths")
    assert v >= 0 and v >> len(BITS) == 0, f"undocumented path bit in {v:#x}"
    return {n for i, n in enumerate(BITS) if v >> i & 1}


def expected_bits(model, S, am, src_tokens):
    right = all(list(row) == sorted(row, reverse=True) for row in am.tolist())
    bits = {"enc_packed" if right and src_tokens != -2 else "enc_unpacked", "cross_small" if S <= 32 else "cross_grouped",
            "t5_enc_attn", "t5_dec_attn", "t5_rms", "t5_gate" if get_model(model)[2].config.is_gated_act else "t5_relu"}
    return bits


def check_bounds(label, got, ref64, ref32):
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isfinite(got), fin), "finiteness pattern differs from float64"
    lg, l64, l32 = log_softmax(got), log_softmax(ref64), log_softmax(ref32)
    e, el = np.abs(got[fin] - ref64[fin]).max(), np.abs(lg[fin] - l64[fin]).max()
    h = np.abs(ref32[fin] - ref64[fin]).max()
    print(f"{label}: ours |dlogit| {e:.2e} |dlogprob| {el:.2e}   fp32 HF |dlogit| {h:.2e}   ratio {e / max(h, 1e-30):.2f}")
    assert el < ABS_LOGPROB, (label, el)
    assert e <= CAL_C * h + CAL_FLOOR, (label, e, h)


# (name, model, Q, S, B, P, kwargs): packed and unpacked sources, sources long enough for the encoder buckets to
# saturate (distance > max_distance: 128 by default, 48 on tiny_gated), decoder positions up to 127 with ancestry,
# B = 1 .. 32, both feed-forward kinds, gemm_mode 3 and 2
CASES = [
    ("tiny_S1", "tiny", 3, 1, 2, 2, dict(share=True)),
    ("tiny_B1_P1", "tiny", 2, 12, 1, 1, dict()),
    ("tiny_S150", "tiny", 2, 150, 3, 5, dict(share=True)),
    ("tiny_holes", "tiny", 3, 40, 3, 4, dict(kind="holes", share=True)),
    ("tiny_left", "tiny", 3, 40, 2, 3, dict(kind="left", share=True)),
    ("tiny_unpacked", "tiny", 3, 20, 4, 3, dict(src_tokens=-2, share=True)),
    ("tiny_P128", "tiny", 2, 12, 2, 128, dict(share=True)),
    ("tiny_B32", "tiny", 2, 16, 32, 6, dict(share=True)),
    ("tiny_mode2", "tiny", 3, 33, 4, 3, dict(gemm_mode=2, share=True)),
    ("gated_S100_P60", "tiny_gated", 2, 100, 4, 60, dict(share=True)),
    ("gated_holes", "tiny_gated", 3, 70, 5, 9, dict(kind="holes", share=True)),
    ("gated_mode2", "tiny_gated", 2, 60, 8, 50, dict(gemm_mode=2, share=True, kind="left")),
    ("gated_R4000", "tiny_gated", 250, 12, 16, 3, dict(share=True)),
    ("med_B15", "medium", 2, 20, 15, 15, dict(share=True)),
    ("med_S140", "medium", 2, 140, 1, 33, dict()),
    ("med_mode2", "medium", 2, 24, 4, 8, dict(gemm_mode=2, share=True)),
    ("medrelu_holes", "medium_relu", 3, 33, 5, 10, dict(kind="holes", share=True)),
    ("medrelu_B24", "medium_relu", 2, 16, 24, 20, dict(share=True)),
]


@pytest.mark.parametrize("name,model,Q,S,B,P,kw", CASES, ids=[c[0] for c in CASES])
def test_forward_vs_float64(name, model, Q, S, B, P, kw):
    m64, m32, cpu, eng = get_model(model)
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(sum(map(ord, name)))
    kind, src_tokens, mode = kw.get("kind", "right"), kw.get("src_tokens", -1), kw.get("gemm_mode", 3)
    ids, am = t5_sources(rng, Q, S, V, kind)
    dec, anc = beam_inputs(rng, Q, B, P, V, kw.get("share", False) and B > 1 and P > 1)
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
    finally:
        if mode != 3:
            eng.set_option("gemm_mode", 3)
    ref64, ref32 = hf_logits(m64, ids, am, B, dec), hf_logits(m32, ids, am, B, dec)
    check_bounds(f"{name} anc", outs[0], ref64, ref32)
    if anc is not None:
        check_bounds(f"{name} identity", outs[1], ref64, ref32)


def test_state_dict_keys_of_both_ffn_kinds():
    """Every key of an HF state_dict of either feed-forward kind loads; the other kind's keys, stray keys and
    wrong sizes are rejected; a missing tensor fails finalize."""
    from seal_b200._lib import SealB200Error, lib, check, T5Config as NativeCfg
    import ctypes as C
    from seal_b200.beam_search import t5_native_config
    for name, other in (("tiny", "DenseReluDense.wi_0"), ("tiny_gated", "DenseReluDense.wi")):
        model = make_t5(name)
        sd = model.state_dict()
        cfg = t5_native_config(model.config, 3)
        h = C.c_void_p()
        check(lib.sealt5_create(C.byref(cfg), 0, C.byref(h)))
        try:
            for k, v in sd.items():
                a = np.ascontiguousarray(v.float().numpy())
                check(lib.sealbart_set_tensor(h, k.encode(), a.ctypes.data, a.size))
            check(lib.sealbart_finalize(h))
            w = np.zeros(128 * 256, dtype=np.float32)
            for bad in (f"encoder.block.0.layer.1.{other}.weight", "encoder.block.0.layer.0.SelfAttention.q.bias",
                        "encoder.block.1.layer.0.SelfAttention.relative_attention_bias.weight",
                        "model.shared.weight", f"encoder.block.2.layer.0.layer_norm.weight"):
                assert lib.sealbart_set_tensor(h, bad.encode(), w.ctypes.data, 128) != 0, bad
            assert lib.sealbart_set_tensor(h, b"encoder.final_layer_norm.weight", w.ctypes.data, 127) != 0
        finally:
            lib.sealbart_free(h)
        h = C.c_void_p()
        check(lib.sealt5_create(C.byref(cfg), 0, C.byref(h)))
        try:
            for k, v in sd.items():
                if k != "decoder.block.1.layer.2.layer_norm.weight":
                    a = np.ascontiguousarray(v.float().numpy())
                    check(lib.sealbart_set_tensor(h, k.encode(), a.ctypes.data, a.size))
            assert lib.sealbart_finalize(h) != 0
        finally:
            lib.sealbart_free(h)
    bad = NativeCfg(2000, 128, 1, 1, 2, 128, 256, 0, 32, 128, 1e-6, 1, 3)            # d_kv 128
    h = C.c_void_p()
    assert lib.sealt5_create(C.byref(bad), 0, C.byref(h)) != 0 and not h.value


# ---- decode ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def corpus():
    from oracle.fm_oracle import OracleIndex
    from seal_b200.index import FMIndex
    docs, teos = title_corpus()
    idx = FMIndex(); idx.initialize(docs, in_memory=True)
    return OracleIndex(docs), idx, teos


def torch_sources(rng, Q, S, V):
    import torch
    ids, am = t5_sources(rng, Q, S, V)
    return torch.from_numpy(ids), torch.from_numpy(am)


def compare_generate(ours, oracle_out, ora, tol=TOL, force=None, keep_q=None):
    """as test_decode_gpu.compare_generate: per query, the hypotheses whose FM-index query force + tokens[1:] occurs"""
    force = list(force or [])
    keep = lambda t: ora.get_count(force + list(t[1:])) > 0
    worst, n = 0.0, 0
    for q, (a, b) in enumerate(zip(ours, oracle_out)):
        if keep_q is not None and not keep_q[q]:
            continue
        fa = sorted([(tuple(t), s) for s, t in a if keep(t)])
        fb = sorted([(tuple(t), s) for s, t, _ in b if keep(t)])
        assert [x[0] for x in fa] == [x[0] for x in fb], f"query {q}: hypothesis sets differ"
        for (ta, sa), (tb, sb) in zip(fa, fb):
            worst = max(worst, abs(sa - sb))
            assert abs(sa - sb) <= tol, (q, ta, sa, sb)
        n += 1
    return worst, n


@pytest.mark.parametrize("model", ["tiny", "tiny_gated"])
@pytest.mark.parametrize("style", ["body", "title"])
def test_fm_index_generate_vs_oracle(model, style, corpus):
    """keep_history=True against the oracle that orders equal scores by flat index, as the kernels do (flat_ties: the
    tied tiny model's logits are sharply peaked, and the order of its equal -inf fill-in candidates decides beams);
    queries whose beams depend on the order of equal finite scores (`tie_sensitive`) are left out"""
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model(model)
    rng = np.random.default_rng(21)
    ids, am = torch_sources(rng, 6, 14, 2000)
    if style == "body":                               # seal/retrieval.py: n-grams of searcher.length
        kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0)
    else:                                             # titles: forced title BOS (1), the title EOS
        kw = dict(num_beams=5, min_length=1, max_length=15, length_penalty=0.0, force_decoding_from=[1], eos_token_id=teos)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, info=info, flat_ties=True, **kw)
    got = fm_index_generate(cpu, idx, ids, am, keep_history=True, **kw)
    assert all(t[0] == PAD for q in got for _, t in q)
    worst, n = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"),
                                keep_q=[not t for t in info["tie_sensitive"]])
    print(f"{model} {style}: worst |dscore| {worst:.2e} over {n} queries, {sum(len(q) for q in got)} hypotheses; "
          f"tie-sensitive: {[q for q, t in enumerate(info['tie_sensitive']) if t]}")
    assert n >= len(got) // 2 + 1


def test_fm_index_generate_topk_groups_and_stock_scorer(corpus):
    """topk, diverse beam groups and keep_history=False on a T5 model; queries whose beams depend on the order of tied
    scores (or, with topk, on a k-th / (k+1)-th logit gap below 1e-4) are excluded, as in the BART tests."""
    from group_oracle import fm_index_generate_groups_oracle
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("tiny")
    rng = np.random.default_rng(33)
    ids, am = torch_sources(rng, 8, 12, 2000)
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
    skw = dict(num_beams=4, min_length=0, max_length=8, length_penalty=1.0, always_allow_eos=True)
    info = {}
    exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, topk=0, info=info, flat_ties=True, keep_history=False, **skw)
    got = fm_index_generate(cpu, idx, ids, am, **skw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"keep_history=False: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1


def assert_identical(a, b):
    for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_graph_replay_and_query_slices_bit_identical(corpus):
    import torch
    from seal_b200._lib import lib, check
    from seal_b200.beam_search import generate_records, generate_records_device
    ora, idx, teos = corpus
    _, _, cpu, eng = get_model("tiny_gated")
    rng = np.random.default_rng(8)
    ids, am = t5_sources(rng, 5, 12, 2000)
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
    # query slices: > 2 048 rows per half, and enough tiles at d = 512 that no GEMM of a slice splits K
    _, _, cpu_m, eng_m = get_model("medium")
    ids, am = t5_sources(np.random.default_rng(9), 280, 12, 2000)
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

def test_rescore_keys_and_unigram_scores_vs_float64():
    import torch
    from seal_b200.keys import compute_unigram_scores, rescore_keys
    m64, m32, cpu, eng = get_model("tiny_gated")
    rng = np.random.default_rng(12)
    inputs = [rng.integers(4, 2000, size=int(rng.integers(3, 40))).tolist() + [EOS] for _ in range(5)]
    keys = [[rng.integers(2, 2000, size=int(rng.integers(1, 9))).tolist() + ([EOS] if rng.random() < 0.5 else [])
             for _ in range(int(rng.integers(1, 6)))] for _ in range(5)]
    got = rescore_keys(cpu, inputs, keys)
    # float64: sum of log p(token) over the key after decoder_start, positions with tokens < 2 masked (seal/keys.py:132)
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

def test_fp16_overflow_falls_back_to_tf32(corpus):
    """Released T5 checkpoints exceed the fp16 range in the feed-forward: a scaled wi_1 pushes an activation past
    65 504.  sealdec_generate re-runs in 3xTF32 and returns the records of a gemm_mode 2 run exactly; the teacher-forced
    entry point reports SEALFM_EINVAL."""
    import torch
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import SealT5Engine, generate_records
    from seal_b200.keys import _teacher_forced
    ora, idx, teos = corpus
    model = make_t5("tiny_gated")
    with torch.no_grad():
        model.decoder.block[0].layer[2].DenseReluDense.wi_1.weight.mul_(3e5)
    eng = SealT5Engine.from_hf(model, device=0, gemm_mode=3)
    ref = SealT5Engine.from_hf(model, device=0, gemm_mode=2)
    rng = np.random.default_rng(5)
    ids, am = t5_sources(rng, 3, 10, 2000)
    kw = dict(num_beams=4, min_length=5, max_length=5, length_penalty=0.0)
    before = eng.stat("overflow_fallbacks")
    got = generate_records(eng, idx, ids, am, **kw)
    assert eng.stat("overflow_fallbacks") == before + 1
    assert_identical(got, generate_records(ref, idx, ids, am, **kw))
    dec = np.full((3, 3), PAD, dtype=np.int64); dec[:, 1:] = rng.integers(2, 2000, size=(3, 2))
    with pytest.raises(SealB200Error) as ei:
        _teacher_forced(eng, ids, am, dec, np.arange(3, dtype=np.int32))
    assert ei.value.code == -1 and "fp16 range exceeded" in str(ei.value)
