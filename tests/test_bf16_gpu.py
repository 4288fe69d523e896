"""GPU: gemm_mode 6 -- models whose weights are bf16, stored once in bf16 and multiplied by the 3xBF16 GEMM
(wgmma_gemm.cuh, include/sealdec.h).  The oracle is the same bf16 model upcast to float64, which is exact.

  1. the GEMM alone (sealdec_debug_gemm_ex / sealdec_debug_gemm, mode 6) against float64 on activations from 2^-30 to
     2^40, on whole tiles, bands, split-K with its finish pass, the GELU and ReLU epilogues and unsplit operands, held to the
     accumulation bound (48 + K / 256 + 8) 2^-23 sum|a w| with no absolute floor; A W with W = I returns A bit for bit
     (the device split is exact);
  2. the lm_head statistics epilogue in mode 6 (sealdec_debug_head_ex) with test_select_step_gpu.py's checks;
  3. last-position logits of BART, Pegasus (relu), mBART (gelu, layernorm_embedding) and T5 (relu, gated-gelu, one
     shallow 4 096-wide model) against float64, within test_t5_gpu.py's bounds relative to fp32 HF on the upcast model,
     over packed / unpacked / holed sources, split-K batches and more than 2 048 rows;
  4. whole generates against the decode oracles on the upcast model (both scorers, topk, diverse groups, titles),
     CUDA-graph replay and query slices bit-identical to the eager call, rescore_keys / compute_unigram_scores;
  5. a T5 whose feed-forward leaves the fp16 range: one pass, no fallback, against float64;
  6. device_bytes() equals the formula of tests/test_bf16_host.py and is below 0.3 x the fp32-format engine's;
  7. a full-depth t5-v1_1-xxl-shaped engine (≈ 22 GB) built one tensor at a time runs a Q = 20, beam-15 generate."""
import copy
import ctypes as C
import math

import numpy as np
import pytest

from preln_models import make_preln
from t5_models import EOS, PAD, make_t5, t5_sources, title_corpus
from test_bf16_host import device_bytes_formula
from test_select_step_gpu import gamma, words_of
from test_t5_gpu import assert_identical, beam_inputs, check_bounds, compare_generate, hf_logits, log_softmax

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GN = 128
BIT_BF16 = 1 << 24
BITS_OTHER_GEMMS = (1 << 12) | (1 << 13) | (1 << 14)


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32


@pytest.fixture(autouse=True)
def default_mode(monkeypatch):
    monkeypatch.delenv("SEALB200_GEMM", raising=False)       # the dtype rule picks the mode


def bf16_round(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


# ---- 1. the GEMM alone ------------------------------------------------------------------------------------------------

def run_gemm(A, W, b, act, band=-1, presplit=True):
    """act: 0 none, 1 GELU, 2 ReLU"""
    from seal_b200._lib import check, lib
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), dtype=np.float32)
    us = C.c_double(0)
    bp = b.ctypes.data if b is not None else None
    if presplit:
        check(lib.sealdec_debug_gemm_ex(6, M, N, K, A.ctypes.data, W.ctypes.data, bp, out.ctypes.data, act, 0,
                                        C.byref(us), band, 1))
    else:
        check(lib.sealdec_debug_gemm(6, M, N, K, A.ctypes.data, W.ctypes.data, bp, out.ctypes.data, act, 0, C.byref(us)))
    return out


def gelu64(x):
    from scipy.special import erf
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


ROW_EXPS = [-30, -20, -10, 0, 10, 20, 30, 40]

# (label, M, N, K, act, band, presplit): whole tiles (80 tiles > 132 / 2), ragged edges and an odd N, bands (m fastest,
# 2 tiles per band), split-K (8 tiles) with the plain, the GELU and the ReLU finish, an operand the GEMM splits itself;
# act 0 none, 1 GELU, 2 ReLU
GEMM_CASES = [("tiles", 1280, 1024, 1024, 0, -1, True), ("tiles_gelu", 1280, 1024, 1024, 1, -1, True),
              ("ragged", 1300, 1157, 192, 0, -1, True), ("bands", 1024, 4096, 512, 0, 2, True),
              ("splitk", 64, 1024, 1024, 0, -1, True), ("splitk_gelu", 64, 1024, 4096, 1, -1, True),
              ("splitk_relu", 64, 1024, 2048, 2, -1, True), ("unsplit", 300, 512, 256, 1, -1, False)]


@pytest.mark.parametrize("label,M,N,K,act,band,presplit", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_vs_float64(label, M, N, K, act, band, presplit):
    rng = np.random.default_rng(M + N + K)
    scale = np.array([2.0 ** ROW_EXPS[i % len(ROW_EXPS)] for i in range(M)])
    A = (rng.standard_normal((M, K)) * scale[:, None]).astype(np.float32)
    W = rng.standard_normal((N, K)).astype(np.float32) / np.float32(math.sqrt(K))
    b = rng.standard_normal(N).astype(np.float32)
    b[::2] *= 0                                               # bias-free columns: the products alone at every scale
    got = run_gemm(A, W, b, act, band, presplit)
    A64, W64 = A.astype(np.float64), bf16_round(W).astype(np.float64)     # the library rounds W to bf16
    pre = A64 @ W64.T + b.astype(np.float64)
    mag = np.abs(A64) @ np.abs(W64).T
    tol = (48 + K // 256 + 8) * 2.0 ** -23 * mag + 2.0 ** -23 * np.abs(pre)
    exp = pre
    if act == 1:                                              # |gelu'| <= 1.13; erff's error relative to |x|
        exp = gelu64(pre)
        tol = 1.2 * tol + 2.0 ** -22 * (np.abs(pre) + np.abs(exp))
    elif act == 2:                                            # ReLU is 1-Lipschitz: the same bound
        exp = np.maximum(pre, 0.0)
    assert np.isfinite(got).all(), label
    err = np.abs(got - exp)
    ratio = err / np.maximum(tol, 1e-300)
    w = np.unravel_index(np.argmax(ratio), err.shape)
    rel = (err / np.maximum(mag, 1e-300))[:, ::2] / U         # the bias-free columns: the product's own error
    per_scale = {e: round(float(rel[np.arange(M) % len(ROW_EXPS) == i].max()), 2) for i, e in enumerate(ROW_EXPS)}
    print(f"{label}: worst err / bound {ratio.max():.3f} at {tuple(int(i) for i in w)}; bias-free columns, max err / "
          f"(u sum|a w|) per row exponent {per_scale}")
    assert (err <= tol).all(), (label, w, err[w], tol[w])


def test_split_is_exact_on_the_device():
    """A W with W = I: C = b3 + b2 + b1 for every element, which is A exactly when the three pieces are (each partial
    sum is then exact, truncating or not), over exponents -100 .. 126 and both operand paths"""
    rng = np.random.default_rng(3)
    M, K = 1000, 64
    e = rng.integers(-100, 127, size=(M, K))
    A = (np.ldexp(1.0 + rng.random((M, K)), e) * rng.choice([-1.0, 1.0], size=(M, K))).astype(np.float32)
    A[0, :8] = [2.0 ** -100, -(2.0 ** -100), 3.38e38, -3.38e38, 1.0, 0.0, -0.0, 1.0 / 3.0]
    W = np.eye(K, dtype=np.float32)
    for presplit in (True, False):
        got = run_gemm(A, W, None, 0, presplit=presplit)
        assert np.array_equal(np.abs(got).view(np.uint32), np.abs(A).view(np.uint32)), presplit


# ---- 2. the lm_head statistics epilogue --------------------------------------------------------------------------------

def run_head(A, W, b, mask, eos=2, pad=1):
    from seal_b200._lib import check, lib
    M, K = A.shape; N = W.shape[0]
    mp = -(-M // GN) * GN
    Cm = np.empty((mp, N), np.float32); st = np.empty((mp, -(-N // GN), 2), np.float32); fused = np.zeros(1, np.int32)
    check(lib.sealdec_debug_head_ex(6, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, np.ascontiguousarray(mask).ctypes.data,
                                    eos, pad, Cm.ctypes.data, st.ctypes.data, fused.ctypes.data))
    return Cm, st, bool(fused[0])


@pytest.mark.parametrize("M,N,K", [(129, 50265, 64), (2100, 50265, 1024), (300, 129, 64), (1, 128, 1024)])
def test_head_epilogue_vs_float64(M, N, K):
    """as test_select_step_gpu.test_head_epilogue_vs_float64, in mode 6: the stored set is the read set, stored values
    equal the dense mode-6 GEMM bit for bit, the tile max is exact and the tile sum within its rounding bound"""
    from seal_b200._lib import SealB200Error, lib
    rng = np.random.default_rng(M + N + K)
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float32)
    W = (rng.standard_normal((N, K)) * (0.5 / math.sqrt(K))).astype(np.float32)
    b = (-400.0 * ((np.arange(N) // GN) % 3 == 1) + rng.standard_normal(N)).astype(np.float32)
    mask = words_of(rng.integers(0, 100, size=(M, N), dtype=np.uint8) == 0)
    Cm, st, fused = run_head(A, W, b, mask)
    dense = run_gemm(A, W, b, 0)
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    split = -(-N // GN) * -(-M // GN) * 2 <= sms and K // 64 >= 4
    assert np.isnan(Cm[M:]).all()
    if not fused:
        assert split
        assert np.array_equal(Cm[:M].view(np.uint32), dense.view(np.uint32))
        return
    bits = np.unpackbits(mask.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
    read = bits.copy(); read[:, :GN] = True; read[:, 2] = True; read[:, 1] = True
    stored = ~np.isnan(Cm[:M])
    assert np.array_equal(stored, read), np.argwhere(stored != read)[:5]
    assert np.array_equal(Cm[:M][read].view(np.uint32), dense[read].view(np.uint32))
    worst = 0.0
    for t in range(-(-N // GN)):
        x = dense[:, t * GN:(t + 1) * GN].astype(np.float64)
        mx = x.max(1)
        assert np.array_equal(st[:M, t, 0], mx.astype(np.float32)), ("tile max", t)
        d = x - mx[:, None]
        e = np.exp(d); S = e.sum(1)
        bound = U * (e * np.abs(d)).sum(1) + 4 * U * S + gamma(19) * S + GN * 2.0 ** -148
        err = np.abs(st[:M, t, 1].astype(np.float64) - S)
        assert (err <= bound).all(), ("tile sum", t)
        worst = max(worst, float((err / bound).max()))
    print(f"head {M}x{N}x{K} mode 6: worst tile-sum err / bound {worst:.3f}")
    # the other modes stay refused by the _ex entry point
    Cx = np.empty_like(Cm); sx = np.empty_like(st); fx = np.zeros(1, np.int32)
    assert lib.sealdec_debug_head_ex(2, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data, mask.ctypes.data, 2, 1,
                                     Cx.ctypes.data, sx.ctypes.data, fx.ctypes.data) != 0


# ---- 3. forward logits --------------------------------------------------------------------------------------------------

def make_model(name):
    """fp32 HF model of shape `name`; converted to bf16 by the caller"""
    if name.startswith("bart"):
        from oracle.decode_oracle import make_bart
        return make_bart(seed=0, layers=2, vocab=2000, d_model=int(name[4:]))
    if name in ("pegasus_relu", "pegasus_gelu", "mbart", "mbart_relu"):
        return make_preln(name)
    if name == "W4096":
        from test_t5_wide_gpu import make_wide
        return make_wide("W4096")
    return make_t5(name)


_MODELS = {}


def get_model(name):
    """(fp64 HF on the GPU, fp32 HF on the GPU, bf16 HF on the CPU, our engine) -- the HF models are the bf16 one
    upcast (exactly)"""
    if name not in _MODELS:
        import torch
        from seal_b200.beam_search import SealBartEngine
        bf = make_model(name).to(torch.bfloat16)
        eng = SealBartEngine.from_hf(bf, device=0)
        assert eng.gemm_mode == 6
        _MODELS[name] = (copy.deepcopy(bf).double().cuda().eval(), copy.deepcopy(bf).float().cuda().eval(), bf, eng)
    return _MODELS[name]


# (name, model, Q, S, B, P, kwargs): split-K batches, unpacked / holed / left-padded sources, > 2 048 rows
LOGIT_CASES = [
    ("bart_small", "bart128", 3, 12, 4, 5, dict(share=True)),
    ("bart_unpacked", "bart128", 3, 20, 4, 3, dict(src_tokens=-2, share=True)),
    ("bart_R2100", "bart128", 140, 10, 15, 2, dict()),
    ("bart512_B15", "bart512", 2, 20, 15, 12, dict(share=True)),
    ("peg_relu", "pegasus_relu", 3, 40, 3, 4, dict(kind="holes", share=True)),
    ("peg_gelu_left", "pegasus_gelu", 2, 24, 4, 8, dict(kind="left", share=True)),
    ("mbart", "mbart", 2, 20, 4, 10, dict(share=True)),
    ("mbart_relu_R2100", "mbart_relu", 140, 10, 15, 2, dict()),
    ("t5_relu", "tiny", 3, 40, 3, 4, dict(kind="holes", share=True)),
    ("t5_gated", "tiny_gated", 2, 60, 8, 20, dict(share=True)),
    ("t5_gated_R4000", "tiny_gated", 250, 12, 16, 3, dict(share=True)),
    ("t5_medium", "medium", 2, 20, 15, 15, dict(share=True)),
    ("t5_medium_relu_unpacked", "medium_relu", 3, 33, 5, 10, dict(src_tokens=-2, share=True)),
    ("t5_w4096", "W4096", 2, 12, 2, 4, dict(share=True)),
]


@pytest.mark.parametrize("name,model,Q,S,B,P,kw", LOGIT_CASES, ids=[c[0] for c in LOGIT_CASES])
def test_forward_vs_float64(name, model, Q, S, B, P, kw):
    m64, m32, bf, eng = get_model(model)
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(sum(map(ord, name)))
    ids, am = t5_sources(rng, Q, S, V, kw.get("kind", "right"))
    dec, anc = beam_inputs(rng, Q, B, P, V, kw.get("share", False) and B > 1 and P > 1)
    got = eng.debug_step_logits(ids, am, B, dec, anc=anc, src_tokens=kw.get("src_tokens", -1))
    p = eng.stat("last_paths")
    assert p & BIT_BF16 and not p & BITS_OTHER_GEMMS, hex(p)
    check_bounds(name, got, hf_logits(m64, ids, am, B, dec), hf_logits(m32, ids, am, B, dec))


def test_mode_is_fixed_at_creation():
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import SealBartEngine
    _, _, bf, eng = get_model("tiny")
    for m in (2, 3, 5):
        with pytest.raises(SealB200Error) as ei:
            eng.set_option("gemm_mode", m)
        assert "gemm_mode 6" in str(ei.value)
    eng.set_option("gemm_mode", 6)                            # unchanged: allowed
    assert eng.stat("gemm_mode") == 6
    fp = SealBartEngine.from_hf(bf.float(), device=0)
    assert fp.gemm_mode == 3
    with pytest.raises(SealB200Error):
        fp.set_option("gemm_mode", 6)


# ---- 4. whole generates -------------------------------------------------------------------------------------------------

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


# BART's final_logits_bias forbids the corpus's title EOS (its last id): BART decodes bodies only
@pytest.mark.parametrize("model,style", [("tiny_gated", "body"), ("tiny_gated", "title"), ("bart128", "body"),
                                         ("pegasus_relu", "body"), ("pegasus_relu", "title")])
def test_fm_index_generate_vs_oracle(model, style, corpus):
    """fm_index_generate on the bf16 model (gemm_mode 6 by the dtype rule) against the oracle on its fp32 upcast"""
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import _engine_for, fm_index_generate
    ora, idx, teos = corpus
    _, _, bf, _ = get_model(model)
    up = copy.deepcopy(bf).float()
    rng = np.random.default_rng(21)
    ids, am = torch_sources(rng, 6, 14, 2000)
    if style == "body":
        kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0)
    else:
        kw = dict(num_beams=5, min_length=1, max_length=15, length_penalty=0.0, force_decoding_from=[1], eos_token_id=teos)
    info = {}
    exp = fm_index_generate_topk_oracle(up, ora, ids, am, topk=0, info=info, flat_ties=True, **kw)
    got = fm_index_generate(bf, idx, ids, am, keep_history=True, **kw)
    assert _engine_for(bf).gemm_mode == 6
    worst, n = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"),
                                keep_q=[not t for t in info["tie_sensitive"]])
    print(f"{model} {style}: worst |dscore| {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1


def test_topk_groups_stock_scorer_and_transformers_output(corpus):
    from group_oracle import fm_index_generate_groups_oracle
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos = corpus
    _, _, bf, _ = get_model("tiny")
    up = copy.deepcopy(bf).float()
    rng = np.random.default_rng(33)
    ids, am = torch_sources(rng, 8, 12, 2000)
    kw = dict(num_beams=5, min_length=0, max_length=8, length_penalty=0.0)
    info = {}
    exp = fm_index_generate_topk_oracle(up, ora, ids, am, topk=40, info=info, flat_ties=True, **kw)
    got = fm_index_generate(bf, idx, ids, am, keep_history=True, topk=40, **kw)
    worst, n = compare_generate(got, exp, ora, keep_q=[g >= 1e-4 for g in info["min_gap"]])
    print(f"topk=40: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    gkw = dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0)
    info = {}
    exp = fm_index_generate_groups_oracle(up, ora, ids, am, info=info, **gkw)
    got = fm_index_generate(bf, idx, ids, am, keep_history=True, **gkw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"diverse groups: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    skw = dict(num_beams=4, min_length=0, max_length=8, length_penalty=1.0, always_allow_eos=True)
    info = {}
    exp = fm_index_generate_topk_oracle(up, ora, ids, am, topk=0, info=info, flat_ties=True, keep_history=False, **skw)
    got = fm_index_generate(bf, idx, ids, am, **skw)
    worst, n = compare_generate(got, exp, ora, keep_q=[not t for t in info["tie_sensitive"]])
    print(f"keep_history=False: worst {worst:.2e} over {n} queries")
    assert n >= len(got) // 2 + 1
    out = fm_index_generate(bf, idx, ids, am, transformers_output=True, **skw)
    assert out is not None


def test_graph_replay_and_query_slices_bit_identical(corpus):
    import torch
    from seal_b200._lib import check, lib
    from seal_b200.beam_search import generate_records, generate_records_device
    ora, idx, teos = corpus
    _, _, _, eng = get_model("tiny_gated")
    ids, am = t5_sources(np.random.default_rng(8), 5, 12, 2000)
    kw = dict(num_beams=4, min_length=6, max_length=6, length_penalty=0.0)
    host = generate_records(eng, idx, ids, am, **kw)
    assert eng.stat("overflow_fallbacks") == 0
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
    _, _, _, eng_m = get_model("medium")
    ids, am = t5_sources(np.random.default_rng(9), 280, 12, 2000)
    kw = dict(num_beams=15, min_length=4, max_length=4, length_penalty=0.0)
    recs = []
    for sl in (0, 1):
        check(lib.sealbart_set_option(eng_m._h, b"query_slices", sl))
        try:
            recs.append(generate_records(eng_m, idx, ids, am, **kw))
        finally:
            check(lib.sealbart_set_option(eng_m._h, b"query_slices", -1))
        assert bool(eng_m.stat("last_paths") >> 15 & 1) == bool(sl)
    assert_identical(recs[0], recs[1])


def test_rescore_keys_and_unigram_scores_vs_float64():
    from seal_b200.keys import compute_unigram_scores, rescore_keys
    m64, _, bf, _ = get_model("tiny_gated")
    rng = np.random.default_rng(12)
    inputs = [rng.integers(4, 2000, size=int(rng.integers(3, 40))).tolist() + [EOS] for _ in range(5)]
    keys = [[rng.integers(2, 2000, size=int(rng.integers(1, 9))).tolist() + ([EOS] if rng.random() < 0.5 else [])
             for _ in range(int(rng.integers(1, 6)))] for _ in range(5)]
    got = rescore_keys(bf, inputs, keys)
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
    full = compute_unigram_scores(bf, inputs, tolist=False)
    ref = log_softmax(hf_logits(m64, ids, am, 1, np.full((5, 1), PAD, dtype=np.int64)))
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(full), fin)
    e = np.abs(full[fin] - ref[fin]).max()
    print(f"compute_unigram_scores: worst |d| {e:.2e}")
    assert e < 1e-4


# ---- 5. range -----------------------------------------------------------------------------------------------------------

def test_activation_beyond_fp16_range_in_one_pass(corpus):
    """test_t5_gpu's overflow model (wi_1 scaled by 3e5: the wo input passes 65 504) in bf16: logits within the
    float64 bounds, a generate with no fallback, teacher-forced scoring without the fp16 error; the same model upcast
    to fp32 goes through the 3xTF32 fallback"""
    import torch
    from seal_b200.beam_search import SealT5Engine, generate_records
    from seal_b200.keys import _teacher_forced
    ora, idx, teos = corpus
    model = make_t5("tiny_gated")
    with torch.no_grad():
        model.decoder.block[0].layer[2].DenseReluDense.wi_1.weight.mul_(3e5)
    bf = model.to(torch.bfloat16)
    eng = SealT5Engine.from_hf(bf, device=0)
    assert eng.gemm_mode == 6
    rng = np.random.default_rng(5)
    ids, am = t5_sources(rng, 3, 10, 2000)
    dec, _ = beam_inputs(rng, 3, 2, 4, 2000, False)
    m64, m32 = copy.deepcopy(bf).double().cuda(), copy.deepcopy(bf).float().cuda()
    check_bounds("overflow model", eng.debug_step_logits(ids, am, 2, dec), hf_logits(m64, ids, am, 2, dec), hf_logits(m32, ids, am, 2, dec))
    kw = dict(num_beams=4, min_length=5, max_length=5, length_penalty=0.0)
    got = generate_records(eng, idx, ids, am, **kw)
    assert eng.stat("overflow_fallbacks") == 0 and got["valid"].any()
    fp = SealT5Engine.from_hf(copy.deepcopy(bf).float(), device=0)
    assert fp.gemm_mode == 3
    generate_records(fp, idx, ids, am, **kw)
    assert fp.stat("overflow_fallbacks") == 1
    tf = np.full((3, 3), PAD, dtype=np.int64); tf[:, 1:] = rng.integers(2, 2000, size=(3, 2))
    lp, _ = _teacher_forced(eng, ids, am, tf, np.arange(3, dtype=np.int32))
    assert np.isfinite(lp).all()


# ---- 6. device memory ----------------------------------------------------------------------------------------------------

def test_device_bytes_equal_the_formula():
    """exact bytes for T5 (tied and untied), BART and mBART; the 0.3 x bound where matrices dominate (d >= 512: at
    d 128 with 2 000 ids the fp32 position / bucket tables and biases are a sizeable share of the small weights)"""
    import torch
    from seal_b200.beam_search import SealBartEngine
    for name in ("tiny_gated", "medium_relu", "bart128", "mbart"):
        _, _, bf, eng = get_model(name)
        c = bf.config
        if c.model_type == "t5":
            kind = "t5"
            cfg = (c.d_model, c.d_ff, c.vocab_size, c.num_heads, c.num_layers, c.num_decoder_layers,
                   c.feed_forward_proj == "gated-gelu", c.relative_attention_num_buckets)
        else:
            kind = "bart" if c.model_type == "bart" else "preln"
            off = 0 if c.model_type == "pegasus" else 2
            cfg = (c.d_model, c.decoder_ffn_dim, c.vocab_size, c.encoder_layers, c.decoder_layers,
                   c.max_position_embeddings + off, c.model_type != "pegasus")
        tied = bf.lm_head.weight.data_ptr() == bf.get_input_embeddings().weight.data_ptr()
        want6 = device_bytes_formula(kind, cfg, 6, tied)
        assert eng.device_bytes() == want6, (name, eng.device_bytes(), want6)
        fp = SealBartEngine.from_hf(copy.deepcopy(bf).float(), device=0)
        assert fp.device_bytes() == device_bytes_formula(kind, cfg, 3, tied), name
        print(f"{name}: {want6} B in gemm_mode 6, {fp.device_bytes()} B in gemm_mode 3 ({want6 / fp.device_bytes():.3f})")
        if c.d_model >= 512:
            assert eng.device_bytes() < 0.3 * fp.device_bytes(), name
        del fp
        torch.cuda.empty_cache()


# ---- 7. capacity: a full-depth XXL shape -------------------------------------------------------------------------------

XXL = dict(vocab_size=32128, d_model=4096, num_heads=64, d_kv=64, d_ff=10240, num_layers=24, num_decoder_layers=24,
           feed_forward_proj="gated-gelu", tie_word_embeddings=False, relative_attention_num_buckets=32)


class LazyStateDict:
    """A t5-v1_1-xxl-shaped bf16 state_dict generated one tensor at a time on the GPU (seeded per key), so that no
    whole model is ever in memory; items() yields each tensor once"""

    def __init__(self, shapes, d):
        self.shapes, self.d = shapes, d

    def _make(self, i, k):
        import torch
        g = torch.Generator(device="cuda").manual_seed(i)
        shape = self.shapes[k]
        if len(shape) == 1:                                    # RMSNorm weights
            return torch.full(shape, 1.0 if "decoder.final" not in k else 0.02, dtype=torch.bfloat16, device="cuda")
        std = 1.0 if k == "lm_head.weight" else (1.0 / math.sqrt(shape[1]) if "relative" not in k else 0.1)
        return (torch.randn(shape, generator=g, device="cuda") * std).to(torch.bfloat16)

    def items(self):
        for i, k in enumerate(self.shapes):
            yield k, self._make(i, k)

    def get(self, k, default=None):
        return None                                            # untied: the engine never compares with shared


def xxl_shapes():
    c = XXL
    d, f, V, H = c["d_model"], c["d_ff"], c["vocab_size"], c["num_heads"]
    s = {"shared.weight": (V, d), "lm_head.weight": (V, d), "encoder.final_layer_norm.weight": (d,),
         "decoder.final_layer_norm.weight": (d,),
         "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (32, H),
         "decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (32, H)}
    for stack, n, subs in (("encoder", c["num_layers"], ["SelfAttention"]), ("decoder", c["num_decoder_layers"], ["SelfAttention", "EncDecAttention"])):
        for i in range(n):
            p = f"{stack}.block.{i}.layer."
            for j, a in enumerate(subs):
                for w in "qkvo":
                    s[f"{p}{j}.{a}.{w}.weight"] = (d, d)
                s[f"{p}{j}.layer_norm.weight"] = (d,)
            j = len(subs)
            s[f"{p}{j}.DenseReluDense.wi_0.weight"] = (f, d)
            s[f"{p}{j}.DenseReluDense.wi_1.weight"] = (f, d)
            s[f"{p}{j}.DenseReluDense.wo.weight"] = (d, f)
            s[f"{p}{j}.layer_norm.weight"] = (d,)
    return s


def test_full_depth_xxl_generates(corpus):
    import torch
    from transformers import T5Config
    from seal_b200.beam_search import SealT5Engine, generate_records
    want = device_bytes_formula("t5", (4096, 10240, 32128, 64, 24, 24, True, 32), 6, tied=False)
    free, _ = torch.cuda.mem_get_info()
    if free < want + (8 << 30):
        pytest.skip(f"{free / 2**30:.1f} GiB free on the shared card; the XXL engine needs {want / 2**30:.1f} GiB plus workspace")
    ora, idx, teos = corpus
    cfg = T5Config(dropout_rate=0.0, pad_token_id=PAD, eos_token_id=EOS, decoder_start_token_id=PAD, **XXL)
    cfg.forced_bos_token_id = None; cfg.forced_eos_token_id = None
    eng = SealT5Engine(LazyStateDict(xxl_shapes(), 4096), cfg, device=0, gemm_mode=6)
    torch.cuda.empty_cache()
    assert eng.device_bytes() == want
    print(f"XXL engine: {eng.device_bytes() / 1e9:.2f} GB of weights")
    assert eng.device_bytes() < 23e9
    ids, am = t5_sources(np.random.default_rng(2), 20, 16, 2000)
    rec = generate_records(eng, idx, ids, am, num_beams=15, min_length=10, max_length=10, length_penalty=0.0)
    assert eng.stat("overflow_fallbacks") == 0
    v = rec["valid"].astype(bool)
    assert v.any() and np.isfinite(rec["scores"][v]).all()
    assert eng.stat("last_paths") & BIT_BF16
    del eng
    torch.cuda.empty_cache()
