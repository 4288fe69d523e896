"""GPU: every kernel branch of the BART forward (seal_b200/csrc/forward.cu: encoder_forward, decoder_step, add_ln;
gemm.cu: gemm_impl) against a float64 forward of the same seeded HF model, at the shapes where they switch branches.

The float64 reference is transformers' BartForConditionalGeneration cast to double (the fp32 weights convert exactly),
re-forwarded over the whole decoder prefix (use_cache=False).  The same model in fp32 runs on the same inputs: its own
error against float64 is the yardstick of what fp32 arithmetic achieves at that shape.  Every case asserts
  - the finiteness pattern of the logits equals the reference's,
  - an absolute bound (the figures of test_decode_gpu.py: 2e-5 on the tiny model's logits, 4e-5 on log-probs above),
  - a calibrated bound: our error <= CAL_C * (fp32 HF's error) + CAL_FLOOR, which catches a branch that is merely
    less accurate than fp32 arithmetic,
  - the kernel branches the call takes (sealbart_get_stat "last_paths", include/sealdec.h), restated from the shapes.
    last_paths is the OR over every decoder position of the call, so a case proves which side of a threshold its
    last position took only where that adds a bit.  That holds for every threshold here except the shared-memory
    limit of dec_self_attn_query_kernel at B = 32: P = 7, the first position past it, takes dec_self_attn_kernel<3>,
    which position 0 of every call takes as well.  Both sides are still compared with float64 there."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BITS = ["enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
        "cross_grouped", "add_ln_row", "add_ln_warp", "splitk_deferred", "splitk_finish", "gemm_full_tile",
        "gemm_cluster", "gemm_tf32"]
ATTN_BITS = set(BITS[:10])          # fully determined by the shapes: asserted exactly; the GEMM bits as a subset

# Calibration, measured on an H100 80 GB HBM3 (700 W): over this grid our max |dlogit| was 1.4 .. 3.7 times fp32 HF's
# on the tiny model (7.3 at B = 1, P = 2, where HF's own error was only 1.5e-7), 1.6 .. 4.9 times on the d = 512 model
# and 2.4 times on bart-large; HF's own error ranged 1.5e-7 .. 6e-6.  Both sides are deterministic for fixed inputs, so
# the bound is not there for noise: c = 8 with a floor of 1e-6 passes every case by >= 1.7x and still fails a branch
# that is several times less accurate than the rest of the forward.
CAL_C = 8.0
CAL_FLOOR = 1e-6
ABS_LOGIT = {"tiny": 2e-5, "tiny_lowvar": 2e-5}
ABS_LOGPROB = {"medium": 4e-5, "large": 4e-5}

SAQ_SMEM_MAX = 112 * 1024
KADDLN_ROW_MAX = 2048
KXKEYS = 32


def saq_smem(P, B):
    """self_attn_query_smem (bart_kernels.cuh): K and V head rows of every (position, beam), two [P][32] int tables,
    128 ints."""
    return 2 * P * B * 64 * 4 + 2 * P * 32 * 4 + 128 * 4


def saq_limit(B):
    """largest P that dec_self_attn_query_kernel takes at B beams"""
    P = 1
    while P + 1 <= 128 and saq_smem(P + 1, B) <= SAQ_SMEM_MAX:
        P += 1
    return P


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32        # fp32 HF must be real fp32


_MODELS = {}
MODEL_KW = {"tiny": dict(layers=2, vocab=2000, d_model=128),
            "medium": dict(layers=2, vocab=5003, d_model=512),       # K = 512 / 2048: the small-row GEMMs split K
            "tiny_lowvar": dict(layers=2, vocab=2000, d_model=128),
            "large": dict()}                                        # BartConfig() = bart-large
# "tiny_lowvar": every LayerNorm weight scaled by 2^-5, so the rows entering add+LayerNorm have a variance of ~1e-3 and
# its eps (1e-5) moves the result by ~0.5 %, well above the rounding noise: a wrong eps cannot hide
LOWVAR_GAMMA = 2.0 ** -5


def get_model(name):
    """(fp64 HF on the GPU, fp32 HF on the GPU, our engine)"""
    if name not in _MODELS:
        import copy
        import torch
        from oracle.decode_oracle import make_bart
        from seal_b200.beam_search import SealBartEngine
        for k in [k for k in _MODELS if "large" in (k, name)]:     # bart-large alone on the device
            del _MODELS[k]
        torch.cuda.empty_cache()
        m32 = make_bart(seed=0, **MODEL_KW[name])
        if name == "tiny_lowvar":
            with torch.no_grad():
                for mod in m32.modules():
                    if isinstance(mod, torch.nn.LayerNorm):
                        mod.weight.mul_(LOWVAR_GAMMA)
        eng = SealBartEngine(m32.state_dict(), m32.config, device=0, gemm_mode=3)
        m64 = copy.deepcopy(m32).double().cuda().eval()
        _MODELS[name] = (m64, m32.cuda().eval(), eng)
    return _MODELS[name]


def hf_logits(model, ids, am, B, dec, rows=None):
    """last-position logits of `model` (its dtype) as float64 numpy; rows: source row of each decoder row
    (default: query-major, B beams per query)"""
    import torch
    from transformers.modeling_outputs import BaseModelOutput
    dev = next(model.parameters()).device
    with torch.inference_mode():
        ids_t = torch.as_tensor(ids, device=dev); am_t = torch.as_tensor(am, device=dev)
        enc = model.get_encoder()(input_ids=ids_t, attention_mask=am_t).last_hidden_state
        sel = torch.as_tensor(rows, device=dev) if rows is not None else torch.arange(len(ids), device=dev).repeat_interleave(B)
        out = []
        for r0 in range(0, len(dec), 1024):
            s = sel[r0:r0 + 1024]
            o = model(encoder_outputs=BaseModelOutput(last_hidden_state=enc[s]), attention_mask=am_t[s],
                      decoder_input_ids=torch.as_tensor(dec[r0:r0 + 1024], device=dev), use_cache=False)
            out.append(o.logits[:, -1, :].double().cpu())
    return torch.cat(out).numpy()


def src_inputs(rng, Q, S, vocab, kind="right"):
    """make_inputs (test_decode_gpu.py) for any S >= 1, with query 0 always full length (the last key of a block
    is live).  kind: 'right' padding, 'holes' (masked positions inside the source), 'left' padding."""
    ids = rng.integers(4, vocab, size=(Q, S)).astype(np.int64)
    am = np.ones((Q, S), dtype=np.int64)
    ids[:, 0] = 0
    for q in range(Q):
        l = S if q == 0 else int(rng.integers(min(max(3, S // 2), S), S + 1))
        ids[q, l - 1] = 2
        ids[q, l:] = 1
        am[q, l:] = 0
        if kind == "holes" and l >= 3:
            am[q, rng.choice(np.arange(1, l - 1), size=max(1, (l - 2) // 4), replace=False)] = 0
        if kind == "left" and l < S:
            ids[q] = np.roll(ids[q], S - l); am[q] = np.roll(am[q], S - l)
    return ids, am


def beam_inputs(rng, Q, B, t, vocab, share):
    """decoder inputs [Q*B, t] (decoder_start 2, then random tokens); share: beam b copies the first k tokens of an
    earlier beam of its query (random k), so beams share prefixes of every length, as in a beam search.  Returns
    (dec, anc) with anc[r][s] = the lowest row of r's query whose dec[:s+1] equals row r's (None without sharing)."""
    dec = rng.integers(4, vocab, size=(Q * B, t)).astype(np.int64)
    dec[:, 0] = 2
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


def expected_attn_bits(Q, S, B, t, am, src_tokens):
    """the shape-determined branches of one debug step call (forward.cu, gemm.cu), restated"""
    bits = set()
    right = all(list(row) == sorted(row, reverse=True) for row in am.tolist())
    packed = right and src_tokens != -2
    bits.add("enc_packed" if packed else "enc_unpacked")
    rows_enc = int(am.sum()) if packed else Q * S
    for rows in (rows_enc, Q * B):
        bits.add("add_ln_row" if rows <= KADDLN_ROW_MAX else "add_ln_warp")
    bits.add("cross_small" if S <= KXKEYS else "cross_grouped")
    for pos in range(t):
        P = pos + 1
        if pos >= 1 and 2 <= B <= 32 and P <= 128 and saq_smem(P, B) <= SAQ_SMEM_MAX:
            bits.add("self_query")
        else:
            bits.add("self_rounds3" if P <= 12 else "self_rounds8" if P <= 32 else "self_long")
    return bits


def paths(eng):
    v = eng.stat("last_paths")
    assert v >= 0
    assert v >> len(BITS) == 0, f"undocumented path bit in {v:#x}"
    return {n for i, n in enumerate(BITS) if v >> i & 1}


def log_softmax(x):
    import torch
    return torch.log_softmax(torch.from_numpy(np.asarray(x, dtype=np.float64)), -1).numpy()


def errors(got, ref64, ref32):
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isfinite(got), fin), "finiteness pattern differs from float64"
    assert np.array_equal(np.isfinite(ref32), fin)
    lg, l64, l32 = log_softmax(got), log_softmax(ref64), log_softmax(ref32)
    return (np.abs(got[fin] - ref64[fin]).max(), np.abs(lg[fin] - l64[fin]).max(),
            np.abs(ref32[fin] - ref64[fin]).max(), np.abs(l32[fin] - l64[fin]).max())


def check_bounds(model, label, got, ref64, ref32):
    e, el, h, hl = errors(got, ref64, ref32)
    print(f"{label}: ours |dlogit| {e:.2e} |dlogprob| {el:.2e}   fp32 HF |dlogit| {h:.2e} |dlogprob| {hl:.2e}   "
          f"ratio {e / max(h, 1e-30):.2f}")
    if model in ABS_LOGIT:
        assert e < ABS_LOGIT[model], (label, e)
    if model in ABS_LOGPROB:
        assert el < ABS_LOGPROB[model], (label, el)
    assert e <= CAL_C * h + CAL_FLOOR, (label, e, h)
    return e


def run_case(model, Q, S, B, t, kind="right", src_tokens=-1, share=False, gemm_mode=3, must=(), seed=0, check=True):
    """one debug step (with and, if share, without ancestry), checked against float64; returns the paths taken"""
    m64, m32, eng = get_model(model)
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(seed)
    ids, am = src_inputs(rng, Q, S, V, kind)
    dec, anc = beam_inputs(rng, Q, B, t, V, share and B > 1 and t > 1)
    if gemm_mode != 3:
        eng.set_option("gemm_mode", gemm_mode)
    try:
        outs = []
        for a in ([anc, None] if anc is not None else [None]):
            outs.append(eng.debug_step_logits(ids, am, B, dec, anc=a, src_tokens=src_tokens))
            got_paths = paths(eng)
            want = expected_attn_bits(Q, S, B, t, am, src_tokens)
            assert got_paths & ATTN_BITS == want, (sorted(got_paths & ATTN_BITS), sorted(want))
            assert set(must) <= got_paths, (sorted(must), sorted(got_paths))
            if gemm_mode == 2:
                assert "gemm_tf32" in got_paths and "gemm_full_tile" not in got_paths
    finally:
        if gemm_mode != 3:
            eng.set_option("gemm_mode", 3)
    if not check:
        return got_paths
    ref64 = hf_logits(m64, ids, am, B, dec)
    ref32 = hf_logits(m32, ids, am, B, dec)
    label = f"{model} Q={Q} S={S} B={B} P={t} {kind} src={src_tokens} mode={gemm_mode}"
    check_bounds(model, label + (" anc" if anc is not None else ""), outs[0], ref64, ref32)
    if anc is not None:
        check_bounds(model, label + " identity", outs[1], ref64, ref32)
        tol = ABS_LOGIT.get(model) or ABS_LOGPROB[model]
        assert np.abs(outs[0] - outs[1])[np.isfinite(ref64)].max() < tol
    return got_paths


# (name, model, Q, S, B, P, kwargs): each case sits next to one threshold of forward.cu or gemm.cu and names the branches it needs
CASES = [
    # cross-attention: cross_attn_small_kernel up to kXKeys = 32 keys
    ("S1", "tiny", 3, 1, 2, 2, dict(share=True, must={"cross_small"})),
    ("S31", "tiny", 3, 31, 4, 3, dict(share=True, must={"cross_small"})),
    ("S32", "tiny", 3, 32, 4, 3, dict(share=True, must={"cross_small"})),
    ("S33", "tiny", 3, 33, 4, 3, dict(share=True, must={"cross_grouped"})),
    ("S64", "tiny", 2, 64, 3, 2, dict(share=True, must={"cross_grouped"})),
    # encoder: packed only for right-padded masks and hint != -2
    ("holes", "tiny", 3, 20, 3, 4, dict(kind="holes", share=True, must={"enc_unpacked"})),
    ("left", "tiny", 3, 40, 2, 3, dict(kind="left", share=True, must={"enc_unpacked", "cross_grouped"})),
    ("unpacked32", "tiny", 3, 32, 4, 2, dict(src_tokens=-2, must={"enc_unpacked", "cross_small"})),
    # self-attention one row per CTA (B = 1): <= 12, <= 32, longer
    *[(f"P{P}", "tiny", 2, 12, 1, P, dict(must={"self_rounds3"})) for P in (1, 2, 12, 13, 32, 33, 128)],
    # self-attention with the beams of a query together: both sides of its shared-memory limit
    # (at B = 32 both sides set the same bits: position 0 always takes dec_self_attn_kernel<3>, see the docstring)
    *[(f"B{B}_P{P}", "tiny", 2, 12, B, P, dict(share=True)) for B in (2, 15, 32)
      for P in (saq_limit(B), saq_limit(B) + 1)],
    # add + LayerNorm: one CTA per row up to kAddLnRowMax = 2048 rows (encoder rows <= 2048 as well)
    ("R2048", "tiny_lowvar", 128, 16, 16, 2, dict(must={"add_ln_row"})),
    ("R2049", "tiny_lowvar", 683, 3, 3, 2, dict(must={"add_ln_warp"})),
    ("R4000", "tiny_lowvar", 250, 12, 16, 3, dict(share=True, must={"add_ln_warp", "gemm_full_tile"})),
    # other GEMM modes
    ("mode5", "tiny", 250, 12, 16, 2, dict(gemm_mode=5, must={"gemm_cluster"})),
    ("mode2", "tiny", 3, 33, 4, 3, dict(gemm_mode=2, share=True, must={"gemm_tf32"})),
    # d = 512: the small-row GEMMs split K; the attention and add+LN kernels sum the slices themselves
    ("med_small", "medium", 2, 12, 4, 3, dict(share=True, must={"splitk_deferred", "splitk_finish", "self_query"})),
    ("med_long", "medium", 2, 40, 1, 13, dict(must={"splitk_deferred", "splitk_finish", "cross_grouped"})),
    ("med_B15", "medium", 2, 32, 15, 15, dict(share=True, must={"splitk_deferred", "self_rounds8"})),
    ("med_mode5", "medium", 24, 16, 8, 2, dict(gemm_mode=5, must={"gemm_cluster"})),
    # bart-large
    ("large_S33", "large", 2, 33, 3, 4, dict(share=True, must={"cross_grouped", "splitk_deferred"})),
    ("large_B15", "large", 2, 20, 15, 15, dict(share=True, must={"self_query", "self_rounds8", "cross_small"})),
]


@pytest.mark.parametrize("name,model,Q,S,B,P,kw", CASES, ids=[c[0] for c in CASES])
def test_forward_path_vs_float64(name, model, Q, S, B, P, kw):
    run_case(model, Q, S, B, P, **kw)


def test_every_path_reached():
    """The union of last_paths over the grid (bart-large left out: it adds no branch) is every defined bit."""
    seen = set()
    for name, model, Q, S, B, P, kw in CASES:
        if model != "large":
            seen |= run_case(model, Q, S, B, P, check=False, **kw)
    print("paths reached:", sorted(seen))
    assert seen == set(BITS), sorted(set(BITS) - seen)


def test_teacher_forced_ragged_groups_vs_float64():
    """sealdec_teacher_forced with ragged row groups larger than kXRows = 16 and sources longer than 32 positions:
    cross_attn_kernel with grp_start.  Full log-prob vector and the per-position target log-probs."""
    from seal_b200.keys import _teacher_forced
    m64, m32, eng = get_model("tiny")
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(5)
    ids, am = src_inputs(rng, 3, 40, V)
    counts = [20, 17, 25]
    rq = np.repeat(np.arange(3), counts).astype(np.int32)
    T, pos = 5, 2
    dec = rng.integers(4, V, size=(len(rq), T)).astype(np.int64); dec[:, 0] = 2
    lp, full = _teacher_forced(eng, ids, am, dec, rq, 1.0, pos)
    got_paths = paths(eng)
    assert {"cross_grouped", "self_rounds3"} <= got_paths and not {"self_query", "cross_small"} & got_paths
    ref64 = log_softmax(hf_logits(m64, ids, am, 1, dec[:, :pos + 1], rows=rq))
    ref32 = log_softmax(hf_logits(m32, ids, am, 1, dec[:, :pos + 1], rows=rq))
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isfinite(full), fin)
    e, h = np.abs(full[fin] - ref64[fin]).max(), np.abs(ref32[fin] - ref64[fin]).max()
    print(f"teacher-forced full log-probs: ours {e:.2e}, fp32 HF {h:.2e}")
    assert e < ABS_LOGIT["tiny"] and e <= CAL_C * h + CAL_FLOOR
    for p in range(T - 1):
        want = log_softmax(hf_logits(m64, ids, am, 1, dec[:, :p + 1], rows=rq))[np.arange(len(rq)), dec[:, p + 1]]
        assert np.abs(lp[:, p] - want).max() < ABS_LOGIT["tiny"], p


def test_all_zero_mask_source_rejected():
    """A source with nothing to attend to leaves the attention kernels' softmax denominator at zero (HF instead
    spreads the weight over the masked keys and gives finite logits).  The host-buffer entry points reject it."""
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import generate_records
    from seal_b200.keys import _teacher_forced
    _, m32, eng = get_model("tiny")
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(6)
    ids, am = src_inputs(rng, 2, 10, V)
    am[1] = 0
    dec, _ = beam_inputs(rng, 2, 2, 3, V, False)
    for call in (lambda: eng.debug_step_logits(ids, am, 2, dec),
                 lambda: eng.debug_step_logits(ids, am, 2, dec, src_tokens=-2),
                 lambda: _teacher_forced(eng, ids, am, dec[::2], np.arange(2, dtype=np.int32), 1.0, 1),
                 lambda: generate_records(eng, None, ids, am, num_beams=2, max_length=3, disable_fm_index=True)):
        with pytest.raises(SealB200Error) as ei:
            call()
        assert ei.value.code == -1 and "all-zero attention mask" in str(ei.value)


def test_debug_step_arguments_checked():
    from seal_b200._lib import SealB200Error
    _, _, eng = get_model("tiny")
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(7)
    ids, am = src_inputs(rng, 2, 10, V)
    dec, anc = beam_inputs(rng, 2, 3, 4, V, True)
    bad = anc.copy(); bad[4, 2] = 6                      # R = 6 rows
    with pytest.raises(SealB200Error):
        eng.debug_step_logits(ids, am, 3, dec, anc=bad)
    with pytest.raises(SealB200Error):                    # a token count that does not match the mask
        eng.debug_step_logits(ids, am, 3, dec, src_tokens=int(am.sum()) + 1)
    a = eng.debug_step_logits(ids, am, 3, dec, src_tokens=int(am.sum()))
    assert "enc_packed" in paths(eng)
    b = eng.debug_step_logits(ids, am, 3, dec, anc=anc, src_tokens=-2)
    assert "enc_unpacked" in paths(eng)
    assert np.abs(a - b)[np.isfinite(a)].max() < ABS_LOGIT["tiny"]
