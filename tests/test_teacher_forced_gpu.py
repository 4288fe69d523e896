"""GPU: teacher-forced key scoring (sealdec_teacher_forced, target_logprob_kernel; seal_b200.keys.rescore_keys and
compute_unigram_scores) against float64, at the kernel's and the chunk loop's boundaries, plus its argument checks.

(a) target_logprob_kernel through sealdec_debug_target_logprob, against x32 = fp32(logit / temperature) (the fp32
    division torch and the kernel both perform) followed by a float64 log-softmax of x32.  The bound is derived from
    the kernel's arithmetic (see target_bound).
(b) sealdec_teacher_forced against transformers' BART cast to double, one forward over the decoder inputs with the
    encoder states gathered by row_query, with the criteria of test_bart_paths_gpu.py: equal finiteness pattern, an
    absolute bound, and err <= CAL_C * (fp32 HF's error) + CAL_FLOOR; plus the kernel branches each case must reach.
(c) rescore_keys / compute_unigram_scores against a float64 restatement of seal/keys.py:64-176.
(d) the error paths: fp16 overflow in the encoder or the decoder, bad out_full_pos, bad row_query, token ids outside
    [0, V) -- each rejected, with the engine still usable afterwards."""
import copy
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BITS = ["enc_packed", "enc_unpacked", "self_query", "self_rounds3", "self_rounds8", "self_long", "cross_small",
        "cross_grouped", "add_ln_row", "add_ln_warp", "splitk_deferred", "splitk_finish", "gemm_full_tile",
        "gemm_cluster", "gemm_tf32"]
ATTN_BITS = set(BITS[:10])
CAL_C = 8.0                  # the calibration of test_bart_paths_gpu.py
CAL_FLOOR = 1e-6
ABS_LOGPROB = {"tiny": 2e-5, "medium": 4e-5, "large": 4e-5}
KCHUNK = 4096                # decoder rows per pass of sealdec_teacher_forced
KADDLN_ROW_MAX = 2048
KXKEYS = 32
U = 2.0 ** -24               # fp32 unit roundoff


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32


# ---------------------------------------------------------------------------------------------------------------
# (a) target_logprob_kernel
# ---------------------------------------------------------------------------------------------------------------

def debug_target_logprob(logits, targets, temperature, ld=None, want_out=True, want_full=True, tgt_stride=1,
                         out_stride=1):
    """sealdec_debug_target_logprob on rows [R][V]; the stride gap ld - V holds NaN.  Returns (out, full): out as
    the kernel wrote it, [(R-1)*out_stride + 1] (gaps included), full [R][V]."""
    from seal_b200._lib import lib, check
    R, V = logits.shape
    ld = V if ld is None else ld
    buf = np.full((R, ld), np.nan, dtype=np.float32)
    buf[:, :V] = logits
    tg = np.full((R - 1) * tgt_stride + 1, -7, dtype=np.int64)
    tg[::tgt_stride] = targets
    out = np.empty((R - 1) * out_stride + 1, dtype=np.float32) if want_out else None
    full = np.empty((R, V), dtype=np.float32) if want_full else None
    check(lib.sealdec_debug_target_logprob(R, V, ld, buf.ctypes.data, tg.ctypes.data if want_out else None, tgt_stride,
                                           C.c_float(temperature), out.ctypes.data if want_out else None, out_stride,
                                           full.ctypes.data if want_full else None, V))
    return out, full


def ref_logprob(x32):
    """float64 log-softmax of the fp32 rows x32 (NaN anywhere in a row makes the row NaN, as in torch); also the row
    max M, the log-sum L and A = sum_i w_i (M - x_i) with w_i = exp(x_i - M) / sum exp, for the bound"""
    x = x32.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        M = x.max(axis=1, keepdims=True)
        z = x - M
        e = np.exp(z)
        tot = e.sum(axis=1, keepdims=True)
        L = np.log(tot)
        w = e / tot
        A = np.where(w > 0, w * -z, 0.0).sum(axis=1, keepdims=True)
        return z - L, M, L, A


def target_bound(x32, ref, M, L, A, V):
    """|kernel - ref| for a finite ref, from the kernel's arithmetic (decode_kernels.cuh target_logprob_kernel):
      - each of 256 threads keeps a running (max, rescaled sum) over n = ceil(V/256) terms: a term is multiplied by
        at most n - 1 later rescales expf(m_old - m_new) and finally by expf(mx - bm), so it passes through at most
        n + 1 expf calls (<= 2 ulp = 2^-22 relative each) and n multiplications; the thread sum adds n terms, then a
        5-level warp tree and an 8-term sequential block sum: 2n + 13 roundings of 2^-24 in all;
      - the expf arguments (each rounded to 2^-24 relative) telescope to x_i - M, so they add 2^-24 (M - x_i)
        relative to term i, 2^-24 * A relative to the sum;
      - so the sum is off by rho = (n+1) 2^-22 + (2n+13 + A) 2^-24 relative, and log(sum) by rho absolute, plus
        logf's 1 ulp (2^-23 |L|);
      - the output is fl(fl(x - M) - logsum): 2^-24 |x - M| + 2^-24 |out|.
    First-order terms, with 1 % slack for the second-order ones and subnormal underflow (<= V 2^-149 on a sum >= 1)."""
    n = -(-V // 256)
    rho = (n + 1) * 2.0 ** -22 + (2 * n + 13 + A) * U
    x = x32.astype(np.float64)
    with np.errstate(invalid="ignore"):
        return 1.01 * (rho + 2.0 ** -23 * np.abs(L) + U * np.abs(x - M) + U * np.abs(ref)) + 1e-30


ROW_KINDS = ["random", "ascending", "ties", "one_high", "neg_inf", "single", "all_neg_inf", "pos_inf", "nan_first",
             "nan_late"]


def make_rows(V, rng):
    """one row of each kind, each with 5 targets: -1, 0, V-1, V and a random in-range one (the row with target V is
    never the last one: the kernel must not read past the row)"""
    rows, kinds = [], []
    for kind in ROW_KINDS:
        r = (rng.standard_normal(V) * 4).astype(np.float32)
        if kind == "ascending":                    # every column a new running max: the rescale runs every time
            r = np.sort(r)
        elif kind == "ties":
            r[:] = 3.0
        elif kind == "one_high":
            r[:] = rng.standard_normal(V).astype(np.float32)
            r[int(rng.integers(V))] += 100.0
        elif kind == "neg_inf":                    # pad, bos and <mask> carry a -inf bias in SEAL's model
            r[[0, min(1, V - 1), V - 1]] = -np.inf
        elif kind == "single":
            r[:] = -np.inf
            r[int(rng.integers(V))] = 1.5
        elif kind == "all_neg_inf":
            r[:] = -np.inf
        elif kind == "pos_inf":
            r[int(rng.integers(V))] = np.inf
        elif kind == "nan_first":                  # thread 0's first column: ahead of any finite entry it sees
            r[0] = np.nan
        elif kind == "nan_late":
            r[V - 1] = np.nan
        for _ in range(5):
            rows.append(r); kinds.append(kind)
    targets = np.array([[-1, 0, V - 1, V, int(rng.integers(V))][i % 5] for i in range(len(rows))], dtype=np.int64)
    targets[-1] = 0
    return np.stack(rows), kinds, targets


def assert_matches(got, ref, bound, what):
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin), f"{what}: finiteness pattern differs"
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN pattern differs"
    assert np.array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)]), f"{what}: infinities differ"
    err = np.abs(got[fin].astype(np.float64) - ref[fin])
    worst = (err / bound[fin]).max() if err.size else 0.0
    assert worst <= 1.0, f"{what}: error / bound = {worst:.3f}"
    return worst


@pytest.mark.parametrize("temperature", [1.0, 0.7, 10.0, 1e-3])
@pytest.mark.parametrize("V", [1, 2, 255, 256, 257, 2000, 50265, 50272])
def test_target_logprob_kernel_vs_float64(V, temperature):
    rng = np.random.default_rng(V * 7 + int(temperature * 1000))
    logits, kinds, targets = make_rows(V, rng)
    R = len(logits)
    x32 = logits / np.float32(temperature)                 # the fp32 division of the reference and the kernel
    ref, M, L, A = ref_logprob(x32)
    bound = target_bound(x32, ref, M, L, A, V)
    ok_t = (targets >= 0) & (targets < V)
    ref_t = np.where(ok_t, ref[np.arange(R), np.clip(targets, 0, V - 1)], 0.0)
    bound_t = np.where(ok_t, bound[np.arange(R), np.clip(targets, 0, V - 1)], 1e-30)
    worst = 0.0
    for ld in (V, V + 5):                                 # V + 5: NaN in the stride gap, which must not be read
        out, full = debug_target_logprob(logits, targets, temperature, ld=ld)
        worst = max(worst, assert_matches(full, ref, bound, f"full ld={ld}"))
        worst = max(worst, assert_matches(out, ref_t, bound_t, f"out ld={ld}"))
        assert np.all(out[~ok_t] == 0.0) and not np.signbit(out[~ok_t]).any(), "out-of-range target must give 0.0"
        inr = np.nonzero(ok_t)[0]
        assert np.array_equal(out[inr].view(np.uint32), full[inr, targets[inr]].view(np.uint32)), "out != full[target]"
        single = [i for i, k in enumerate(kinds) if k == "single"]
        for i in single:
            assert full[i, np.argmax(np.isfinite(logits[i]))] == 0.0
        # each output alone, and the strided layout of sealdec_teacher_forced (targets at stride T, out at T - 1)
        out2, none = debug_target_logprob(logits, targets, temperature, ld=ld, want_full=False, tgt_stride=3, out_stride=2)
        assert none is None
        assert np.array_equal(out2[::2].view(np.uint32), out.view(np.uint32))
        assert np.isnan(out2[1::2]).all(), "the kernel wrote between the output stride"
        none, full2 = debug_target_logprob(logits, targets, temperature, ld=ld, want_out=False)
        assert none is None and np.array_equal(full2.view(np.uint32), full.view(np.uint32))
    print(f"V={V} T={temperature}: worst error / bound {worst:.3f}")


def test_debug_target_logprob_rejects_what_production_never_passes():
    from seal_b200._lib import lib, SealB200Error, check
    x = np.zeros((2, 8), dtype=np.float32)
    t = np.zeros(2, dtype=np.int64)
    out = np.zeros(2, dtype=np.float32)
    full = np.zeros((2, 8), dtype=np.float32)
    good = dict(R=2, V=8, ld=8, tgt_stride=1, temp=1.0, out_stride=1, full_ld=8, out=True, full=True)
    bad = [dict(ld=7), dict(temp=0.0), dict(temp=-1.0), dict(temp=float("inf")), dict(temp=float("nan")),
           dict(tgt_stride=0), dict(out_stride=0), dict(full_ld=7), dict(out=False, full=False), dict(R=0), dict(V=0)]
    call = lambda a: lib.sealdec_debug_target_logprob(a["R"], a["V"], a["ld"], x.ctypes.data, t.ctypes.data, a["tgt_stride"],
                                                      C.c_float(a["temp"]), out.ctypes.data if a["out"] else None,
                                                      a["out_stride"], full.ctypes.data if a["full"] else None, a["full_ld"])
    for b in bad:
        with pytest.raises(SealB200Error) as ei:
            check(call({**good, **b}))
        assert ei.value.code == -1, b
    check(call(good))
    assert np.allclose(out, -np.log(8.0)) and np.allclose(full, -np.log(8.0))


# ---------------------------------------------------------------------------------------------------------------
# (b) sealdec_teacher_forced against a float64 HF forward
# ---------------------------------------------------------------------------------------------------------------

_MODELS = {}
MODEL_KW = {"tiny": dict(layers=2, vocab=2000, d_model=128),
            "medium": dict(layers=2, vocab=5003, d_model=512),
            "large": dict()}


def get_model(name):
    """(fp64 HF on the GPU, fp32 HF on the GPU, our engine)"""
    if name not in _MODELS:
        import torch
        from oracle.decode_oracle import make_bart
        from seal_b200.beam_search import SealBartEngine
        for k in [k for k in _MODELS if "large" in (k, name)]:
            del _MODELS[k]
        torch.cuda.empty_cache()
        m32 = make_bart(seed=0, **MODEL_KW[name])
        eng = SealBartEngine(m32.state_dict(), m32.config, device=0, gemm_mode=3)
        m64 = copy.deepcopy(m32).double().cuda().eval()
        _MODELS[name] = (m64, m32.cuda().eval(), eng)
    return _MODELS[name]


def hf_logprobs(model, ids, am, dec, rq, full_pos=-1, temperature=1.0, chunk=None):
    """float64 log-probs of `model` (its own dtype up to the logits): one forward over dec[:, :T] per row chunk with
    the encoder states of row_query.  Returns (lp [N][T-1] of the targets dec[:, 1:], full [N][V] at full_pos)."""
    import torch
    from transformers.modeling_outputs import BaseModelOutput
    dev = next(model.parameters()).device
    N, T = dec.shape
    V = model.config.vocab_size
    chunk = chunk or max(16, min(1024, (1 << 27) // (T * V)))
    lps, fulls = [], []
    with torch.inference_mode():
        ids_t = torch.as_tensor(ids, device=dev); am_t = torch.as_tensor(am, device=dev)
        enc = model.get_encoder()(input_ids=ids_t, attention_mask=am_t).last_hidden_state
        rq_t = torch.as_tensor(np.asarray(rq, dtype=np.int64), device=dev)
        dec_t = torch.as_tensor(dec, device=dev)
        upto = T if full_pos == T - 1 else T - 1
        for r0 in range(0, N, chunk):
            s = rq_t[r0:r0 + chunk]
            lg = model(encoder_outputs=BaseModelOutput(last_hidden_state=enc[s]), attention_mask=am_t[s],
                       decoder_input_ids=dec_t[r0:r0 + chunk, :upto], use_cache=False).logits.double()
            lsm = torch.log_softmax(lg / temperature, -1)
            if T > 1:
                lps.append(torch.gather(lsm[:, :T - 1], -1, dec_t[r0:r0 + chunk, 1:].unsqueeze(-1)).squeeze(-1).cpu())
            if full_pos >= 0:
                fulls.append(lsm[:, full_pos].cpu())
    lp = torch.cat(lps).numpy() if lps else np.zeros((N, 0))
    return lp, (torch.cat(fulls).numpy() if fulls else None)


def sources(rng, Q, S, V, kind):
    """Q sources of S positions; query 0 is full length.  kind 'right': right-padded (packed encoder); 'holes': pad
    ids inside the source as well, masked as keys.py's _pad_inputs masks them (unpacked encoder)."""
    ids = rng.integers(4, V - 1, size=(Q, S)).astype(np.int64)
    ids[:, 0] = 0
    for q in range(Q):
        l = S if q == 0 else int(rng.integers(max(3, S // 2), S + 1))
        ids[q, l - 1] = 2
        ids[q, l:] = 1
        if kind == "holes" and l >= 4:
            ids[q, rng.choice(np.arange(1, l - 1), size=max(1, (l - 2) // 4), replace=False)] = 1
    return ids, (ids != 1).astype(np.int64)


def keys_for(rng, counts, T, V):
    """decoder rows: decoder_start 2, then 1 .. T-1 key tokens, right-padded with pad 1; the last row of every
    group has the full length T"""
    N = int(sum(counts))
    dec = np.ones((N, T), dtype=np.int64)
    dec[:, 0] = 2
    lens = rng.integers(1, T, size=N) if T > 1 else np.zeros(N, dtype=np.int64)
    ends = np.cumsum(counts)
    lens[ends[np.asarray(counts) > 0] - 1] = T - 1
    for r in range(N):
        dec[r, 1:1 + lens[r]] = rng.integers(4, V - 1, size=lens[r])
    rq = np.repeat(np.arange(len(counts)), counts).astype(np.int32)
    return dec, rq


def expected_bits(am, N, T, full_pos):
    Q, S = am.shape
    right = all(list(row) == sorted(row, reverse=True) for row in am.tolist())
    bits = {"enc_packed" if right else "enc_unpacked"}
    rows_enc = int(am.sum()) if right else Q * S
    for rows in [rows_enc] + [min(KCHUNK, N - r0) for r0 in range(0, N, KCHUNK)]:
        bits.add("add_ln_row" if rows <= KADDLN_ROW_MAX else "add_ln_warp")
    bits.add("cross_small" if S <= KXKEYS else "cross_grouped")
    for p in list(range(T - 1)) + ([T - 1] if full_pos == T - 1 else []):
        bits.add("self_rounds3" if p + 1 <= 12 else "self_rounds8" if p + 1 <= 32 else "self_long")
    return bits


def paths(eng):
    v = eng.stat("last_paths")
    assert v >= 0 and v >> len(BITS) == 0, f"undocumented path bit in {v:#x}"
    return {n for i, n in enumerate(BITS) if v >> i & 1}


def calibrated(model, label, got, ref64, ref32):
    """the test_bart_paths_gpu.py criteria on log-probs; returns the per-element bound they establish"""
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isfinite(got), fin), f"{label}: finiteness pattern differs from float64"
    assert np.array_equal(np.isfinite(ref32), fin)
    if not fin.any():
        return 0.0
    e = np.abs(got[fin] - ref64[fin]).max()
    h = np.abs(ref32[fin] - ref64[fin]).max()
    print(f"{label}: ours {e:.2e}  fp32 HF {h:.2e}  ratio {e / max(h, 1e-30):.2f}")
    assert e < ABS_LOGPROB[model], (label, e)
    assert e <= CAL_C * h + CAL_FLOOR, (label, e, h)
    return min(ABS_LOGPROB[model], CAL_C * h + CAL_FLOOR)


# (name, model, Q, S, kind, T, counts, full_pos, gemm_mode, must)
TF_CASES = [
    ("N1", "tiny", 1, 12, "right", 5, [1], 0, 3, set()),
    # ragged groups of 33, 1, 16 and 17 rows (cross_attn_small_kernel loops over 16-row blocks), empty queries at the
    # start, in the middle and at the end; 2 048 rows: add+LN one CTA per row; position 12 (P = 13) on full_pos = T-1
    ("N2048_S32_T13", "tiny", 8, 32, "right", 13, [0, 33, 1, 0, 16, 17, 1981, 0], 12, 3,
     {"cross_small", "self_rounds8", "add_ln_row"}),
    ("N2049_S33", "tiny", 7, 33, "holes", 3, [0, 1, 16, 0, 17, 2015, 0], 1, 3, {"cross_grouped", "add_ln_warp"}),
    ("N4096_one_group", "tiny", 2, 32, "right", 2, [4096, 0], 0, 3, {"cross_small"}),
    # query 3's keys straddle row 4 096: the second pass starts inside its group
    ("N4097_straddle", "tiny", 5, 33, "holes", 4, [0, 1, 4090, 6, 0], 3, 3, {"cross_grouped"}),
    ("N6145_straddle", "tiny", 6, 32, "right", 3, [0, 3000, 0, 1500, 1645, 0], 1, 3, {"cross_small", "add_ln_warp"}),
    # key lengths across the self-attention thresholds (12 / 32 keys) up to kMaxLen = 128
    ("T12", "tiny", 3, 20, "right", 12, [5, 0, 7], 11, 3, {"self_rounds3"}),
    ("T33", "tiny", 3, 20, "holes", 33, [5, 0, 7], 32, 3, {"self_rounds8", "self_long"}),    # P = 33 via full_pos
    ("T128", "tiny", 3, 20, "right", 128, [3, 0, 4], 127, 3, {"self_long"}),
    # GEMM modes on one mid-size case
    ("med_mode3", "medium", 4, 40, "holes", 6, [60, 0, 100, 40], 2, 3, {"gemm_full_tile"}),
    ("med_mode2", "medium", 4, 40, "holes", 6, [60, 0, 100, 40], 2, 2, {"gemm_tf32"}),
    ("med_mode5", "medium", 4, 40, "holes", 6, [60, 0, 100, 40], 2, 5, {"gemm_cluster"}),
    # bart-large, ~300 keys of two queries, V = 50 265
    ("large_300", "large", 2, 24, "right", 6, [150, 150], 2, 3, set()),
]
assert all(c[2] == len(c[6]) for c in TF_CASES)


@pytest.mark.parametrize("name,model,Q,S,kind,T,counts,full_pos,gemm_mode,must", TF_CASES, ids=[c[0] for c in TF_CASES])
def test_teacher_forced_vs_float64(name, model, Q, S, kind, T, counts, full_pos, gemm_mode, must):
    from seal_b200.keys import _teacher_forced
    m64, m32, eng = get_model(model)
    V = int(eng.config.vocab_size)
    rng = np.random.default_rng(len(name) * 31 + T)
    ids, am = sources(rng, Q, S, V, kind)
    dec, rq = keys_for(rng, counts, T, V)
    N = len(dec)
    if gemm_mode != 3:
        eng.set_option("gemm_mode", gemm_mode)
    try:
        lp, full = _teacher_forced(eng, ids, am, dec, rq, 1.0, full_pos)
        got = paths(eng)
    finally:
        if gemm_mode != 3:
            eng.set_option("gemm_mode", 3)
    want = expected_bits(am, N, T, full_pos)
    assert got & ATTN_BITS == want, (sorted(got & ATTN_BITS), sorted(want))
    assert must <= got, (sorted(must), sorted(got))
    if gemm_mode == 2:
        assert "gemm_full_tile" not in got
    if full_pos < T - 1:                                  # the target log-probs are the full vector's entries
        r = np.arange(N)
        assert np.array_equal(lp[:, full_pos].view(np.uint32), full[r, dec[r, full_pos + 1]].view(np.uint32))
    lp64, full64 = hf_logprobs(m64, ids, am, dec, rq, full_pos)
    lp32, full32 = hf_logprobs(m32, ids, am, dec, rq, full_pos)
    label = f"{name} N={N} T={T} S={S} {kind} mode={gemm_mode}"
    calibrated(model, label + " targets", lp, lp64, lp32)
    calibrated(model, label + f" full@{full_pos}", full, full64, full32)


def test_teacher_forced_key_length_limit():
    from seal_b200._lib import SealB200Error
    from seal_b200.keys import _teacher_forced
    _, _, eng = get_model("tiny")
    rng = np.random.default_rng(1)
    ids, am = sources(rng, 2, 8, 2000, "right")
    dec, rq = keys_for(rng, [2, 1], 129, 2000)
    with pytest.raises(SealB200Error) as ei:
        _teacher_forced(eng, ids, am, dec, rq)
    assert ei.value.code == -1
    _teacher_forced(eng, ids, am, dec[:, :128], rq)


# ---------------------------------------------------------------------------------------------------------------
# (c) rescore_keys / compute_unigram_scores against a float64 restatement of seal/keys.py:64-176
# ---------------------------------------------------------------------------------------------------------------

def rescore64(m64, m32, inputs, keys, length_penalty=0.0, prefix=(), strip_from_bos=(), strip_from_eos=()):
    """keys.py:64-141 in float64 (oracle/keys_oracle.py's steps, without its fp32 cast).  Returns, per query, a list of
    (score, key, bound): bound = sum over the counted positions of the per-position bound of (b), plus the fp32
    summation error gamma_T sum |lp| and the division's rounding."""
    from oracle.keys_oracle import strip
    cfg = m64.config
    maxlen = max(len(i) for i in inputs)
    ids = np.array([list(i) + [cfg.pad_token_id] * (maxlen - len(i)) for i in inputs], dtype=np.int64)
    am = (ids != cfg.pad_token_id).astype(np.int64)
    keys = [[x[1] if isinstance(x[0], float) else x for x in xx] for xx in keys]
    rows, rq, orig = [], [], []
    for q, kk in enumerate(keys):
        for di in kk:
            rows.append([cfg.decoder_start_token_id] + list(prefix) + strip(list(di), strip_from_bos, strip_from_eos))
            rq.append(q); orig.append(list(di))
    T = max(len(r) for r in rows)
    dec = np.full((len(rows), T), cfg.pad_token_id, dtype=np.int64)
    for r, toks in enumerate(rows):
        dec[r, :len(toks)] = toks
    lp64, _ = hf_logprobs(m64, ids, am, dec, rq)
    lp32, _ = hf_logprobs(m32, ids, am, dec, rq)
    counted = (dec[:, 1:] >= 2) & (np.arange(T - 1) >= len(prefix))
    fin = np.isfinite(lp64) & counted
    h = np.abs(lp32[fin] - lp64[fin]).max()
    b = min(ABS_LOGPROB["tiny"], CAL_C * h + CAL_FLOOR)
    out = [[] for _ in keys]
    for r in range(len(rows)):
        c = counted[r]
        s = lp64[r, c].sum()
        g = (T * U) / (1 - T * U)
        den = len(orig[r]) ** length_penalty
        bound = (c.sum() * b + g * np.abs(lp64[r, c]).sum()) / den
        s = s / den
        out[rq[r]].append((s, orig[r], bound + U * abs(s) if np.isfinite(s) else 0.0))
    return out


def keys_case(rng, V):
    """6 sources (one with a pad id inside it: a mask hole), keys of 0 .. 12 per query with leading bos / trailing
    eos, bos or pad in the middle, token V-1 (<mask>, -inf bias), and the (score, key) form"""
    inputs = [[0] + rng.integers(4, V - 1, size=int(rng.integers(3, 14))).tolist() + [2] for _ in range(6)]
    inputs[3][2] = 1
    keys = []
    for q in range(6):
        kk = []
        for j in range(int(rng.integers(0, 13)) if q not in (0, 4) else (0 if q == 4 else 12)):
            toks = rng.integers(4, V - 1, size=int(rng.integers(1, 9))).tolist()
            u = rng.random()
            if u < 0.2: toks = [0] + toks
            if u > 0.7: toks = toks + [2]
            if j == 1: toks = toks[:1] + [V - 1] + toks[1:]
            if j == 2: toks = toks[:1] + [0] + toks[1:] + [5]
            if j == 3: toks = toks[:1] + [1] + toks[1:] + [6]
            kk.append((float(rng.random()), toks) if j % 2 else toks)
        keys.append(kk)
    return inputs, keys


@pytest.mark.parametrize("kw", [dict(), dict(length_penalty=1.0), dict(prefix=[7, 9]),
                                dict(strip_from_bos=[0], strip_from_eos=[2])],
                         ids=["plain", "length_penalty", "prefix", "strip"])
def test_rescore_keys_vs_float64(kw):
    from seal_b200.keys import rescore_keys
    m64, m32, eng = get_model("tiny")
    V = int(eng.config.vocab_size)
    inputs, keys = keys_case(np.random.default_rng(21), V)
    got = rescore_keys(eng, inputs, keys, **kw)
    assert "enc_unpacked" in paths(eng)                  # the pad id inside source 3 is a mask hole
    exp = rescore64(m64, m32, inputs, keys, **kw)
    n_inf = worst = 0
    for a, b in zip(got, exp):
        assert [k for _, k in a] == [k for _, k, _ in b]
        for (sa, k), (sb, _, bound) in zip(a, b):
            if not np.isfinite(sb):
                assert sa == sb, (k, sa, sb)
                n_inf += 1
                continue
            assert abs(sa - sb) <= bound, (k, sa, sb, bound)
            worst = max(worst, abs(sa - sb) / bound)
    assert n_inf >= 1, "no key with token V-1 scored"
    print(f"rescore {kw}: worst error / bound {worst:.3f}, {n_inf} keys at -inf")


@pytest.mark.parametrize("kw", [dict(temperature=0.7), dict(prefix=[11, 13])], ids=["temperature", "prefix"])
def test_unigram_scores_4097_queries_vs_float64(kw):
    """Q = 4 097 one-row groups: two passes of the chunk loop, the second one row long."""
    from seal_b200.keys import compute_unigram_scores
    m64, m32, eng = get_model("tiny")
    cfg = eng.config
    V = int(cfg.vocab_size)
    rng = np.random.default_rng(33)
    inputs = [[0] + rng.integers(4, V - 1, size=int(rng.integers(2, 20))).tolist() + [2] for _ in range(4097)]
    got = compute_unigram_scores(eng, inputs, tolist=False, **kw)
    prefix = kw.get("prefix", [])
    maxlen = max(len(i) for i in inputs)
    ids = np.array([i + [1] * (maxlen - len(i)) for i in inputs], dtype=np.int64)
    am = (ids != 1).astype(np.int64)
    dec = np.array([[2] + prefix] * len(inputs), dtype=np.int64)
    t = kw.get("temperature", 1.0)
    _, f64 = hf_logprobs(m64, ids, am, dec, np.arange(len(inputs)), full_pos=len(prefix), temperature=t)
    _, f32 = hf_logprobs(m32, ids, am, dec, np.arange(len(inputs)), full_pos=len(prefix), temperature=t)
    calibrated("tiny", f"unigram Q=4097 {kw}", got, f64, f32)


# ---------------------------------------------------------------------------------------------------------------
# (d) errors
# ---------------------------------------------------------------------------------------------------------------

def scaled_model(param):
    """the tiny model with one fc1 weight scaled by 2e6: its activations leave the fp16 range (|x| > 65504)"""
    import torch
    from oracle.decode_oracle import make_bart
    from seal_b200.beam_search import SealBartEngine
    m32 = make_bart(seed=0, **MODEL_KW["tiny"])
    with torch.no_grad():
        dict(m32.named_parameters())[param].mul_(2e6)
    eng = SealBartEngine(m32.state_dict(), m32.config, device=0, gemm_mode=3)
    return copy.deepcopy(m32).double().cuda().eval(), m32.cuda().eval(), eng


@pytest.mark.parametrize("param", ["model.encoder.layers.0.fc1.weight", "model.decoder.layers.0.fc1.weight"],
                         ids=["encoder", "decoder"])
def test_teacher_forced_fp16_overflow_raises(param):
    """An activation past the fp16 range makes the 3xFP16 path saturate: the call must report it rather than return
    log-probs computed from saturated values.  The encoder's flag used to be cleared after the encoder ran."""
    from seal_b200._lib import SealB200Error
    from seal_b200.keys import _teacher_forced
    m64, m32, eng = scaled_model(param)
    rng = np.random.default_rng(4)
    ids, am = sources(rng, 3, 16, 2000, "right")
    dec, rq = keys_for(rng, [4, 3, 5], 6, 2000)
    lp64, _ = hf_logprobs(m64, ids, am, dec, rq)
    lp32, _ = hf_logprobs(m32, ids, am, dec, rq)
    try:
        lp, _ = _teacher_forced(eng, ids, am, dec, rq)
    except SealB200Error as e:
        assert e.code == -1 and "fp16 range" in str(e)
    else:
        fin = np.isfinite(lp64)
        err = np.abs(lp[fin] - lp64[fin]).max() if np.array_equal(np.isfinite(lp), fin) else np.inf
        pytest.fail(f"fp16 overflow not reported; the returned log-probs are off float64 by {err:.3e}")
    # the remedy the error names: gemm_mode 2 (3xTF32, fp32 range) gives float64's results
    eng.set_option("gemm_mode", 2)
    lp, _ = _teacher_forced(eng, ids, am, dec, rq)
    fin = np.isfinite(lp64)
    assert np.array_equal(np.isfinite(lp), fin)
    e, h = np.abs(lp[fin] - lp64[fin]).max(), np.abs(lp32[fin] - lp64[fin]).max()
    print(f"{param} x 2e6, 3xTF32: ours {e:.2e} fp32 HF {h:.2e}")
    assert e <= CAL_C * h + CAL_FLOOR


def test_teacher_forced_bad_out_full_pos_rejected():
    """out_full with out_full_pos outside [0, T) used to copy a never-written buffer back and return success."""
    from seal_b200._lib import lib, SealB200Error, check
    _, _, eng = get_model("tiny")
    rng = np.random.default_rng(8)
    ids, am = sources(rng, 2, 10, 2000, "right")
    dec, rq = keys_for(rng, [3, 2], 4, 2000)
    out = np.zeros((5, 3), dtype=np.float32)
    full = np.zeros((5, 2000), dtype=np.float32)
    for pos in (-1, 4, 9):
        with pytest.raises(SealB200Error) as ei:
            check(lib.sealdec_teacher_forced(eng._h, ids.ctypes.data, am.ctypes.data, 2, 10, dec.ctypes.data,
                                             rq.ctypes.data, 5, 4, C.c_float(1.0), out.ctypes.data, pos, full.ctypes.data))
        assert ei.value.code == -1 and "out_full_pos" in str(ei.value), pos
    check(lib.sealdec_teacher_forced(eng._h, ids.ctypes.data, am.ctypes.data, 2, 10, dec.ctypes.data, rq.ctypes.data,
                                     5, 4, C.c_float(1.0), out.ctypes.data, -1, None))       # no full vector: any pos
    check(lib.sealdec_teacher_forced(eng._h, ids.ctypes.data, am.ctypes.data, 2, 10, dec.ctypes.data, rq.ctypes.data,
                                     5, 4, C.c_float(1.0), out.ctypes.data, 3, full.ctypes.data))
    assert np.isfinite(full[:, 2:-1]).all()


BAD_IDS = [-1, 2000, 2 ** 32 + 5]


def test_bad_row_query_and_token_ids_rejected():
    """Each bad input gives SEALFM_EINVAL before any launch (an out-of-range id would index the embedding table
    unchecked), and the engine still returns the same results afterwards."""
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import generate_records
    from seal_b200.keys import _teacher_forced, rescore_keys
    _, _, eng = get_model("tiny")
    rng = np.random.default_rng(9)
    ids, am = sources(rng, 2, 10, 2000, "right")
    dec, rq = keys_for(rng, [3, 2], 4, 2000)
    base, _ = _teacher_forced(eng, ids, am, dec, rq)
    inputs = [list(r[:int(m.sum())]) for r, m in zip(ids, am)]
    keys = [[[5, 6, 7], [8]], [[9, 10]]]
    base_keys = rescore_keys(eng, inputs, keys)
    gen = lambda i: generate_records(eng, None, i, am, num_beams=2, max_length=3, disable_fm_index=True)
    base_gen = gen(ids)

    def rejected(call):
        with pytest.raises(SealB200Error) as ei:
            call()
        assert ei.value.code == -1

    for bad in ([1, 0, 0, 1, 1], [0, 0, 0, 1, -1], [0, 0, 0, 1, 2]):      # unsorted, -1, Q
        rejected(lambda: _teacher_forced(eng, ids, am, dec, np.array(bad, dtype=np.int32)))
    for v in BAD_IDS:
        d2 = dec.copy(); d2[3, 2] = v
        rejected(lambda: _teacher_forced(eng, ids, am, d2, rq))                          # key token
        i2 = ids.copy(); i2[1, 3] = v
        rejected(lambda: _teacher_forced(eng, i2, am, dec, rq))                          # source token
        rejected(lambda: rescore_keys(eng, inputs, [[[5, v, 7]], [[9]]]))                # key via rescore_keys
        rejected(lambda: rescore_keys(eng, inputs, keys, prefix=[v]))                     # prefix
        rejected(lambda: gen(i2))                                                          # sealdec_generate's input_ids
        rejected(lambda: eng.debug_step_logits(i2, am, 1, dec[[0, 3]]))
        rejected(lambda: eng.debug_step_logits(ids, am, 1, d2[[0, 3]]))
    after, _ = _teacher_forced(eng, ids, am, dec, rq)
    assert np.array_equal(after.view(np.uint32), base.view(np.uint32))
    assert rescore_keys(eng, inputs, keys) == base_keys
    g = gen(ids)
    assert all(np.array_equal(g[k], base_gen[k]) for k in ("scores", "lens", "tokens", "valid"))
