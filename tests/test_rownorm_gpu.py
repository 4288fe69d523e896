"""GPU: the producers that normalise or gate a row and write the next GEMM's split operand (BART embedding + LN, add+LN
in its CTA-per-row and warp-per-row forms, T5 RMSNorm in both widths, the pre-LayerNorm row, the T5 gate), one at a time
through sealdec_debug_rownorm -- the layer loops' own launchers -- against rownorm_ref.py's float64 reference and its
running-error bound, on crafted row sets at the dispatch boundaries; and BART's position-table limit end to end.

Exact checks: the residual each kernel writes; beta from constant rows; every element written (outputs start as NaN);
the split pieces equal the host splitters applied to the fp32 value, which is the same in every split instantiation;
the fp16 range flag at 65 504; the last_paths bit of the kernel that ran."""
import ctypes as C

import numpy as np
import pytest

import rownorm_ref as R
from test_gemm_split_out_host import HALF_MAX, split_half

pytestmark = pytest.mark.gpu

ROW, WARP, T5, T5_GATE, T5_WIDE, PRELN, PRELN_EMB = 1 << 8, 1 << 9, 1 << 18, 1 << 20, 1 << 21, 1 << 22, 1 << 23


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


def bf16_split(x):
    import torch
    from test_bf16_host import split3
    return [p.numpy() for p in split3(torch.from_numpy(np.ascontiguousarray(x, np.float32)))]


def bf16_round(x):
    """RNE to bf16 as sealbart_set_tensor rounds the embedding table in gemm_mode 6"""
    return bf16_split(x)[0].astype(np.float32)


def run(kind, d, rows, fmt, **kw):
    """one sealdec_debug_rownorm call: (out or None, pieces as float32 arrays, overflow, path)"""
    from seal_b200._lib import NormCase, check, lib
    c = NormCase()
    keep = []
    scal = dict(kind=kind, d=d, rows=rows, out_split=fmt, tok_stride=1, scale=1.0, eps=1e-6, out_scale=1.0, split_unscale=1.0)
    scal.update({k: v for k, v in kw.items() if not isinstance(v, np.ndarray)})
    for k, v in scal.items():
        setattr(c, k, v)
    for k, v in kw.items():
        if isinstance(v, np.ndarray):
            v = np.ascontiguousarray(v); keep.append(v)
            setattr(c, k, v.ctypes.data)
    n = rows * d
    out = np.empty(n, np.float32)
    dt = {1: np.float32, 2: np.float16, 3: np.uint16}.get(fmt, np.float32)
    sp = [np.empty(n, dt) for _ in range(3)]
    ovf = np.full(1, -1, np.int32); path = np.zeros(1, np.uint32)
    check(lib.sealdec_debug_rownorm(C.byref(c), out.ctypes.data, *[s.ctypes.data for s in sp], ovf.ctypes.data, path.ctypes.data))
    if fmt == 3:
        pieces = [(s.astype(np.uint32) << 16).view(np.float32).reshape(rows, d) for s in sp]
    else:
        pieces = [s.astype(np.float32).reshape(rows, d) for s in sp[:2]] if fmt else []
    return (out.reshape(rows, d) if kind != 4 else None), pieces, int(ovf[0]), int(path[0])


def check_formats(label, kind, d, rows, ref, bound, path, fmts=(1, 2, 3), residual=None, groups=None, **kw):
    """Run the case in each split format; check every element written, the path bit, the residual (kinds 2, 3) or
    the output (kinds 0, 1) identical in every format, the split pieces against the host splitters, the fp16 flag,
    and the fp32 value against ref within bound.  groups: row labels for the per-group ratio print.  Returns the
    fp32 value."""
    value = None; plain = None
    for fmt in fmts:
        out, pieces, ovf, got_path = run(kind, d, rows, fmt, **kw)
        assert got_path == path, (label, fmt, hex(got_path), hex(path))
        for i, p in enumerate(pieces):
            assert not np.isnan(p).any(), (label, fmt, "piece", i, np.argwhere(np.isnan(p))[:4])
        if out is not None:
            assert not np.isnan(out).any(), (label, fmt, "out", np.argwhere(np.isnan(out))[:4])
            if plain is None:
                plain = out
            else:
                assert np.array_equal(out, plain), (label, fmt, "plain output differs between split instantiations")
        if residual is not None:
            assert np.array_equal(out, residual), (label, fmt, "residual", np.argwhere(out != residual)[:4])
        if fmt == 1:
            hi, lo = pieces
            assert not (hi.view(np.uint32) & 0x1FFF).any(), (label, "hi is not TF32")
            s64 = hi.astype(np.float64) + lo.astype(np.float64)
            v1 = s64.astype(np.float32)
            assert np.array_equal(v1.astype(np.float64), s64), (label, "hi + lo is not an fp32 value")
            value = out if kind in (0, 1) else v1
            assert np.array_equal(v1, value), (label, "hi + lo != out")
            assert ovf == 0, (label, fmt, ovf)
            continue
        v = out if kind in (0, 1) else value
        assert v is not None, "format 1 runs first for kinds 2 .. 4"
        want = split_half(v) if fmt == 2 else bf16_split(v)
        for i, (p, w) in enumerate(zip(pieces, want)):
            w = np.asarray(w, np.float32)
            assert np.array_equal(p, w), (label, fmt, "piece", i, np.argwhere(p != w)[:4])
        assert ovf == (int((np.abs(v) > HALF_MAX).any()) if fmt == 2 else 0), (label, fmt, ovf)
        if value is None:
            value = v
    err = np.abs(value.astype(np.float64) - ref)
    r = err / bound
    names = groups if groups is not None else np.array(["all"] * rows)
    worst = {g: float(r[names == g].max()) for g in dict.fromkeys(names.tolist())}
    print(f"{label}: worst err/bound " + ", ".join(f"{g} {w:.3g}" for g, w in worst.items()))
    assert (err <= bound).all(), (label, worst, np.argwhere(err > bound)[:4])
    if "zero_mean" in worst:
        assert worst["zero_mean"] < 0.5, (label, worst)
    return value


def mixed_rows(rng, rows, d):
    """rows drawn from the crafted sets in turn, and each row's set"""
    names = np.array([R.DISTS[i % len(R.DISTS)] for i in range(rows)])
    v = np.empty((rows, d), np.float32)
    for dist in R.DISTS:
        m = names == dist
        if m.any():
            v[m] = R.craft_rows(rng, dist, int(m.sum()), d)
    return v, names


def add_inputs(rng, v, names, ks=1, unscale=1.0):
    """a, b (or split-K slices of b) with fp32(a + b) near v; constant rows get a = 0.5, b = 0.25 (exact)"""
    a, b = R.add_parts(rng, v)
    const = names == "constant"
    a[const] = v[const] - np.float32(0.25); b[const] = 0.25
    kw = dict(a=a)
    if ks > 1:
        parts, bias, fin = R.split_k(rng, b, ks, unscale)
        kw.update(split_part=parts, split_ks=ks, split_unscale=unscale, split_bias=bias)
        b = fin
    else:
        kw["b"] = b
    return kw, (a + b).astype(np.float32)


LN_D = [128, 384, 896, 1024]
ROWS = [1, 3, 2048, 2049, 4100]


def check_constant_rows(label, value, names, beta):
    const = names == "constant"
    if const.any():
        assert np.array_equal(value[const], np.broadcast_to(beta, value[const].shape)), (label, "constant rows must give beta")


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("d", LN_D)
def test_bart_add_ln(d, rows):
    rng = np.random.default_rng(d * 7 + rows)
    v, names = mixed_rows(rng, rows, d)
    kw, x = add_inputs(rng, v, names)
    g, b = R.norm_weights(rng, d)
    row = rows <= 2048
    ref, bound = R.ln_ref(x, 0.0, g, b, R.depth_cta() if row else R.depth_warp(d))
    val = check_formats(f"add_ln d={d} rows={rows}", 1, d, rows, ref, bound, ROW if row else WARP, groups=names, gamma=g, beta=b, **kw)
    check_constant_rows("add_ln", val, names, b)


@pytest.mark.parametrize("d,rows,ks,unscale", [(384, 3, 2, 1.0), (1024, 2048, 3, 0.25), (896, 37, 8, 2.0 ** -3)])
def test_bart_add_ln_split_k(d, rows, ks, unscale):
    rng = np.random.default_rng(ks)
    v, names = mixed_rows(rng, rows, d)
    kw, x = add_inputs(rng, v, names, ks, unscale)
    g, b = R.norm_weights(rng, d)
    ref, bound = R.ln_ref(x, 0.0, g, b, R.depth_cta())
    check_formats(f"add_ln split-K d={d} rows={rows} ks={ks}", 1, d, rows, ref, bound, ROW, groups=names, gamma=g, beta=b, **kw)


T5_D = [512, 768, 1024, 2048, 3072, 4096]


@pytest.mark.parametrize("rows,ks,out_scale", [(1, 1, 1.0), (3, 2, 1.0), (37, 3, 1.0), (300, 8, -1), (2049, 1, -1), (4100, 1, 1.0)])
@pytest.mark.parametrize("d", T5_D)
def test_t5_rms_add(d, rows, ks, out_scale):
    rng = np.random.default_rng(d + rows)
    v, names = mixed_rows(rng, rows, d)
    kw, x = add_inputs(rng, v, names, ks, 0.5 if ks > 1 else 1.0)
    w = (1.0 + 0.25 * rng.standard_normal(d)).astype(np.float32)
    osc = float(np.float32(d ** -0.5)) if out_scale == -1 else out_scale
    ref, bound = R.rms_ref(x, w, 1e-6, osc, R.depth_t5(d))
    check_formats(f"t5_rms d={d} rows={rows} ks={ks} out_scale={osc:.3g}", 2, d, rows, ref, bound, T5_WIDE if d > 1024 else T5,
                  residual=x, groups=names, gamma=w, eps=1e-6, out_scale=osc, **kw)


@pytest.mark.parametrize("d", T5_D)
def test_t5_rms_embedding(d):
    """the embedding form: rows tok[r * tok_stride] of a bf16-valued table (so every format reads the same values);
    x_out is the table row itself"""
    rng = np.random.default_rng(d)
    V, rows, stride = 50, 67, 3
    emb = bf16_round(rng.standard_normal((V, d)).astype(np.float32) * 4)
    tok = rng.integers(0, V, size=rows * stride).astype(np.int32)
    x = emb[tok[::stride]]
    w = (1.0 + 0.25 * rng.standard_normal(d)).astype(np.float32)
    ref, bound = R.rms_ref(x, w, 1e-6, 1.0, R.depth_t5(d))
    check_formats(f"t5_rms embedding d={d}", 2, d, rows, ref, bound, T5_WIDE if d > 1024 else T5, residual=x, gamma=w, eps=1e-6,
                  tok=tok, tok_stride=stride, V=V, embed=emb)


def test_bf16_table_rounded_like_set_tensor():
    """out_split 3 rounds an fp32 table to bf16 as sealbart_set_tensor does: the same result as the rounded table"""
    rng = np.random.default_rng(4)
    d, V, rows = 1024, 20, 9
    emb = rng.standard_normal((V, d)).astype(np.float32)
    tok = rng.integers(0, V, size=rows).astype(np.int32)
    w = np.ones(d, np.float32)
    a = run(2, d, rows, 3, tok=tok, V=V, embed=emb, gamma=w)
    b = run(2, d, rows, 3, tok=tok, V=V, embed=bf16_round(emb), gamma=w)
    assert np.array_equal(a[0], bf16_round(emb)[tok]) and np.array_equal(a[0], b[0])
    assert all(np.array_equal(p, q) for p, q in zip(a[1], b[1]))


@pytest.mark.parametrize("rows", [1, 3, 2049, 4100])
@pytest.mark.parametrize("d", LN_D)
def test_preln_add(d, rows):
    rng = np.random.default_rng(d * 3 + rows)
    ks = 2 if rows == 3 else 8 if rows == 4100 else 1
    v, names = mixed_rows(rng, rows, d)
    kw, x = add_inputs(rng, v, names, ks, 2.0 if ks > 1 else 1.0)
    g, b = R.norm_weights(rng, d)
    ref, bound = R.ln_ref(x, 0.0, g, b, R.depth_cta())
    val = check_formats(f"preln d={d} rows={rows} ks={ks}", 3, d, rows, ref, bound, PRELN, residual=x, groups=names, gamma=g, beta=b,
                        **kw)
    if ks == 1:                                      # slices fold to 0.25 only approximately
        check_constant_rows("preln", val, names, b)


def embedding_inputs(rng, d, rows, V, pos_rows, stride=2, scale=1.0):
    """a bf16-valued table, strided tokens, per-row positions that include the table's last row and rows past it"""
    emb = bf16_round(rng.standard_normal((V, d)).astype(np.float32))
    tok = rng.integers(0, V, size=rows * stride).astype(np.int32)
    ptab = (0.5 * rng.standard_normal((pos_rows, d))).astype(np.float32)
    pos = rng.integers(0, 1025, size=rows).astype(np.int32)
    special = [0, pos_rows - 3, pos_rows - 2, pos_rows - 1, 1024]       # the last row with offset 2 / 0, past it, the limit
    n = min(rows, len(special))
    pos[:n] = special[-n:]
    return dict(tok=tok, tok_stride=stride, V=V, embed=emb, pos_table=ptab, pos_rows=pos_rows, scale=scale, pos=pos)


@pytest.mark.parametrize("rows", [1, 3, 2049])
@pytest.mark.parametrize("d", LN_D)
def test_bart_embedding(d, rows):
    """kind 0: positions p read row min(p + 2, pos_rows - 1) -- past the table its last row, never the NaN guard rows"""
    rng = np.random.default_rng(d + 5 * rows)
    kw = embedding_inputs(rng, d, rows, 40, 130, scale=float(np.float32(np.sqrt(d))))
    g, b = R.norm_weights(rng, d)
    e = kw["embed"][kw["tok"][::2]].astype(np.float64)
    prow = kw["pos_table"][np.minimum(kw["pos"] + 2, 129)].astype(np.float64)
    v = e * kw["scale"] + prow                       # the kernel rounds it once (fma): within u |v|
    ref, bound = R.ln_ref(v, R.U * np.abs(v), g, b, R.depth_warp(d))
    check_formats(f"embed_ln d={d} rows={rows}", 0, d, rows, ref, bound, 0, gamma=g, beta=b, **kw)
    # a decoder step: every row at one position, here past the table (reads the last row)
    kw2 = dict(kw, pos=None, pos_const=600)
    kw2 = {k: v2 for k, v2 in kw2.items() if v2 is not None}
    v2 = e * kw["scale"] + kw["pos_table"][129].astype(np.float64)
    ref2, bound2 = R.ln_ref(v2, R.U * np.abs(v2), g, b, R.depth_warp(d))
    check_formats(f"embed_ln d={d} rows={rows} pos_const=600", 0, d, rows, ref2, bound2, 0, fmts=(1,), gamma=g, beta=b, **kw2)


@pytest.mark.parametrize("ln_emb", [False, True])
@pytest.mark.parametrize("d", LN_D)
def test_preln_embedding(d, ln_emb):
    """kind 3, Pegasus (offset 0) and mBART (offset 2, layernorm_embedding): x_out = fp32(fp32(e * scale) + pos row), or
    its LayerNorm with ln_emb; the output split the LayerNorm of x_out"""
    rng = np.random.default_rng(d + ln_emb)
    rows, off, pos_rows = 2100, 2 if ln_emb else 0, 66
    kw = embedding_inputs(rng, d, rows, 60, pos_rows, scale=float(np.float32(np.sqrt(d))) if not ln_emb else 1.0)
    kw["pos_offset"] = off
    g, b = R.norm_weights(rng, d)
    e = kw["embed"][kw["tok"][::2]]
    x = (e * np.float32(kw["scale"])).astype(np.float32) + kw["pos_table"][np.minimum(kw["pos"] + off, pos_rows - 1)]
    path = PRELN
    if ln_emb:
        lg, lb = R.norm_weights(rng, d)
        kw.update(ln_emb_g=lg, ln_emb_b=lb)
        path |= PRELN_EMB
        out, _, _, _ = run(3, d, rows, 1, gamma=g, beta=b, **kw)
        ref1, bound1 = R.ln_ref(x, 0.0, lg, lb, R.depth_cta())
        r = np.abs(out.astype(np.float64) - ref1) / bound1
        print(f"preln embedding d={d} layernorm_embedding: worst err/bound {r.max():.3g}")
        assert (r <= 1).all()
        x = out                                       # the second LayerNorm reads these fp32 values
    ref, bound = R.ln_ref(x, 0.0, g, b, R.depth_cta())
    check_formats(f"preln embedding d={d} ln_emb={ln_emb}", 3, d, rows, ref, bound, path, residual=x if not ln_emb else None,
                  gamma=g, beta=b, **kw)


@pytest.mark.parametrize("f,rows", [(64, 60000), (2816, 1100), (10240, 300)])
def test_t5_gate(f, rows):
    """rows * f / 4 float4 is several times the gate's grid (8 CTAs of 256 threads per SM): rows past a grid-stride
    boundary are written too"""
    rng = np.random.default_rng(f)
    h = rng.standard_normal((rows, 2 * f)).astype(np.float32) * np.float32(2.0)
    h[::7, :f] *= 8                                  # saturated tanh
    h[::5, :f] *= np.float32(0.01)
    ref, bound = R.gate_ref(h)
    check_formats(f"gate f={f} rows={rows}", 4, f, rows, ref, bound, T5_GATE, h=h)


@pytest.mark.parametrize("over", [False, True])
@pytest.mark.parametrize("kind", [0, 1, 3, 4])
def test_fp16_flag_at_its_threshold(kind, over):
    """gamma = 0 in column 5: LayerNorm gives beta there exactly; the gate gives x * g exactly once tanhf saturates.  65 504
    raises nothing, 65 504 + 2^-8 raises the flag and saturates to (65 504, 0); formats 1 and 3 never raise it."""
    rng = np.random.default_rng(kind)
    d, rows = 256, 5
    edge = np.float32(HALF_MAX + 2.0 ** -8) if over else np.float32(HALF_MAX)
    if kind == 4:
        h = rng.standard_normal((rows, 2 * d)).astype(np.float32)
        h[:, 5] = edge; h[:, d + 5] = 1.0
        kw = dict(h=h)
    else:
        g, b = R.norm_weights(rng, d)
        g[5] = 0.0; b[5] = edge
        kw = dict(gamma=g, beta=b)
        if kind == 0:
            kw.update(tok=np.arange(rows, dtype=np.int32), V=rows, embed=rng.standard_normal((rows, d)).astype(np.float32),
                      pos_table=rng.standard_normal((10, d)).astype(np.float32), pos_rows=10, pos_const=1)
        else:
            kw.update(a=rng.standard_normal((rows, d)).astype(np.float32), b=rng.standard_normal((rows, d)).astype(np.float32))
    vals = {}
    for fmt in (1, 2, 3):
        out, pieces, ovf, _ = run(kind, d, rows, fmt, **kw)
        if fmt == 1:
            vals = (pieces[0].astype(np.float64) + pieces[1]).astype(np.float32)
            assert (vals[:, 5] == edge).all()
            if kind in (0, 1):
                assert (out[:, 5] == edge).all()
        assert ovf == (int(over) if fmt == 2 else 0), (fmt, ovf)
        if fmt == 2:
            assert (pieces[0][:, 5] == HALF_MAX).all() and (pieces[1][:, 5] == 0).all()


# ---- BART's position table ----------------------------------------------------------------------------------------
def tiny_bart(P):
    import torch
    from transformers import BartConfig, BartForConditionalGeneration
    from oracle.decode_oracle import NEG_INF
    cfg = BartConfig(vocab_size=2000, d_model=128, encoder_layers=2, decoder_layers=2, encoder_attention_heads=2,
                     decoder_attention_heads=2, encoder_ffn_dim=512, decoder_ffn_dim=512, max_position_embeddings=P)
    cfg.forced_bos_token_id = None
    torch.manual_seed(3)
    model = BartForConditionalGeneration(cfg).eval().float()
    with torch.no_grad():
        for t in (cfg.pad_token_id, cfg.bos_token_id, cfg.vocab_size - 1):
            model.final_logits_bias[0, t] = NEG_INF
    return model


def test_bart_position_limit():
    """max_position_embeddings = 8: a 10-row table, decoder position p reads row p + 2, valid for p <= 7.  A generate
    whose last position is 8 raises the reference's IndexError; one that ends at 7 runs and matches the oracle;
    teacher-forced decoder inputs of 9 tokens are refused, 8 run; the embedding at positions past the table reads
    its last row."""
    import torch
    from oracle.decode_oracle import fm_index_generate_oracle
    from oracle.fm_oracle import OracleIndex
    from seal_b200._lib import SealB200Error
    from seal_b200.beam_search import SealBartEngine, fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    model = tiny_bart(8)
    docs = make_corpus(n_docs=200, doc_len=24, n_phrases=400, seed=11, vocab=2000)
    seqs = [dd.tolist() for dd in docs]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    rng = np.random.default_rng(0)
    ids = torch.tensor(rng.integers(4, 2000, size=(2, 8)), dtype=torch.long); ids[:, 0] = 0; ids[:, -1] = 2
    am = torch.ones_like(ids)
    kw = dict(num_beams=3, length_penalty=0.0)
    with pytest.raises(IndexError) as e_ref:
        fm_index_generate_oracle(model, ora, ids, am, min_length=10, max_length=10, **kw)
    with pytest.raises(IndexError) as e_got:
        fm_index_generate(model, idx, ids, am, keep_history=True, min_length=10, max_length=10, **kw)
    assert str(e_got.value) == str(e_ref.value)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, min_length=9, max_length=9, **kw)
    exp = fm_index_generate_oracle(model, ora, ids, am, min_length=9, max_length=9, **kw)
    for a, b in zip(got, exp):
        fa = sorted((tuple(t), s) for s, t in a if ora.get_count(list(t[1:])) > 0)
        fb = sorted((tuple(t), s) for s, t, _ in b if ora.get_count(list(t[1:])) > 0)
        assert [x[0] for x in fa] == [x[0] for x in fb]
        assert all(abs(x[1] - y[1]) < 1e-4 for x, y in zip(fa, fb))
    # teacher-forced scoring: T = 9 decoder tokens reach position 8
    from seal_b200._lib import check, lib
    eng = SealBartEngine.from_hf(model, device=0)
    assert eng.max_positions == 8
    src, msk = ids.numpy().astype(np.int64), am.numpy().astype(np.int64)
    for T, ok in ((8, True), (9, False)):
        dec = np.ascontiguousarray(rng.integers(4, 2000, size=(2, T)).astype(np.int64))
        rq = np.arange(2, dtype=np.int32)
        out = np.empty((2, T - 1), np.float32)
        rc = lib.sealdec_teacher_forced(eng._h, src.ctypes.data, msk.ctypes.data, 2, 8, dec.ctypes.data, rq.ctypes.data, 2, T,
                                        1.0, out.ctypes.data, 0, None)
        if ok:
            check(rc)
            assert np.isfinite(out).all()
        else:
            assert rc == -1, rc
            with pytest.raises(SealB200Error):
                eng.debug_step_logits(src, msk, 1, dec)
    # the embedding hook on this model's decoder table: positions 8, 9 and 1024 read row 9, the last
    sd = model.state_dict()
    table = sd["model.decoder.embed_positions.weight"].numpy().astype(np.float32)
    assert table.shape[0] == 10
    emb = sd["model.shared.weight"].numpy().astype(np.float32)
    g = sd["model.decoder.layernorm_embedding.weight"].numpy(); b = sd["model.decoder.layernorm_embedding.bias"].numpy()
    tok = np.array([5, 17, 300], np.int32)
    v = emb[tok].astype(np.float64) + table[9]
    ref, bound = R.ln_ref(v, R.U * np.abs(v), g, b, R.depth_warp(128))
    for p in (8, 9, 1024):
        out, _, _, _ = run(0, 128, 3, 1, tok=tok, V=2000, embed=emb, pos_table=table, pos_rows=10, pos_const=p, gamma=g, beta=b)
        assert not np.isnan(out).any() and (np.abs(out - ref) <= bound).all(), p
