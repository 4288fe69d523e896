"""CPU: the argument checks and C layout of sealdec_debug_rownorm (include/sealdec.h), and the running-error bound of
rownorm_ref.py checked against a float32 emulation of each kernel's operation order: the emulation stays within the
bound on every crafted row set, and the mistakes the GPU test must catch -- a one-pass variance, eps 1e-6 for 1e-5,
the unbiased variance, T5's out_scale applied to the residual, the erf GELU in the gate -- exceed it."""
import ctypes as C
import re

import numpy as np
import pytest

import rownorm_ref as R
from test_gemm_split_out_host import header_args

EINVAL, ENODEVICE = -1, -4


def base_case(kind):
    """a small valid case of each kind (the add form for kinds 2 and 3); the arrays are kept alive in the dict"""
    d = 256 if kind == 4 else 128
    rows = 3
    arr = dict(gamma=np.ones(d, np.float32), beta=np.zeros(d, np.float32))
    scal = dict(kind=kind, d=d, rows=rows, out_split=1, tok_stride=1, V=10, scale=1.0, eps=1e-6, out_scale=1.0, pos_rows=12,
                split_unscale=1.0)
    if kind == 0:
        arr.update(tok=np.arange(rows, dtype=np.int32), embed=np.zeros((10, d), np.float32), pos_table=np.zeros((12, d), np.float32))
    elif kind == 4:
        arr = dict(h=np.zeros((rows, 2 * d), np.float32))
    else:
        arr.update(a=np.zeros((rows, d), np.float32), b=np.zeros((rows, d), np.float32))
    return scal, arr


def call(scal, arr):
    from seal_b200._lib import NormCase, lib
    c = NormCase()
    for k, v in scal.items():
        setattr(c, k, v)
    for k, v in arr.items():
        setattr(c, k, v.ctypes.data if v is not None else None)
    n = max(int(scal["rows"]), 1) * scal["d"]
    out = np.empty(n, np.float32)
    sp = [np.empty(n, np.float32) for _ in range(3)]
    ovf = np.zeros(1, np.int32)
    path = np.zeros(1, np.uint32)
    rc = lib.sealdec_debug_rownorm(C.byref(c), out.ctypes.data, *[s.ctypes.data for s in sp], ovf.ctypes.data, path.ctypes.data)
    return rc, lib.sealfm_last_error().decode()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def _valid_cases():
    emb_t5 = dict(tok=np.arange(3, dtype=np.int32), embed=np.zeros((10, 128), np.float32), a=None, b=None)
    emb_pre = dict(emb_t5, pos_table=np.zeros((12, 128), np.float32))
    sk = dict(split_part=np.zeros((3, 3, 128), np.float32), split_bias=np.zeros(128, np.float32), b=None)
    return {
        "bart_embedding": (0, {}, {}),
        "bart_add_ln": (1, {}, {}),
        "bart_add_ln_split_k": (1, dict(split_ks=3), sk),
        "t5_add": (2, {}, {}),
        "t5_embedding_wide": (2, dict(d=2048), dict(tok=np.arange(3, dtype=np.int32), embed=np.zeros((10, 2048), np.float32), a=None,
                                                    b=None, gamma=np.ones(2048, np.float32))),
        "t5_embedding": (2, {}, emb_t5),
        "preln_add_split_k": (3, dict(split_ks=8), dict(sk, split_part=np.zeros((8, 3, 128), np.float32))),
        "preln_embedding_ln_emb": (3, dict(pos_offset=2), dict(emb_pre, ln_emb_g=np.ones(128, np.float32), ln_emb_b=np.zeros(128, np.float32))),
        "preln_embedding_last_position": (3, dict(pos_const=1024), emb_pre),
        "gate": (4, {}, {}),
    }


@pytest.mark.parametrize("name", sorted(_valid_cases()))
def test_valid_case_reaches_the_device_check(name):
    kind, so, ao = _valid_cases()[name]
    scal, arr = base_case(kind)
    scal.update(so); arr.update(ao)
    rc, msg = call(scal, arr)
    assert rc == (0 if have_gpu() else ENODEVICE), (name, rc, msg)


def _bad_cases():
    z = lambda *s: np.zeros(s, np.float32)
    sk = dict(split_part=z(2, 3, 128), split_bias=z(128), b=None)
    emb_t5 = dict(tok=np.arange(3, dtype=np.int32), embed=z(10, 128), a=None, b=None)
    emb_pre = dict(emb_t5, pos_table=z(12, 128))
    big = dict(a=z(2049, 128), b=None, split_part=z(2, 2049, 128), split_bias=z(128))
    return {
        "unknown_kind": (5, {}, {}),
        "negative_kind": (-1, {}, {}),
        "bart_d_not_128_multiple": (1, dict(d=192), dict(a=z(3, 192), b=z(3, 192), gamma=z(192), beta=z(192))),
        "bart_d_over_1024": (1, dict(d=1152), dict(a=z(3, 1152), b=z(3, 1152), gamma=z(1152), beta=z(1152))),
        "preln_d_2048": (3, dict(d=2048), dict(a=z(3, 2048), b=z(3, 2048), gamma=z(2048), beta=z(2048))),
        "t5_d_1536": (2, dict(d=1536), dict(a=z(3, 1536), b=z(3, 1536), gamma=z(1536))),
        "t5_d_over_4096": (2, dict(d=5120), dict(a=z(3, 5120), b=z(3, 5120), gamma=z(5120))),
        "gate_f_not_64_multiple": (4, dict(d=96), dict(h=z(3, 192))),
        "rows_zero": (1, dict(rows=0), {}),
        "rows_negative": (2, dict(rows=-1), {}),
        "ks_9": (1, dict(split_ks=9), dict(sk, split_part=z(9, 3, 128))),
        "ks_negative": (1, dict(split_ks=-2), sk),
        "split_k_on_warp_kernel": (1, dict(rows=2049, split_ks=2), big),
        "split_k_on_bart_embedding": (0, dict(split_ks=2), dict(split_part=z(2, 3, 128), split_bias=z(128))),
        "split_k_on_t5_embedding": (2, dict(split_ks=2), dict(emb_t5, split_part=z(2, 3, 128), split_bias=z(128))),
        "split_k_on_gate": (4, dict(split_ks=2), dict(split_part=z(2, 3, 256), split_bias=z(256))),
        "split_k_bias_missing": (3, dict(split_ks=2), dict(sk, split_bias=None)),
        "token_past_vocab": (0, {}, dict(tok=np.array([0, 10, 1], np.int32))),
        "token_negative": (2, {}, dict(emb_t5, tok=np.array([0, -1, 1], np.int32))),
        "token_past_vocab_strided": (3, dict(tok_stride=2), dict(emb_pre, tok=np.array([0, 0, 10, 0, 1, 0], np.int32))),
        "position_negative": (0, {}, dict(pos=np.array([0, -1, 2], np.int32))),
        "position_past_1024": (0, dict(pos_const=1025), {}),
        "preln_position_past_1024": (3, {}, dict(emb_pre, pos=np.array([0, 1025, 2], np.int32))),
        "pos_rows_past_1026": (0, dict(pos_rows=1027), dict(pos_table=z(1027, 128))),
        "bart_pos_rows_below_3": (0, dict(pos_rows=2), {}),
        "preln_pos_offset_1": (3, dict(pos_offset=1), emb_pre),
        "preln_ln_emb_half": (3, {}, dict(emb_pre, ln_emb_g=z(128))),
        "t5_split_none": (2, dict(out_split=0), {}),
        "preln_split_none": (3, dict(out_split=0), {}),
        "gate_split_none": (4, dict(out_split=0), {}),
        "unknown_split": (1, dict(out_split=4), {}),
        "tok_and_a": (3, {}, dict(emb_pre, a=z(3, 128), b=z(3, 128))),
        "b_missing": (1, {}, dict(b=None)),
        "a_missing": (2, {}, dict(a=None)),
        "gamma_missing": (1, {}, dict(gamma=None)),
        "beta_missing": (3, {}, dict(beta=None)),
        "embed_missing": (0, {}, dict(embed=None)),
        "pos_table_missing": (0, {}, dict(pos_table=None)),
        "h_missing": (4, {}, dict(h=None)),
        "t5_eps_nan": (2, dict(eps=float("nan")), {}),
    }


@pytest.mark.parametrize("name", sorted(_bad_cases()))
def test_bad_arguments_rejected_before_device_work(name):
    kind, so, ao = _bad_cases()[name]
    scal, arr = base_case(min(max(kind, 0), 4))
    scal["kind"] = kind
    scal.update(so); arr.update(ao)
    rc, msg = call(scal, arr)
    assert rc == EINVAL, (name, rc, msg)


def test_missing_outputs_rejected():
    from seal_b200._lib import NormCase, lib
    scal, arr = base_case(1)
    c = NormCase()
    for k, v in scal.items():
        setattr(c, k, v)
    for k, v in arr.items():
        setattr(c, k, v.ctypes.data)
    buf = np.empty(3 * 128 * 2, np.float32); path = np.zeros(1, np.uint32); ovf = np.zeros(1, np.int32)
    p = buf.ctypes.data
    assert lib.sealdec_debug_rownorm(None, p, p, p, p, ovf.ctypes.data, path.ctypes.data) == EINVAL
    assert lib.sealdec_debug_rownorm(C.byref(c), None, p, p, p, ovf.ctypes.data, path.ctypes.data) == EINVAL       # out
    assert lib.sealdec_debug_rownorm(C.byref(c), p, p, None, p, ovf.ctypes.data, path.ctypes.data) == EINVAL       # split2
    assert lib.sealdec_debug_rownorm(C.byref(c), p, p, p, p, ovf.ctypes.data, None) == EINVAL                      # path
    c.out_split = 2
    assert lib.sealdec_debug_rownorm(C.byref(c), p, p, p, p, None, path.ctypes.data) == EINVAL                     # overflow
    c.out_split = 3
    assert lib.sealdec_debug_rownorm(C.byref(c), p, p, p, None, ovf.ctypes.data, path.ctypes.data) == EINVAL       # split3


def test_hook_signature_matches_the_header():
    from seal_b200._lib import lib
    decl = header_args("sealdec_debug_rownorm")
    types = lib.sealdec_debug_rownorm.argtypes
    assert len(types) == len(decl), (len(types), decl)
    for d, t in zip(decl, types):
        assert "*" in d and (t is C.c_void_p or issubclass(t, C._Pointer)), (d, t)


def test_case_struct_matches_the_header():
    """sealdec_norm_case_t field by field: name, order, pointer or scalar type; so ctypes' offsets are the C offsets"""
    import os
    from seal_b200._lib import NormCase
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "sealdec.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} sealdec_norm_case_t;", text).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        base = re.match(r"(const\s+)?(\w+)", decl).group(2)
        for name in decl[decl.index(base) + len(base):].split(","):
            ptr = "*" in name
            fields.append((name.replace("*", "").strip(), "ptr" if ptr else base))
    ours = NormCase._fields_
    assert [n for n, _ in ours] == [n for n, _ in fields]
    ctype = {"int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float}
    for (n, t), (_, kind) in zip(ours, fields):
        assert (t is C.c_void_p) if kind == "ptr" else (t is ctype[kind]), (n, t, kind)


# ---- the bound against the fp32 emulation ---------------------------------------------------------------------------
def ratio(got, ref, bound):
    err = np.abs(got.astype(np.float64) - ref)
    return float((err / bound).max())


LN_D = [128, 384, 896, 1024]


@pytest.mark.parametrize("form", ["cta", "warp"])
@pytest.mark.parametrize("d", LN_D)
def test_layernorm_bound_holds_and_catches_mistakes(form, d):
    rng = np.random.default_rng(d + (form == "warp"))
    D = R.depth_cta() if form == "cta" else R.depth_warp(d)
    g, b = R.norm_weights(rng, d)
    caught = {"one_pass": False, "eps": False, "unbiased": False}
    for dist in R.DISTS:
        v = R.craft_rows(rng, dist, 24, d)
        ref, bound = R.ln_ref(v, 0.0, g, b, D)
        r = ratio(R.emulate_ln(v, g, b, form, rng), ref, bound)
        print(f"{form} d={d} {dist}: worst err/bound {r:.3g}")
        assert r <= 1.0, (dist, r)
        if dist == "zero_mean":
            assert r < 0.5, r
        if dist == "constant":
            assert np.array_equal(R.emulate_ln(v, g, b, form, rng), np.broadcast_to(b, v.shape))
        for mut, kw in (("one_pass", dict(one_pass=True)), ("eps", dict(eps=1e-6)), ("unbiased", dict(unbiased=True))):
            with np.errstate(invalid="ignore"):
                m = R.emulate_ln(v, g, b, form, rng, **kw)
            caught[mut] |= not (np.abs(m.astype(np.float64) - ref) <= bound).all()
    assert all(caught.values()), caught


@pytest.mark.parametrize("d", [512, 768, 1024, 2048, 3072, 4096])
def test_rmsnorm_bound_holds_and_catches_mistakes(d):
    rng = np.random.default_rng(d)
    D = R.depth_t5(d)
    w = (1.0 + 0.25 * rng.standard_normal(d)).astype(np.float32)
    caught = {"residual_scale": False}
    for dist in R.DISTS:
        v = R.craft_rows(rng, dist, 16, d)
        for eps, osc in ((1e-6, 1.0), (1e-6, 1.0 / np.sqrt(d)), (1e-5, 1.0)):
            ref, bound = R.rms_ref(v, w, eps, osc, D)
            x, out = R.emulate_rms(v, w, eps, osc, rng)
            assert np.array_equal(x, v)
            r = ratio(out, ref, bound)
            print(f"rms d={d} {dist} eps={eps} out_scale={osc:.3g}: worst err/bound {r:.3g}")
            assert r <= 1.0, (dist, eps, osc, r)
            x_m, out_m = R.emulate_rms(v, w, eps, osc, rng, residual_scale=True)
            if osc != 1.0:
                caught["residual_scale"] |= not np.array_equal(x_m, v) and not (np.abs(out_m - ref) <= bound).all()
    assert all(caught.values()), caught


def test_gate_bound_holds_and_catches_the_erf_gelu():
    rng = np.random.default_rng(5)
    for scale in (0.01, 1.0, 3.0, 30.0):
        h = (scale * rng.standard_normal((64, 2 * 1024))).astype(np.float32)
        ref, bound = R.gate_ref(h)
        r = ratio(R.emulate_gate(h, rng), ref, bound)
        print(f"gate scale {scale}: worst err/bound {r:.3g}")
        assert r <= 1.0, (scale, r)
    h = rng.standard_normal((64, 2 * 1024)).astype(np.float32)
    ref, bound = R.gate_ref(h)
    assert not (np.abs(R.emulate_gate(h, rng, erf=True) - ref) <= bound).all()


def test_split_k_fold_reference():
    """the slices fold back to the finished value in fp32 exactly, and a fold with unscale after the bias does not"""
    rng = np.random.default_rng(3)
    b = rng.standard_normal((8, 256)).astype(np.float32)
    for ks, unscale in ((2, 1.0), (3, 0.25), (8, 2.0 ** -3)):
        parts, bias, fin = R.split_k(rng, b, ks, unscale)
        assert parts.shape == (ks, 8, 256)
        y = parts[0].copy()
        for s in range(1, ks):
            y = y + parts[s]
        assert np.array_equal((y * np.float32(unscale) + bias).astype(np.float32), fin)
        assert np.abs(fin.astype(np.float64) - b).max() < 1e-5
        if unscale != 1.0:
            assert not np.array_equal(((y + bias) * np.float32(unscale)).astype(np.float32), fin)
