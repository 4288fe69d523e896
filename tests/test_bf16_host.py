"""CPU: the host side of gemm_mode 6 (bf16 weights, the 3xBF16 GEMM; include/sealdec.h).

  - the three-piece bf16 split of an fp32 activation, with torch's round-to-nearest-even conversion, is exact for
    every 2^-100 <= |a| < (2 - 2^-8) 2^127 (random and extreme values, both boundaries), can be inexact far below the
    lower one, and gives an infinite first piece from the upper one on (the values that round past bf16's largest);
  - the engines' default gemm_mode: explicit argument, then $SEALB200_GEMM, then 6 iff every weight matrix is bf16;
  - the engine cache sees a model converted in place by `.to(torch.bfloat16)`;
  - the C ABI accepts gemm_mode 6 at creation for all three handle kinds and still rejects unknown modes;
  - the device-memory formula (device_bytes_formula, also used by the GPU tests) at the shapes the docs quote."""
import ctypes as C

import numpy as np
import pytest

K_T5_MAX_SOURCE, K_MAX_LEN = 1024, 128          # t5_kernels.cuh / decode_kernels.cuh: the bucket tables' lengths


def split3(a):
    """b1, b2, b3 (as float32 tensors) of the bf16 split_value (operand_split.cuh) computed with torch's RNE conversion"""
    import torch
    b1 = a.to(torch.bfloat16).float()
    r = a - b1
    b2 = r.to(torch.bfloat16).float()
    b3 = (r - b2).to(torch.bfloat16).float()
    return b1, b2, b3


def inexact(a):
    b1, b2, b3 = split3(a)
    return (b1.double() + b2.double() + b3.double()) != a.double()


def random_fp32(rng, n, lo_exp, hi_exp):
    """n fp32 values with uniform exponents in [lo_exp, hi_exp], random mantissas and signs"""
    import torch
    e = rng.integers(lo_exp, hi_exp + 1, size=n)
    m = rng.integers(0, 1 << 23, size=n, dtype=np.int64)
    bits = ((e + 127).astype(np.int64) << 23) | m | (rng.integers(0, 2, size=n, dtype=np.int64) << 31)
    return torch.from_numpy(bits.astype(np.uint32).view(np.float32).copy())


BF16_ROUNDS_TO_INF = (2.0 - 2.0 ** -8) * 2.0 ** 127     # the midpoint between bf16's largest value and 2^128


def test_split_is_exact_in_range():
    import torch
    rng = np.random.default_rng(0)
    a = random_fp32(rng, 2_000_000, -100, 127)
    inside = a.abs().double() < BF16_ROUNDS_TO_INF
    assert not inexact(a[inside]).any()
    # extremes: the largest value below the upper boundary, all-ones mantissas (the rounding carries), halfway
    # mantissas (ties to even), powers of two, the lower boundary
    top = np.nextafter(np.float32(BF16_ROUNDS_TO_INF), np.float32(0))
    ext = [top, -top, 2.0 ** -100, -(2.0 ** -100), 1.0, 3.0, 1.0 / 3.0]
    ones = np.array([((e + 127) << 23) | 0x7FFFFF for e in range(-100, 127)], dtype=np.uint32).view(np.float32)
    halfway = np.array([((e + 127) << 23) | 0x8000 | (0x7F << 16) for e in range(-100, 127)], dtype=np.uint32).view(np.float32)
    pieces = torch.from_numpy(np.concatenate([np.array(ext, dtype=np.float32), ones, halfway, -ones]))
    assert not inexact(pieces).any()
    # from the upper boundary on, the first piece is infinite (torch and __float2bfloat16_rn round alike)
    big = torch.tensor([BF16_ROUNDS_TO_INF, np.finfo(np.float32).max, -BF16_ROUNDS_TO_INF], dtype=torch.float32)
    assert torch.isinf(split3(big)[0]).all()
    # the boundary's neighbourhood: every value with exponent -100 .. -98 and a dense mantissa sample
    near = random_fp32(rng, 200_000, -100, -98)
    assert not inexact(near).any()


def test_split_can_be_inexact_far_below_the_qualifier():
    """below |a| ~ 2^-110 the last residual can fall under bf16's normal range (2^-126), where it loses bits: the
    qualifier is a real limit of the split, not an artefact of the proof"""
    rng = np.random.default_rng(1)
    bad = inexact(random_fp32(rng, 200_000, -126, -111))
    assert bad.any()
    assert not inexact(random_fp32(rng, 200_000, -109, -100)).any()


# ---- default mode and the engine cache ------------------------------------------------------------------------------

def bart_like_state_dict(dtype, overrides=None):
    import torch
    sd = {"model.shared.weight": torch.zeros(8, 4, dtype=dtype),
          "model.encoder.embed_positions.weight": torch.zeros(6, 4, dtype=dtype),
          "model.encoder.layers.0.fc1.weight": torch.zeros(8, 4, dtype=dtype),
          "model.encoder.layers.0.fc1.bias": torch.zeros(8, dtype=dtype),
          "model.encoder.layers.0.final_layer_norm.weight": torch.zeros(4, dtype=dtype),
          "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": torch.zeros(32, 2, dtype=dtype)}
    for k, v in (overrides or {}).items():
        sd[k] = sd[k].to(v)
    return sd


def test_default_gemm_mode(monkeypatch):
    import torch
    from seal_b200.beam_search import default_gemm_mode
    monkeypatch.delenv("SEALB200_GEMM", raising=False)
    assert default_gemm_mode(bart_like_state_dict(torch.float32)) == 3
    assert default_gemm_mode(bart_like_state_dict(torch.float16)) == 3
    assert default_gemm_mode(bart_like_state_dict(torch.bfloat16)) == 6
    # a matrix kept in fp32 (a T5 whose wo stays fp32): the upcast path
    assert default_gemm_mode(bart_like_state_dict(torch.bfloat16, {"model.encoder.layers.0.fc1.weight": torch.float32})) == 3
    assert default_gemm_mode(bart_like_state_dict(torch.bfloat16, {"model.shared.weight": torch.float32})) == 3
    # vectors and the fp32 tables (positions, relative-attention bias) do not decide the mode
    sd = bart_like_state_dict(torch.bfloat16, {"model.encoder.layers.0.fc1.bias": torch.float32,
                                               "model.encoder.embed_positions.weight": torch.float32,
                                               "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": torch.float32})
    assert default_gemm_mode(sd) == 6
    monkeypatch.setenv("SEALB200_GEMM", "2")
    assert default_gemm_mode(bart_like_state_dict(torch.bfloat16)) == 2
    monkeypatch.setenv("SEALB200_GEMM", "6")
    assert default_gemm_mode(bart_like_state_dict(torch.float32)) == 6


def test_explicit_mode_wins_over_the_dtype(monkeypatch):
    """the gemm_mode each engine class hands to the library: the explicit argument, else the dtype rule (the library
    call is replaced by a probe that records the configuration and fails)"""
    import torch
    from transformers import BartConfig, PegasusConfig, T5Config
    from seal_b200 import beam_search
    seen = []

    def probe(*args):
        seen.append(args[0]._obj.gemm_mode)
        return -1

    for name in ("sealbart_create", "sealt5_create"):
        monkeypatch.setattr(beam_search.lib, name, probe)
    monkeypatch.delenv("SEALB200_GEMM", raising=False)
    small = dict(vocab_size=64, d_model=128, encoder_layers=1, decoder_layers=1, encoder_attention_heads=2,
                 decoder_attention_heads=2, encoder_ffn_dim=256, decoder_ffn_dim=256, max_position_embeddings=32)
    cfgs = [(beam_search.SealBartEngine, BartConfig(**small)), (beam_search.SealPreLnEngine, PegasusConfig(**small)),
            (beam_search.SealT5Engine, T5Config(vocab_size=64, d_model=128, num_heads=2, d_kv=64, d_ff=256, num_layers=1))]
    for cls, cfg in cfgs:
        for sd_dtype, mode in ((torch.bfloat16, None), (torch.bfloat16, 3), (torch.float32, None), (torch.float32, 6)):
            with pytest.raises(Exception):
                cls(bart_like_state_dict(sd_dtype), cfg, device=0, gemm_mode=mode)
    assert seen == [6, 3, 3, 6] * 3, seen


def test_engine_cache_sees_in_place_bf16_conversion(monkeypatch):
    import torch
    from seal_b200 import beam_search
    built = []

    class FakeEngine:
        def __init__(self, dtypes):
            self.dtypes = dtypes

    def fake_from_hf(model, device=None, gemm_mode=None):
        built.append(FakeEngine(frozenset(p.dtype for p in model.parameters())))
        return built[-1]

    monkeypatch.setattr(beam_search.SealBartEngine, "from_hf", staticmethod(fake_from_hf))
    model = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.LayerNorm(4))
    e1 = beam_search._engine_for(model)
    assert beam_search._engine_for(model) is e1 and len(built) == 1
    assert model.to(torch.bfloat16) is model                   # in place: the same object comes back
    e2 = beam_search._engine_for(model)
    assert e2 is not e1 and e2.dtypes == {torch.bfloat16}
    assert beam_search._engine_for(model) is e2 and len(built) == 2
    model.float()
    assert beam_search._engine_for(model) is not e2 and len(built) == 3


# ---- the C ABI --------------------------------------------------------------------------------------------------------

def create_rc(kind, gemm_mode):
    """sealbart_create (no variant, or a pre-LayerNorm one) / sealt5_create of a tiny shape; returns (rc, message).  A
    device-less host answers a valid configuration with SEALFM_ENODEVICE; a GPU host creates (and frees) the model."""
    from seal_b200._lib import BartConfig, BartVariant, T5Config, lib
    h = C.c_void_p()
    if kind == "bart":
        rc = lib.sealbart_create(C.byref(BartConfig(64, 128, 1, 1, 2, 256, 32, 0, gemm_mode)), None, 0, C.byref(h))
    elif kind == "preln":
        rc = lib.sealbart_create(C.byref(BartConfig(64, 128, 1, 1, 2, 256, 32, 0, gemm_mode)),
                                 C.byref(BartVariant(1, 0, 0, 1)), 0, C.byref(h))
    else:
        rc = lib.sealt5_create(C.byref(T5Config(64, 128, 1, 1, 2, 64, 256, 1, 32, 128, 1e-6, 1, gemm_mode)), 0, C.byref(h))
    msg = lib.sealfm_last_error().decode()
    if h.value:
        lib.sealbart_free(h.value)
    return rc, msg


@pytest.mark.parametrize("kind", ["bart", "preln", "t5"])
def test_create_accepts_mode_6_and_rejects_unknown_modes(kind):
    from seal_b200._lib import lib
    for bad in (0, 1, 4, 7, -1):
        rc, msg = create_rc(kind, bad)
        assert rc != 0 and "gemm_mode must be" in msg and "6 (3xBF16" in msg, (bad, rc, msg)
    for good in (2, 3, 5, 6):
        rc, msg = create_rc(kind, good)
        assert rc == 0 or "gemm_mode" not in msg, (good, rc, msg)


def test_header_documents_mode_6():
    import os
    h = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "sealdec.h")).read()
    assert "6 = 3xBF16" in h and "24 3xBF16 GEMM" in h and "sealdec_debug_head_ex" in h


# ---- device memory ----------------------------------------------------------------------------------------------------

def device_bytes_formula(kind, cfg, gemm_mode, tied=True):
    """sealbart_device_bytes after finalize, from the shapes: gemm_mode 6 holds 2 bytes per matrix element (every GEMM
    weight, the embedding table, an untied lm_head) and 4 per element of every fp32 vector and table; the other modes
    4 per element of everything plus the two fp16 halves (2 x 2 bytes) of every GEMM weight, the lm_head included.
    kind "t5": cfg = (d, d_ff, V, heads, enc layers, dec layers, gated, buckets); "bart" / "preln": cfg = (d, ffn, V,
    enc layers, dec layers, position rows, layernorm_embedding)."""
    if kind == "t5":
        d, f, V, H, Le, Ld, gated, nb = cfg
        F1 = 2 * f if gated else f
        enc = [(3 * d, d), (d, d), (F1, d), (d, f)]
        dec = [(3 * d, d), (d, d), (d, d), (2 * d, d), (d, d), (F1, d), (d, f)]
        vec = V + Le * 2 * d + Ld * 3 * d + 2 * d + 2 * nb * H               # final_bias, norms, relative tables
        tables = (2 * K_T5_MAX_SOURCE - 1) + K_MAX_LEN                         # int32 bucket tables
    else:
        d, f, V, Le, Ld, P, ln_emb = cfg
        enc = [(3 * d, d), (d, d), (f, d), (d, f)]
        dec = [(3 * d, d), (d, d), (d, d), (2 * d, d), (d, d), (f, d), (d, f)]
        vec = V + 2 * P * d + (Le * 2 + Ld * 3) * 2 * d + (2 * 2 * d if ln_emb else 0) + (2 * 2 * d if kind == "preln" else 0)
        tables = 0
    lin = Le * sum(o * i for o, i in enc) + Ld * sum(o * i for o, i in dec)
    vec += Le * sum(o for o, _ in enc) + Ld * sum(o for o, _ in dec)       # the Lin biases (zero for T5)
    mat = lin + V * d * (1 if tied else 2)
    if gemm_mode == 6:
        return 2 * mat + 4 * vec + 4 * tables
    return 4 * mat + 4 * (lin + V * d) + 4 * vec + 4 * tables


def test_device_memory_formula_at_the_documented_shapes():
    """INTEGRATION.md's table: t5-v1_1-xxl / flan-t5-xxl ~ 22 GB in gemm_mode 6 (~ 89 GB in the fp32-master layout),
    mT5-XXL ~ 26 GB (~ 99 GB), bart-large 0.8 GB (3.2 GB)"""
    xxl = (4096, 10240, 32128, 64, 24, 24, True, 32)
    mt5 = (4096, 10240, 250112, 64, 24, 24, True, 32)
    bart = (1024, 4096, 50265, 12, 12, 1026, True)
    got = {n: (device_bytes_formula(k, c, 6, tied) / 1e9, device_bytes_formula(k, c, 3, tied) / 1e9)
           for n, k, c, tied in [("xxl", "t5", xxl, False), ("mt5", "t5", mt5, False), ("bart", "bart", bart, True)]}
    print(got)
    assert 22.2 < got["xxl"][0] < 22.4 and 88.4 < got["xxl"][1] < 88.7
    assert 25.8 < got["mt5"][0] < 25.9 and 99.2 < got["mt5"][1] < 99.4
    assert 0.8 < got["bart"][0] < 0.85 and 3.2 < got["bart"][1] < 3.3
    for n, (b6, b3) in got.items():
        assert b6 < 0.3 * b3, n
