"""CPU: the T5 width rule at the XL / XXL widths.  d_model is a multiple of 128 up to 1 024 or a multiple of 1 024 up to
4 096, with 64-wide heads and num_heads * 64 == d_model; t5_native_config fills the native config of the widths it
accepts, and every other width, head count or head size is rejected in Python before the library is called and by
sealt5_create itself (SEALFM_EINVAL, before it looks for a device)."""
import ctypes as C

import pytest

EINVAL = -1


def t5_config(**kw):
    from transformers import T5Config
    base = dict(vocab_size=300, d_kv=64, d_ff=512, num_layers=2, num_decoder_layers=3)
    base.update(kw)
    return T5Config(**base)


@pytest.mark.parametrize("d", [2048, 3072, 4096])
@pytest.mark.parametrize("proj,kind", [("relu", 0), ("gated-gelu", 1)])
def test_wide_widths_fill_the_native_config(d, proj, kind):
    from seal_b200.beam_search import t5_native_config
    cfg = t5_config(d_model=d, num_heads=d // 64, feed_forward_proj=proj, tie_word_embeddings=kind == 0,
                    layer_norm_epsilon=1e-6)
    c = t5_native_config(cfg, 3)
    assert (c.vocab_size, c.d_model, c.num_layers, c.num_decoder_layers) == (300, d, 2, 3)
    assert (c.num_heads, c.d_kv, c.d_ff, c.ffn_kind) == (d // 64, 64, 512, kind)
    assert (c.relative_attention_num_buckets, c.relative_attention_max_distance) == (32, 128)
    assert c.layer_norm_epsilon == pytest.approx(1e-6) and c.gemm_mode == 3
    assert c.scale_decoder_outputs == (1 if kind == 0 else 0)


class _NoCall:
    def __init__(self):
        self.called = False

    def __call__(self, *a):
        self.called = True
        raise AssertionError("the library was called")


# widths between and beyond the two ranges, a head count that does not match d_model, 128-wide heads
REJECTED = [
    (dict(d_model=1152, num_heads=18), "multiple of 128"),
    (dict(d_model=1536, num_heads=24), "multiple of 128"),
    (dict(d_model=5120, num_heads=80), "multiple of 128"),
    (dict(d_model=8192, num_heads=128), "multiple of 128"),
    (dict(d_model=2048, num_heads=16), "num_heads"),
    (dict(d_model=4096, num_heads=32, d_kv=128), "d_kv"),
]


@pytest.mark.parametrize("change,match", REJECTED, ids=[f"{c['d_model']}_{c['num_heads']}_{c.get('d_kv', 64)}" for c, _ in REJECTED])
def test_uncovered_widths_raise_before_the_library(change, match, monkeypatch):
    from seal_b200 import beam_search
    fake = _NoCall()
    monkeypatch.setattr(beam_search.lib, "sealt5_create", fake)
    with pytest.raises(ValueError, match=match):
        beam_search.SealT5Engine({}, t5_config(**change), device=0, gemm_mode=3)
    assert not fake.called


@pytest.mark.parametrize("d,heads,d_kv", [(1152, 18, 64), (1536, 24, 64), (5120, 80, 64), (8192, 128, 64),
                                          (2048, 16, 64), (4096, 32, 128), (576, 9, 64), (1024, 8, 128), (128, 3, 64)])
def test_sealt5_create_rejects_uncovered_widths(d, heads, d_kv):
    from seal_b200._lib import T5Config as NativeCfg, lib
    cfg = NativeCfg(300, d, 1, 1, heads, d_kv, 256, 0, 32, 128, 1e-6, 1, 3)
    h = C.c_void_p()
    assert lib.sealt5_create(C.byref(cfg), 0, C.byref(h)) == EINVAL
    assert not h.value
