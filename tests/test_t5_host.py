"""CPU: the host side of the T5 path -- the relative position bucket table (sealt5_relative_buckets) against
transformers' _relative_position_bucket, the config resolution and shape checks of SealT5Engine (ValueError before the
library is called), and the decode oracle on a T5 model (its KV-cached and re-forwarding steppers agree)."""
import numpy as np
import pytest

from t5_models import EOS, make_t5, title_corpus


@pytest.mark.parametrize("num_buckets,max_distance", [(32, 128), (16, 48), (64, 256), (8, 20), (33, 100), (4, 3)])
@pytest.mark.parametrize("bidirectional", [True, False])
def test_bucket_table_equals_hf(num_buckets, max_distance, bidirectional):
    """Every distance the kernels index: -1023 .. 1023 for the encoder (bidirectional), 0 .. -127 for the decoder."""
    import torch
    from transformers.models.t5.modeling_t5 import T5Attention
    from seal_b200._lib import lib, check
    n = 1024 if bidirectional else 128
    out = np.empty(2 * n - 1 if bidirectional else n, dtype=np.int32)
    check(lib.sealt5_relative_buckets(num_buckets, max_distance, int(bidirectional), n, out.ctypes.data))
    rel = torch.arange(-(n - 1), n) if bidirectional else -torch.arange(n)
    want = T5Attention._relative_position_bucket(rel, bidirectional=bidirectional, num_buckets=num_buckets,
                                                 max_distance=max_distance).numpy()
    assert np.array_equal(out, want)
    # the [query, key] grid HF builds in compute_bias, indexed through the table
    q, k = np.arange(n)[:, None], np.arange(n)[None, :]
    grid = T5Attention._relative_position_bucket(torch.from_numpy(k - q), bidirectional=bidirectional,
                                                 num_buckets=num_buckets, max_distance=max_distance).numpy()
    if bidirectional:
        assert np.array_equal(out[k - q + n - 1], grid)
    else:
        lower = np.tril_indices(n)                      # keys up to the query (the decoder's causal window)
        assert np.array_equal(out[(q - k).clip(0)][lower], grid[lower])
    assert out.max() < num_buckets


def test_bucket_table_rejects_uncovered_settings():
    from seal_b200._lib import lib
    out = np.empty(64, dtype=np.int32)
    for nb, md in [(3, 100), (2048, 4096), (32, 16), (32, 8)]:
        assert lib.sealt5_relative_buckets(nb, md, 1, 8, out.ctypes.data) != 0


class _NoCall:
    def __init__(self):
        self.called = False

    def __call__(self, *a):
        self.called = True
        raise AssertionError("the library was called")


@pytest.mark.parametrize("change,match", [
    (dict(d_kv=128, d_model=1024, num_heads=8), "d_kv"),
    (dict(num_heads=3), "num_heads"),
    (dict(d_model=576, num_heads=9), "multiple of 128"),
    (dict(d_model=1152, num_heads=18), "multiple of 128"),
    (dict(d_ff=200), "d_ff"),
    (dict(feed_forward_proj="gated-relu"), "feed_forward_proj"),
    (dict(feed_forward_proj="gelu"), "feed_forward_proj"),
    (dict(relative_attention_num_buckets=2), "buckets"),
    (dict(relative_attention_num_buckets=32, relative_attention_max_distance=16), "buckets"),
])
def test_config_checks_raise_before_the_library(change, match, monkeypatch):
    from transformers import T5Config, T5ForConditionalGeneration
    from seal_b200 import beam_search
    base = dict(vocab_size=300, d_model=128, d_kv=64, num_heads=2, d_ff=256, num_layers=1, num_decoder_layers=1)
    base.update(change)
    cfg = T5Config(**base)
    fake = _NoCall()
    monkeypatch.setattr(beam_search.lib, "sealt5_create", fake)
    with pytest.raises(ValueError, match=match):
        beam_search.SealT5Engine({}, cfg, device=0, gemm_mode=3)
    model = T5ForConditionalGeneration(T5Config(**dict(base, num_layers=1, num_decoder_layers=1)))
    with pytest.raises(ValueError, match=match):
        beam_search.SealBartEngine.from_hf(model)          # dispatches on model_type before any device work
    assert not fake.called


def test_config_view_resolution():
    """decoder_start_token_id: config, else generation_config, else pad_token_id; forced BOS / EOS None where missing;
    the output scale from scale_decoder_outputs, else tie_word_embeddings."""
    from types import SimpleNamespace
    from transformers import T5Config
    from seal_b200.beam_search import T5ConfigView, t5_native_config
    cfg = T5Config(vocab_size=300, d_model=128, num_heads=2, d_ff=256, pad_token_id=0, eos_token_id=1)
    for a in ("decoder_start_token_id", "forced_bos_token_id", "forced_eos_token_id"):
        if a in cfg.__dict__:
            delattr(cfg, a)
    v = T5ConfigView(cfg)
    assert v.decoder_start_token_id == 0 and v.forced_bos_token_id is None and v.forced_eos_token_id is None
    assert v.eos_token_id == 1 and v.pad_token_id == 0 and v.vocab_size == 300
    assert T5ConfigView(cfg, SimpleNamespace(decoder_start_token_id=7)).decoder_start_token_id == 7
    cfg.decoder_start_token_id = 5
    assert T5ConfigView(cfg, SimpleNamespace(decoder_start_token_id=7)).decoder_start_token_id == 5
    ns = SimpleNamespace(**{k: getattr(cfg, k) for k in ("vocab_size", "d_model", "num_heads", "d_kv", "d_ff", "num_layers",
                                                         "relative_attention_num_buckets", "layer_norm_epsilon",
                                                         "pad_token_id", "eos_token_id")})
    for tie, scale, want in [(True, None, 1), (False, None, 0), (True, False, 0), (False, True, 1)]:
        ns.tie_word_embeddings = tie
        if scale is None:
            ns.__dict__.pop("scale_decoder_outputs", None)
        else:
            ns.scale_decoder_outputs = scale
        assert T5ConfigView(ns).scale_decoder_outputs == bool(want)
        c = t5_native_config(ns, 3)
        assert c.scale_decoder_outputs == want and c.ffn_kind == 0 and c.num_decoder_layers == c.num_layers
        assert c.relative_attention_max_distance == 128          # transformers 4.13's T5Config has no such attribute


def test_oracle_cached_stepper_equals_reforwarding_stepper_on_t5():
    """oracle/decode_oracle.py drives any HF seq2seq model through get_encoder() and model(...): on a T5 model its
    KV-cached and re-forwarding steppers give the same hypotheses, as they do for BART."""
    import torch
    from oracle.decode_oracle import fm_index_generate_oracle
    from oracle.fm_oracle import OracleIndex
    docs, teos = title_corpus()
    ora = OracleIndex(docs)
    model = make_t5("tiny")
    rng = np.random.default_rng(12)
    ids = torch.tensor(rng.integers(4, 2000, size=(3, 10)), dtype=torch.long); ids[:, -1] = EOS
    am = torch.ones_like(ids); ids[1, 7:] = 0; ids[1, 6] = EOS; am[1, 7:] = 0
    for kw in (dict(num_beams=5, min_length=7, max_length=7, length_penalty=0.0),
               dict(num_beams=4, min_length=1, max_length=9, length_penalty=0.0, force_decoding_from=[1], eos_token_id=teos)):
        a = fm_index_generate_oracle(model, ora, ids, am, **kw)
        b = fm_index_generate_oracle(model, ora, ids, am, use_cache=True, **kw)
        for qa, qb in zip(a, b):
            assert [tuple(t) for _, t, _ in qa] == [tuple(t) for _, t, _ in qb]
            # scores reach ~150 nats here, where one fp32 ulp is 1.5e-5: the project's decode bound
            assert all(abs(x[0] - y[0]) <= 1e-4 for x, y in zip(qa, qb))
        assert all(t[0] == 0 for q in a for _, t, _ in q)                # decoder_start = pad = 0
