"""CPU: the host side of the pre-LayerNorm BART family (Pegasus, mBART) -- config rules, engine routing, generation-id
resolution, the position-table rule of fm_index_generate, and the decode oracle's steppers on both architectures."""
import numpy as np
import pytest
import torch

from preln_models import EOS, PAD, hf_config, make_preln, preln_sources


def test_native_config_of_both_architectures():
    from seal_b200.beam_search import preln_native_config
    cfg, var = preln_native_config(hf_config("pegasus_relu"), 3)
    assert (cfg.d_model, cfg.heads, cfg.ffn_dim, cfg.max_positions, cfg.scale_embedding, cfg.gemm_mode) == (128, 2, 256, 60, 1, 3)
    assert (var.pre_layer_norm, var.position_offset, var.layernorm_embedding, var.activation) == (1, 0, 0, 1)
    cfg, var = preln_native_config(hf_config("mbart"), 2)
    assert (cfg.d_model, cfg.heads, cfg.encoder_layers, cfg.decoder_layers, cfg.max_positions) == (1024, 16, 1, 2, 128)
    assert (var.pre_layer_norm, var.position_offset, var.layernorm_embedding, var.activation) == (1, 2, 1, 0)
    # PegasusConfig() defaults: gelu, d 1024, 16 heads
    from transformers import PegasusConfig
    cfg, var = preln_native_config(PegasusConfig(), 3)
    assert (cfg.d_model, cfg.heads, var.activation, var.position_offset) == (1024, 16, 0, 0)


@pytest.mark.parametrize("over,msg", [
    (dict(activation_function="silu"), "activation_function 'silu' is not implemented"),
    (dict(activation_function="gelu_new"), "activation_function 'gelu_new' is not implemented"),
    (dict(encoder_ffn_dim=512), "encoder and decoder must have the same heads and ffn_dim"),
    (dict(encoder_attention_heads=4, d_model=256, decoder_attention_heads=4), None),
    (dict(encoder_attention_heads=1), "encoder and decoder must have the same heads and ffn_dim"),
    (dict(d_model=192, encoder_attention_heads=3, decoder_attention_heads=3), "d_model must be a multiple of 128 up to 1 024"),
    (dict(d_model=2048, encoder_attention_heads=32, decoder_attention_heads=32), "d_model must be a multiple of 128 up to 1 024"),
    (dict(d_model=256, encoder_attention_heads=2, decoder_attention_heads=2), "64-wide heads"),
    (dict(encoder_ffn_dim=200, decoder_ffn_dim=200), "ffn_dim must be a positive multiple of 64"),
])
@pytest.mark.parametrize("name", ["pegasus_relu", "mbart_relu"])
def test_native_config_rejects_before_device_work(name, over, msg):
    from seal_b200.beam_search import preln_native_config
    cfg = hf_config(name, **over)
    if msg is None:
        preln_native_config(cfg, 3)
        return
    with pytest.raises(ValueError, match=msg):
        preln_native_config(cfg, 3)


def test_from_hf_rejects_before_device_work(monkeypatch):
    """An unsupported config raises ValueError from SealBartEngine.from_hf before the library is called"""
    import seal_b200.beam_search as bs
    called = []
    monkeypatch.setattr(bs, "_torch", lambda: called.append(1))
    model = make_preln("pegasus_relu")
    model.config.activation_function = "silu"
    with pytest.raises(ValueError, match="not implemented"):
        bs.SealBartEngine.from_hf(model)
    assert not called


def test_routing(monkeypatch):
    """bart -> SealBartEngine itself, pegasus / mbart -> SealPreLnEngine, t5 -> SealT5Engine"""
    import seal_b200.beam_search as bs
    seen = []
    monkeypatch.setattr(bs.SealPreLnEngine, "from_hf", classmethod(lambda cls, m, device=None, gemm_mode=None: seen.append("preln") or "preln"))
    monkeypatch.setattr(bs.SealT5Engine, "from_hf", classmethod(lambda cls, m, device=None, gemm_mode=None: seen.append("t5") or "t5"))
    monkeypatch.setattr(bs.SealBartEngine, "__init__", lambda self, sd, cfg, device=0, gemm_mode=None: seen.append("bart"))

    class Fake:
        def __init__(self, mt):
            self.config = type("C", (), {"model_type": mt})()

        def state_dict(self):
            return {}

        def parameters(self):
            return iter([torch.zeros(1)])

    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    for mt, want in (("pegasus", "preln"), ("mbart", "preln"), ("t5", "t5"), ("bart", "bart"), ("marian", "bart"),
                     ("bigbird_pegasus", "bart")):
        seen.clear()
        bs.SealBartEngine.from_hf(Fake(mt))
        assert seen == [want], (mt, seen)


def test_start_token_resolution():
    from seal_b200.beam_search import PreLnConfigView
    v = PreLnConfigView(hf_config("pegasus_relu"))
    assert (v.decoder_start_token_id, v.forced_eos_token_id, v.forced_bos_token_id) == (PAD, EOS, None)
    # mBART checkpoints often leave decoder_start_token_id None: bos_token_id then, as transformers 4.13 reads it
    from transformers import MBartConfig, PegasusConfig
    m = MBartConfig()
    assert m.decoder_start_token_id is None
    v = PreLnConfigView(m)
    assert (v.decoder_start_token_id, v.forced_eos_token_id) == (m.bos_token_id, 2)
    assert PreLnConfigView(PegasusConfig()).forced_eos_token_id == 1
    m.bos_token_id = None
    with pytest.raises(ValueError, match="`decoder_start_token_id` or `bos_token_id` has to be defined"):
        PreLnConfigView(m)
    assert PreLnConfigView(hf_config("mbart", decoder_start_token_id=7)).decoder_start_token_id == 7


def test_keep_history_position_limit():
    """keep_history=True runs every step: positions 0 .. max_length - 2 (constrained_beam_search: cur_len starts at 1,
    the newest token sits at cur_len - 1), so a 60-row table takes max_length 61 and refuses 62 -- and so does the
    reference's forward"""
    from seal_b200.beam_search import _check_decoder_positions
    eng = type("E", (), {"max_positions": 60})()
    _check_decoder_positions(eng, 61)
    with pytest.raises(IndexError, match="index out of range in self"):
        _check_decoder_positions(eng, 62)
    _check_decoder_positions(type("B", (), {})(), 128)          # no position table (T5): no bound
    # the HF forward at the boundary: position 59 runs, position 60 raises the same IndexError
    model = make_preln("pegasus_relu")
    ids, am = preln_sources(np.random.default_rng(0), 1, 6, 2000)
    with torch.inference_mode():
        enc = model.get_encoder()(input_ids=torch.tensor(ids), attention_mask=torch.tensor(am))
        from transformers.modeling_outputs import BaseModelOutput
        kw = dict(encoder_outputs=BaseModelOutput(last_hidden_state=enc.last_hidden_state), attention_mask=torch.tensor(am), use_cache=False)
        model(decoder_input_ids=torch.zeros((1, 60), dtype=torch.long), **kw)
        with pytest.raises(IndexError, match="index out of range in self"):
            model(decoder_input_ids=torch.zeros((1, 61), dtype=torch.long), **kw)


def _records(done_after, n_steps, B=2, T=None, fail_at=None):
    """Synthetic per-step records of one query per entry of done_after: the query's candidates are non-EOS tokens
    except that at step done_after[q] its top B candidates are EOS with equal scores, which makes the stock scorer done
    right there (None: never done); fail_at[q]: a step at which fewer than B non-EOS candidates exist."""
    Q, K = len(done_after), 2 * B
    T = T or n_steps + 1
    H = n_steps * K + B
    scores = np.full((Q, H), -5.0, dtype=np.float32)
    toks = np.full((Q, H, T), 7, dtype=np.int32)
    lens = np.full((Q, H), T, dtype=np.int32)
    toks[:, :, 0] = PAD
    for q in range(Q):
        for st in range(n_steps):
            base = st * K
            scores[q, base:base + K] = -1.0 - 0.1 * np.arange(K) - st
            if done_after[q] is not None and st == done_after[q]:
                # B equal EOS hypotheses at the top: B finished beams whose worst equals the best candidate -> done
                toks[q, base:base + B, st + 1] = EOS
                scores[q, base:base + B] = 10.0
            if fail_at is not None and fail_at[q] == st:
                toks[q, base:base + K, st + 1] = EOS
    return {"scores": scores, "lens": lens, "tokens": toks}


def test_stock_scorer_position_limit_both_sides():
    """keep_history=False: the reference runs step st while some query is not done; a step st >= the table's rows
    raises IndexError, any earlier end does not (positions past the table are never read)"""
    from seal_b200.beam_search import _replay_beam_search_scorer
    n_steps, B = 12, 2
    rp = lambda rec, P: _replay_beam_search_scorer(rec, B, 1.0, EOS, PAD, n_steps + 1, n_positions=P)
    rec = _records([3, 5], n_steps, B)                  # every query done after step 5: steps 0 .. 5 run
    ref = _replay_beam_search_scorer(rec, B, 1.0, EOS, PAD, n_steps + 1)
    for P in (6, 7, 100, None):
        got = rp(rec, P)
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1])
    with pytest.raises(IndexError, match="index out of range in self"):
        rp(rec, 5)                                      # step 5 reads position 5 of a 5-row table
    rec = _records([3, None], n_steps, B)               # query 1 runs every step
    assert rp(rec, n_steps)[0] == _replay_beam_search_scorer(rec, B, 1.0, EOS, PAD, n_steps + 1)[0]
    with pytest.raises(IndexError):
        rp(rec, n_steps - 1)
    # a num_beams failure before the first step past the table is met first; one after it is not reached
    rec = _records([None, None], n_steps, B, fail_at=[4, None])
    with pytest.raises(ValueError, match="At most 2 tokens"):
        rp(rec, 8)
    with pytest.raises(IndexError):
        rp(rec, 4)
    with pytest.raises(ValueError, match="At most 2 tokens"):
        rp(rec, None)


@pytest.mark.parametrize("name", ["pegasus_relu", "mbart_relu"])
def test_oracle_steppers_cached_vs_uncached(name):
    from oracle.decode_oracle import HFBartCachedStepper, HFBartStepper
    model = make_preln(name)
    rng = np.random.default_rng(4)
    ids, am = preln_sources(rng, 3, 9, 2000)
    ids, am = torch.from_numpy(ids), torch.from_numpy(am)
    B = 2
    a, b = HFBartStepper(model, ids, am, B), HFBartCachedStepper(model, ids, am, B)
    dec = torch.full((3 * B, 1), PAD, dtype=torch.long)
    worst = 0.0
    for t in range(5):
        la, lb = a(dec), b(dec)
        worst = max(worst, float((la - lb).abs().max()))
        perm = torch.arange(3 * B).view(3, B).flip(1).reshape(-1)
        nxt = torch.from_numpy(rng.integers(2, 2000, size=(3 * B, 1)))
        dec = torch.cat([dec[perm], nxt], dim=1)
        b.reorder(perm)
    print(f"{name}: cached vs uncached |dlogit| {worst:.2e}")
    assert worst < 1e-5
