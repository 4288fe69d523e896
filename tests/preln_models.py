"""Seeded random-init HF Pegasus and mBART models (the pre-LayerNorm BART family) for the pre-LN tests; nothing is
downloaded.  Token conventions: Pegasus's own (pad = decoder_start = 0, eos = 1 = forced EOS), used for the mBART test
models too so that one corpus and one source builder serve both (tests/t5_models.py has the same ids)."""
import numpy as np

PAD, EOS = 0, 1

# name -> (model_type, config arguments, vocab, target standard deviation of the logits)
#   pegasus_relu   d 128, relu, scaled embedding, a 60-row sinusoidal table, tied lm_head
#   pegasus_gelu   d 512, gelu (PegasusConfig() default), unscaled, 2 encoder / 3 decoder layers, untied lm_head
#   mbart          d 1024, gelu, layernorm_embedding, 1 encoder / 2 decoder layers, learned table with offset 2
#   mbart_relu     d 128, relu (mBART's layer with Pegasus's activation), 3 encoder / 2 decoder layers, untied lm_head
#   pegasus_96k    d 128, pegasus-large's vocabulary (96 103 ids): two-CTA top-k clusters
#   mbart_250k     d 128, mbart-large's vocabulary (250 027 ids): five-CTA top-k clusters
SHAPES = {
    "pegasus_relu": ("pegasus", dict(d_model=128, encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=256,
                                     decoder_ffn_dim=256, encoder_layers=2, decoder_layers=2, activation_function="relu",
                                     scale_embedding=True, max_position_embeddings=60), 2000, 3.0, True),
    "pegasus_gelu": ("pegasus", dict(d_model=512, encoder_attention_heads=8, decoder_attention_heads=8, encoder_ffn_dim=1024,
                                     decoder_ffn_dim=1024, encoder_layers=2, decoder_layers=3, activation_function="gelu",
                                     scale_embedding=False, max_position_embeddings=128), 2000, 3.0, False),
    "mbart": ("mbart", dict(d_model=1024, encoder_attention_heads=16, decoder_attention_heads=16, encoder_ffn_dim=2048,
                            decoder_ffn_dim=2048, encoder_layers=1, decoder_layers=2, activation_function="gelu",
                            scale_embedding=True, max_position_embeddings=128), 2000, 3.0, True),
    "mbart_relu": ("mbart", dict(d_model=128, encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=320,
                                 decoder_ffn_dim=320, encoder_layers=3, decoder_layers=2, activation_function="relu",
                                 scale_embedding=False, max_position_embeddings=128), 2000, 3.0, False),
    "pegasus_96k": ("pegasus", dict(d_model=128, encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=256,
                                    decoder_ffn_dim=256, encoder_layers=2, decoder_layers=2, activation_function="relu",
                                    scale_embedding=True, max_position_embeddings=128), 96103, 1.5, True),
    "mbart_250k": ("mbart", dict(d_model=128, encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=256,
                                 decoder_ffn_dim=256, encoder_layers=2, decoder_layers=2, activation_function="gelu",
                                 scale_embedding=True, max_position_embeddings=128), 250027, 1.0, True),
}


def hf_config(name, **over):
    """The HF config of shape `name` with the generation ids a released checkpoint carries (decoder_start 0, forced EOS
    = EOS, no forced BOS); `over` replaces any argument."""
    from transformers import MBartConfig, PegasusConfig
    mt, kw, vocab, _, _ = SHAPES[name]
    args = dict(vocab_size=vocab, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, pad_token_id=PAD,
                eos_token_id=EOS, bos_token_id=PAD, decoder_start_token_id=PAD, forced_eos_token_id=EOS, **kw)
    args.update(over)
    cfg = (PegasusConfig if mt == "pegasus" else MBartConfig)(**args)
    cfg.forced_bos_token_id = None
    return cfg


def make_preln(name="pegasus_relu", seed=0, **over):
    """Pegasus / MBartForConditionalGeneration in fp32, eval mode.  Random init gives logits of standard deviation
    ~ 0.02 sqrt(d) (tied) or ~ sqrt(d) (an untied lm_head of unit entries); the decoder's final layer_norm weight sets it
    to the shape's target (3: beam scores neither tie nearly everywhere nor reach hundreds of nats; 1 at 250 027 ids,
    where a full fp32 log-softmax of ~4 puts the fp32 oracle itself near the 1e-4 score bound, and 1.5 at 96 103)."""
    import torch
    from transformers import MBartForConditionalGeneration, PegasusForConditionalGeneration
    mt, _, vocab, target, tied = SHAPES[name]
    cfg = hf_config(name, **over)
    torch.manual_seed(seed)
    model = (PegasusForConditionalGeneration if mt == "pegasus" else MBartForConditionalGeneration)(cfg).eval().float()
    d = cfg.d_model
    with torch.no_grad():
        if not tied:
            g = torch.Generator().manual_seed(seed + 1)
            model.lm_head.weight = torch.nn.Parameter(torch.randn(vocab, d, generator=g))
        w = model.lm_head.weight
        model.model.decoder.layer_norm.weight.fill_(target / (float(w.std()) * d ** 0.5))
        # layer norms start at gamma 1, beta 0: give them values so that a misplaced gamma or beta shows
        g = torch.Generator().manual_seed(seed + 2)
        for n, p in model.named_parameters():
            if "layer_norm" in n or "layernorm_embedding" in n:
                if n.endswith("bias"):
                    p.copy_(0.1 * torch.randn(p.shape, generator=g))
                elif "decoder.layer_norm" not in n:
                    p.mul_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
    return model


def preln_sources(rng, Q, S, vocab, kind="right"):
    """int64 [Q, S] sources ending in EOS, padded with PAD; query 0 is full length (tests/t5_models.py's builder)."""
    from t5_models import t5_sources
    return t5_sources(rng, Q, S, vocab, kind)
