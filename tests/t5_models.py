"""Seeded random-init HF T5 models for the T5 tests (nothing is downloaded), and SEAL's T5 token conventions
(seal/retrieval.py:494-504): pad = decoder_start = 0, eos = 1 = the title BOS, an in-vocabulary title EOS."""
import numpy as np

PAD, EOS, TITLE_BOS = 0, 1, 1

# name -> T5Config arguments.  The four shapes the T5 path is checked on:
#   tiny        d = 128, 2 heads, relu, tied lm_head (output scaled by d^-0.5)
#   tiny_gated  d = 128, gated-gelu, untied lm_head, d_ff a multiple of 64 but not of 128, non-default buckets
#   medium      d = 512, 8 heads, gated-gelu, num_layers != num_decoder_layers
#   medium_relu d = 512, relu, tied, num_layers != num_decoder_layers the other way round
SHAPES = {
    "tiny": dict(d_model=128, num_heads=2, d_ff=256, num_layers=2, num_decoder_layers=2, feed_forward_proj="relu",
                 tie_word_embeddings=True),
    "tiny_gated": dict(d_model=128, num_heads=2, d_ff=320, num_layers=2, num_decoder_layers=2,
                       feed_forward_proj="gated-gelu", tie_word_embeddings=False, relative_attention_num_buckets=16,
                       relative_attention_max_distance=48),
    "medium": dict(d_model=512, num_heads=8, d_ff=1024, num_layers=2, num_decoder_layers=3,
                   feed_forward_proj="gated-gelu", tie_word_embeddings=False),
    "medium_relu": dict(d_model=512, num_heads=8, d_ff=2048, num_layers=3, num_decoder_layers=2,
                        feed_forward_proj="relu", tie_word_embeddings=True),
}


def make_t5(name="tiny", vocab=2000, seed=0):
    """T5ForConditionalGeneration in fp32, eval mode, with the generation attributes a released T5 config.json
    carries (decoder_start_token_id 0; no forced BOS / EOS), which the decode oracle reads from the config."""
    import torch
    from transformers import T5Config, T5ForConditionalGeneration
    cfg = T5Config(vocab_size=vocab, d_kv=64, dropout_rate=0.0, pad_token_id=PAD, eos_token_id=EOS, **SHAPES[name])
    cfg.decoder_start_token_id = PAD
    cfg.forced_bos_token_id = None
    cfg.forced_eos_token_id = None
    torch.manual_seed(seed)
    model = T5ForConditionalGeneration(cfg).eval().float()
    # transformers ties lm_head to shared whatever the config says (tie_word_embeddings=False only clears
    # scale_decoder_outputs); an untied shape gets an lm_head of its own, of unit standard deviation.  HF's init gives
    # logits of standard deviation ~ sqrt(d_model) untied and ~ 1 tied: the decoder's final_layer_norm weight sets it to
    # ~ 4 for both, so that beam scores neither tie nearly everywhere nor reach hundreds of nats
    d = cfg.d_model
    untied = not SHAPES[name]["tie_word_embeddings"]
    with torch.no_grad():
        if untied:
            g = torch.Generator().manual_seed(seed + 1)
            model.lm_head.weight = torch.nn.Parameter(torch.randn(vocab, d, generator=g))
        model.decoder.final_layer_norm.weight.fill_(4.0 / d ** 0.5 if untied else 4.0)
    return model


def title_corpus(vocab=2000, n_docs=300, doc_len=30, seed=3):
    """Synthetic documents laid out as SEAL indexes T5 titles: title BOS (1), five title tokens, the title EOS
    (vocab - 1), then the body."""
    from seal_b200.synthetic import make_corpus
    docs = make_corpus(n_docs=n_docs, doc_len=doc_len, n_phrases=2 * n_docs, seed=seed, vocab=vocab - 1)
    teos = vocab - 1
    return [[TITLE_BOS] + d[:5].tolist() + [teos] + d[5:].tolist() for d in docs], teos


def t5_sources(rng, Q, S, vocab, kind="right"):
    """int64 [Q, S] sources ending in EOS (1), padded with PAD (0); query 0 is full length.  kind: 'right' padding,
    'holes' (masked positions inside the source) or 'left' padding."""
    ids = rng.integers(4, vocab, size=(Q, S)).astype(np.int64)
    am = np.ones((Q, S), dtype=np.int64)
    for q in range(Q):
        l = S if q == 0 else int(rng.integers(min(max(3, S // 2), S), S + 1))
        ids[q, l - 1] = EOS
        ids[q, l:] = PAD
        am[q, l:] = 0
        if kind == "holes" and l >= 3:
            am[q, rng.choice(np.arange(1, l - 1), size=max(1, (l - 2) // 4), replace=False)] = 0
        if kind == "left" and l < S:
            ids[q] = np.roll(ids[q], S - l); am[q] = np.roll(am[q], S - l)
    return ids, am
