"""Drop-in for ``seal.beam_search`` (/root/reference/seal/beam_search.py) on the H100 kernels.

* ``IndexBasedLogitsProcessor`` — same constructor, attributes and HF ``LogitsProcessor`` protocol
  (``__call__(input_ids, scores) -> scores + mask``, beam_search.py:33-140); the FM-index work and
  the mask run as CUDA kernels on the tensors' device, no ``.tolist()`` / H2D round trips.
* ``fm_index_generate`` — same signature and return value (beam_search.py:391-557), no sampling: encoder,
  every decoder step, the top-k logits warp (``topk``), log-softmax, processors, FM-index constraint, top-k and
  BeamSearchScorerWithMemory all run inside libsealb200.so.  ``keep_history=True`` is the path SEALSearcher uses, also with diverse beam
  groups (``diverse_bs_groups`` / ``diverse_bs_penalty``); ``keep_history=False`` (transformers' stock
  BeamSearchScorer, the signature's default) and ``transformers_output=True`` run the same kernels and replay
  the stock scorer over the per-step records (one beam group only).
* ``SealBartEngine`` — device copy of an HF ``BartForConditionalGeneration``'s weights (``SealPreLnEngine``: Pegasus and
  mBART, the pre-LayerNorm BART family; ``SealT5Engine``: T5).

No CPU path: CPU tensors are rejected.
"""
import ctypes as C
import math
import os
import weakref
from typing import List, Optional

import numpy as np

from ._lib import lib, check, vp, ProcessorCfg, BartConfig, BartVariant, DecParams, GroupParams, T5Config
from .index import FMIndex, SHIFT

stopword_token_ids = [10, 41, 660, 5, 1941, 20, 7, 6]      # beam_search.py:22-31


def _torch():
    import torch
    return torch


def _occurring_mask(index, vocab, device=None):
    """uint32 bitmask of index.occurring_distinct (first-step rule, beam_search.py:73-77)."""
    cache = index.__dict__.setdefault("_occ_cache", {})
    key = (vocab, str(device))
    if key not in cache:
        words = np.zeros((vocab + 31) // 32, dtype=np.uint32)
        toks = np.asarray([t for t in index.occurring_distinct if 0 <= t < vocab], dtype=np.int64)
        np.bitwise_or.at(words, toks >> 5, (np.uint32(1) << (toks & 31).astype(np.uint32)))
        if device is None:
            cache[key] = words
        else:
            torch = _torch()
            cache[key] = torch.from_numpy(words.view(np.int32)).to(device)
    return cache[key]


class IndexBasedLogitsProcessor:
    """beam_search.py:33-140.  (Does not inherit transformers.LogitsProcessor so that importing the
    drop-in never depends on the installed transformers version; HF only duck-types `__call__`.)"""

    def __init__(self, index: FMIndex, num_beams: int, pad_token_id: int = 0, eos_token_id: int = 2,
                 force_decoding_from: Optional[List[int]] = None, stop_at_count: int = 0,
                 always_allow_eos: bool = False, forced_bos_token_id: Optional[int] = None):
        self.index = index
        self.pad_token_id = pad_token_id
        self.eos_token_id = eos_token_id
        self._num_beams = num_beams
        self.log_odds_weight = 0.0
        self.force_decoding_from = force_decoding_from
        self.force_decoding_second_token = None
        self.block_initial_stopwords = False
        self.stop_at_count = stop_at_count
        self.always_allow_eos = always_allow_eos
        self.forced_bos_token_id = forced_bos_token_id

    def __call__(self, input_ids, scores):
        torch = _torch()
        if not (scores.is_cuda and input_ids.is_cuda):
            raise RuntimeError("seal_b200.IndexBasedLogitsProcessor runs on CUDA tensors only (no CPU fallback)")
        if scores.dtype != torch.float32:
            raise TypeError("scores must be float32 (the reference decodes in fp32)")
        ids = input_ids.to(torch.int64).contiguous()
        sc = scores.contiguous()
        R, t = ids.shape
        V = sc.shape[-1]
        out = torch.empty_like(sc)
        force = self.force_decoding_from or []
        farr = (C.c_int64 * max(len(force), 1))(*force)
        cfg = ProcessorCfg(self._num_beams, self.pad_token_id, self.eos_token_id, int(self.stop_at_count),
                           int(bool(self.always_allow_eos)),
                           -1 if self.forced_bos_token_id is None else int(self.forced_bos_token_id),
                           len(force), farr, SHIFT)
        with torch.cuda.device(sc.device):
            occ = _occurring_mask(self.index, V, sc.device)
            check(lib.sealdec_apply_index_mask_d(self.index._dev(), torch.cuda.current_stream().cuda_stream,
                                                 C.byref(cfg), ids.data_ptr(), R, t, occ.data_ptr(),
                                                 sc.data_ptr(), out.data_ptr(), V, sc.stride(0)))
        return out


# 2-D state_dict tensors that are tables read in fp32, not GEMM operands or the token embedding: they do not take part
# in choosing the bf16-weight mode
_FP32_TABLES = ("embed_positions.weight", "relative_attention_bias.weight")


def _is_weight_matrix(key, tensor):
    return key.endswith(".weight") and tensor.dim() == 2 and not key.endswith(_FP32_TABLES)


def default_gemm_mode(state_dict):
    """The gemm_mode an engine gets when none is given: $SEALB200_GEMM if set; else 6 (3xBF16, the weights stored once in
    bf16) when every weight matrix the GEMMs and the embedding read is torch.bfloat16; else 3 (3xFP16).  fp32, fp16 and
    mixed-dtype models therefore keep the fp32-master path (their weights are upcast, which is lossless)."""
    env = os.environ.get("SEALB200_GEMM")
    if env is not None:
        return int(env)
    torch = _torch()
    mats = [v for k, v in state_dict.items() if _is_weight_matrix(k, v)]
    return 6 if mats and all(v.dtype == torch.bfloat16 for v in mats) else 3


def _weight_dtypes(model):
    """The set of parameter dtypes of a model: `model.to(torch.bfloat16)` converts in place and changes it."""
    return frozenset(p.dtype for p in model.parameters())


def _hf_device(model):
    """The CUDA device of an HF model's engine: that of its parameters, else the current device."""
    p = next(model.parameters())
    return p.device.index if p.is_cuda else _torch().cuda.current_device()


def _load_weights(h, state_dict, shared_key):
    """Copies every tensor of `state_dict` to the handle h and finalizes it.  When `shared_key` (the shared token
    embedding) is present, its tied aliases are skipped: the embed_tokens keys, and an lm_head stored in the same
    memory (the library ties that itself)."""
    shared = state_dict.get(shared_key)
    for k, v in state_dict.items():
        if shared is not None and (k.endswith("embed_tokens.weight") or
                                   (k == "lm_head.weight" and v.data_ptr() == shared.data_ptr())):
            continue
        a = np.ascontiguousarray(v.detach().to("cpu").float().numpy())
        check(lib.sealbart_set_tensor(h, k.encode(), a.ctypes.data, a.size))
    check(lib.sealbart_finalize(h))


class SealBartEngine:
    """Device-resident BART weights + workspace (include/sealdec.h `sealbart_t`)."""

    def __init__(self, state_dict, config, device=0, gemm_mode=None):
        # gemm_mode: 3 = 3xFP16 with one CTA per tile, 5 = 3xFP16 in 2-CTA clusters sharing the W tile, 2 = 3xTF32 (fp32
        # range, the automatic fallback on fp16 overflow), 6 = 3xBF16 with bf16 weights; None: default_gemm_mode.
        if gemm_mode is None:
            gemm_mode = default_gemm_mode(state_dict)
        self.gemm_mode = int(gemm_mode)
        d = int(config.d_model)
        self.config = config
        self.device = int(device)
        cfg = BartConfig(int(config.vocab_size), d, int(config.encoder_layers), int(config.decoder_layers),
                         int(config.decoder_attention_heads), int(config.decoder_ffn_dim),
                         int(config.max_position_embeddings), int(bool(getattr(config, "scale_embedding", False))),
                         int(gemm_mode))
        if config.encoder_ffn_dim != config.decoder_ffn_dim or config.encoder_attention_heads != config.decoder_attention_heads:
            raise ValueError("encoder/decoder shapes must match (bart-large layout)")
        if getattr(config, "activation_function", "gelu") != "gelu":
            raise ValueError("only the exact-erf 'gelu' activation of bart-large is implemented")
        h = vp()
        check(lib.sealbart_create(C.byref(cfg), None, self.device, C.byref(h)))
        self._h = h.value
        _load_weights(self._h, state_dict, "model.shared.weight")

    @classmethod
    def from_hf(cls, model, device=None, gemm_mode=None):
        model_type = getattr(model.config, "model_type", None)
        if model_type == "t5":
            return SealT5Engine.from_hf(model, device=device, gemm_mode=gemm_mode)
        if model_type in PRELN_MODEL_TYPES:
            return SealPreLnEngine.from_hf(model, device=device, gemm_mode=gemm_mode)
        return cls(model.state_dict(), model.config, device=_hf_device(model) if device is None else device,
                   gemm_mode=gemm_mode)

    @property
    def max_positions(self):
        """the positions the decoder's position table covers (without BART's and mBART's offset of 2); None for T5,
        which has no table"""
        return int(self.config.max_position_embeddings)

    def __del__(self):
        h = self.__dict__.get("_h")
        if h:
            lib.sealbart_free(h)
            self._h = None

    def device_bytes(self):
        return int(lib.sealbart_device_bytes(self._h))

    def debug_step_logits(self, input_ids, attention_mask, num_beams, decoder_input_ids, anc=None, src_tokens=-1):
        """Teacher-forced logits of the last decoder position for explicit decoder inputs [R,t].
        anc: optional int32 [R,t] beam ancestry (row r reads the decoder cache of position s from row anc[r,s]);
        src_tokens: -1 pack right-padded sources, -2 never pack (include/sealdec.h sealdec_debug_step_logits)."""
        ids = np.ascontiguousarray(np.asarray(input_ids, dtype=np.int64))
        am = np.ascontiguousarray(np.asarray(attention_mask, dtype=np.int64))
        dec = np.ascontiguousarray(np.asarray(decoder_input_ids, dtype=np.int64))
        Q, S = ids.shape
        R, t = dec.shape
        assert R == Q * num_beams
        a = None
        if anc is not None:
            a = np.ascontiguousarray(np.asarray(anc, dtype=np.int32))
            assert a.shape == (R, t)
        out = np.empty((R, int(self.config.vocab_size)), dtype=np.float32)
        check(lib.sealdec_debug_step_logits(self._h, ids.ctypes.data, am.ctypes.data, Q, S, num_beams,
                                            dec.ctypes.data, t, a.ctypes.data if a is not None else None,
                                            int(src_tokens), out.ctypes.data))
        return out

    def stat(self, name):
        """sealbart_get_stat (include/sealdec.h), e.g. "last_paths"."""
        return int(lib.sealbart_get_stat(self._h, name.encode()))

    def set_option(self, name, value):
        check(lib.sealbart_set_option(self._h, name.encode(), int(value)))

    def last_phase_us(self):
        a = (C.c_double * 5)()
        check(lib.sealdec_last_phase_us(self._h, a))
        return {"encoder": a[0], "decoder_layers": a[1], "lm_head": a[2], "select_expand": a[3], "total": a[4]}

    def profile_gemm(self, enable):
        """Enable/disable CUDA-event bracketing of every GEMM launch; returns the record so far."""
        us = C.c_double(0); n = C.c_int64(0); fl = C.c_double(0)
        check(lib.sealdec_profile_gemm(self._h, int(bool(enable)), C.byref(us), C.byref(n), C.byref(fl)))
        return {"total_us": us.value, "launches": n.value, "flops": fl.value}

    def last_launch_count(self):
        """kernel launches of the last generate / teacher-forced / debug-step call (the "launches" stat)"""
        return self.stat("launches")


T5_FFN_KINDS = {"relu": 0, "gated-gelu": 1}      # sealt5_config_t.ffn_kind


class T5ConfigView:
    """A T5 config as the decode reads it, resolved the way transformers 4.13 (the reference's pin) sees a T5
    checkpoint: decoder_start_token_id from the config, else from the model's generation_config, else pad_token_id (0);
    forced_bos_token_id / forced_eos_token_id None where the attribute is missing; the decoder output scale
    d_model^-0.5 applied iff config.scale_decoder_outputs, or tie_word_embeddings where that attribute is missing.
    Every other attribute is the HF config's."""

    def __init__(self, config, generation_config=None):
        self._hf = config
        start = getattr(config, "decoder_start_token_id", None)
        if start is None and generation_config is not None:
            start = getattr(generation_config, "decoder_start_token_id", None)
        if start is None:
            start = config.pad_token_id
        self.decoder_start_token_id = int(start)
        self.forced_bos_token_id = getattr(config, "forced_bos_token_id", None)
        self.forced_eos_token_id = getattr(config, "forced_eos_token_id", None)
        self.bos_token_id = getattr(config, "bos_token_id", None)
        scale = getattr(config, "scale_decoder_outputs", None)
        self.scale_decoder_outputs = bool(config.tie_word_embeddings if scale is None else scale)

    def __getattr__(self, name):
        return getattr(self.__dict__["_hf"], name)


def t5_native_config(config, gemm_mode):
    """sealt5_config_t for an HF T5Config; ValueError for a shape or feed-forward the kernels do not cover (the same
    limits sealt5_create enforces, include/sealdec.h), before anything touches the device."""
    d, heads, d_kv, d_ff = int(config.d_model), int(config.num_heads), int(config.d_kv), int(config.d_ff)
    proj = getattr(config, "feed_forward_proj", "relu")
    if proj not in T5_FFN_KINDS:
        raise ValueError(f"T5 feed_forward_proj {proj!r} is not implemented (supported: {sorted(T5_FFN_KINDS)})")
    if d_kv != 64 or heads * 64 != d:
        raise ValueError(f"T5 shape not covered: d_kv must be 64 and num_heads * 64 == d_model (d_kv={d_kv}, "
                         f"num_heads={heads}, d_model={d})")
    if not (d > 0 and d % 128 == 0 and d <= 1024) and not (d > 0 and d % 1024 == 0 and d <= 4096):
        raise ValueError(f"T5 shape not covered: d_model must be a multiple of 128 up to 1 024, or a multiple of 1 024 "
                         f"up to 4 096 (d_model={d})")
    if d_ff % 64:
        raise ValueError(f"T5 shape not covered: d_ff must be a multiple of 64 (d_ff={d_ff})")
    nb = int(config.relative_attention_num_buckets)
    md = int(getattr(config, "relative_attention_max_distance", 128))
    if not 4 <= nb <= 1024 or md <= nb // 2:
        raise ValueError(f"T5 relative attention buckets not covered: num_buckets must be in [4, 1024] and "
                         f"max_distance > num_buckets / 2 (num_buckets={nb}, max_distance={md})")
    view = T5ConfigView(config)
    n_dec = getattr(config, "num_decoder_layers", None)
    return T5Config(int(config.vocab_size), d, int(config.num_layers), int(n_dec if n_dec is not None else config.num_layers),
                    heads, d_kv, d_ff, T5_FFN_KINDS[proj], nb, md, float(config.layer_norm_epsilon),
                    int(view.scale_decoder_outputs), int(gemm_mode))


class SealT5Engine(SealBartEngine):
    """Device-resident T5 weights + workspace behind the same handle (include/sealdec.h `sealt5_create`): every method
    of SealBartEngine, and every entry point that takes an engine, works the same way.  `config` is a T5ConfigView."""

    max_positions = None

    def __init__(self, state_dict, config, device=0, gemm_mode=None, generation_config=None):
        if gemm_mode is None:
            gemm_mode = default_gemm_mode(state_dict)
        cfg = t5_native_config(config, gemm_mode)
        self.gemm_mode = int(gemm_mode)
        self.config = T5ConfigView(config, generation_config)
        self.device = int(device)
        h = vp()
        check(lib.sealt5_create(C.byref(cfg), self.device, C.byref(h)))
        self._h = h.value
        _load_weights(self._h, state_dict, "shared.weight")

    @classmethod
    def from_hf(cls, model, device=None, gemm_mode=None):
        t5_native_config(model.config, 3 if gemm_mode is None else gemm_mode)      # ValueError before any device work
        return cls(model.state_dict(), model.config, device=_hf_device(model) if device is None else device,
                   gemm_mode=gemm_mode, generation_config=getattr(model, "generation_config", None))


PRELN_MODEL_TYPES = ("pegasus", "mbart")          # HF model types of the pre-LayerNorm BART family
PRELN_ACTIVATIONS = {"gelu": 0, "relu": 1}         # sealbart_variant_t.activation (SEALBART_ACT_GELU / _RELU)


class PreLnConfigView:
    """A Pegasus / mBART config as the decode reads it, resolved the way transformers 4.13 (the reference's pin) does for
    fm_index_generate: decoder_start_token_id from the config, else bos_token_id, else the ValueError of
    `_get_decoder_start_token_id`; forced_eos_token_id from the config (1 for Pegasus, 2 for mBART), which feeds the
    ForcedEOS rule; forced_bos_token_id None where the attribute is missing.  Every other attribute is the HF config's."""

    def __init__(self, config):
        self._hf = config
        start = getattr(config, "decoder_start_token_id", None)
        if start is None:
            start = getattr(config, "bos_token_id", None)
        if start is None:
            raise ValueError("`decoder_start_token_id` or `bos_token_id` has to be defined for encoder-decoder generation.")
        self.decoder_start_token_id = int(start)
        self.forced_bos_token_id = getattr(config, "forced_bos_token_id", None)
        self.forced_eos_token_id = getattr(config, "forced_eos_token_id", None)

    def __getattr__(self, name):
        return getattr(self.__dict__["_hf"], name)


def preln_native_config(config, gemm_mode):
    """(sealbart_config_t, sealbart_variant_t) for an HF Pegasus or mBART config; ValueError for an activation or shape
    the kernels do not cover (the limits sealbart_create enforces, include/sealdec.h), before anything touches the
    device."""
    mt = getattr(config, "model_type", None)
    if mt not in PRELN_MODEL_TYPES:
        raise ValueError(f"model_type {mt!r} is not a pre-LayerNorm BART-family model (supported: {list(PRELN_MODEL_TYPES)})")
    act = getattr(config, "activation_function", "gelu")
    if act not in PRELN_ACTIVATIONS:
        raise ValueError(f"{mt} activation_function {act!r} is not implemented (supported: {sorted(PRELN_ACTIVATIONS)})")
    d = int(config.d_model)
    heads, ffn = int(config.decoder_attention_heads), int(config.decoder_ffn_dim)
    if int(config.encoder_attention_heads) != heads or int(config.encoder_ffn_dim) != ffn:
        raise ValueError(f"{mt} shape not covered: encoder and decoder must have the same heads and ffn_dim "
                         f"(encoder {config.encoder_attention_heads} / {config.encoder_ffn_dim}, decoder {heads} / {ffn})")
    if not (0 < d <= 1024 and d % 128 == 0) or heads * 64 != d:
        raise ValueError(f"{mt} shape not covered: d_model must be a multiple of 128 up to 1 024 with 64-wide heads "
                         f"(d_model={d}, heads={heads})")
    if ffn <= 0 or ffn % 64:
        raise ValueError(f"{mt} shape not covered: ffn_dim must be a positive multiple of 64 (ffn_dim={ffn})")
    P = int(config.max_position_embeddings)
    if P < 1:
        raise ValueError(f"{mt}: max_position_embeddings must be >= 1 (got {P})")
    cfg = BartConfig(int(config.vocab_size), d, int(config.encoder_layers), int(config.decoder_layers), heads, ffn, P,
                     int(bool(getattr(config, "scale_embedding", False))), int(gemm_mode))
    var = BartVariant(1, 2 if mt == "mbart" else 0, 1 if mt == "mbart" else 0, PRELN_ACTIVATIONS[act])
    return cfg, var


class SealPreLnEngine(SealBartEngine):
    """Device-resident Pegasus / mBART weights + workspace behind the same handle (include/sealdec.h
    `sealbart_create` with a `sealbart_variant_t`): every method of SealBartEngine, and every entry point that takes an
    engine, works the same way.  `config` is a PreLnConfigView."""

    def __init__(self, state_dict, config, device=0, gemm_mode=None):
        if gemm_mode is None:
            gemm_mode = default_gemm_mode(state_dict)
        cfg, var = preln_native_config(config, gemm_mode)
        self.config = PreLnConfigView(config)
        self.gemm_mode = int(gemm_mode)
        self.device = int(device)
        h = vp()
        check(lib.sealbart_create(C.byref(cfg), C.byref(var), self.device, C.byref(h)))
        self._h = h.value
        _load_weights(self._h, state_dict, "model.shared.weight")

    @classmethod
    def from_hf(cls, model, device=None, gemm_mode=None):
        preln_native_config(model.config, 3 if gemm_mode is None else gemm_mode)   # ValueError before any device work
        PreLnConfigView(model.config)
        return cls(model.state_dict(), model.config, device=_hf_device(model) if device is None else device,
                   gemm_mode=gemm_mode)


def _position_error():
    # what torch.nn.functional.embedding raises for an index past the position table (the reference's forward)
    return IndexError("index out of range in self")


def _check_decoder_positions(eng, max_length):
    """A generate that runs every step (keep_history=True, the record entry points) feeds decoder positions
    0 .. max_length - 2 (cur_len - 1 at cur_len = 1 .. max_length - 1, constrained_beam_search).  A model with a
    position table (BART, Pegasus, mBART) raises the reference's IndexError before any device work when the last one is
    past the table."""
    P = getattr(eng, "max_positions", None)
    if P is not None and int(max_length) - 2 >= P:
        raise _position_error()


_ENGINES = weakref.WeakKeyDictionary()


def _engine_for(model):
    """The engine of an HF model, built on first use and cached per model object and weight dtypes (a model converted
    in place, e.g. by `.to(torch.bfloat16)`, gets an engine of the new format)."""
    if isinstance(model, SealBartEngine):
        return model
    key = _weight_dtypes(model)
    hit = _ENGINES.get(model)
    if hit is None or hit[0] != key:
        hit = (key, SealBartEngine.from_hf(model))
        _ENGINES[model] = hit
    return hit[1]


def _make_params(cfg, num_beams, min_length, max_length, length_penalty, eos_token_id, force_decoding_from,
                 always_allow_eos, disable_fm_index, stop_at_count, forced_bos_token_id, top_k=0):
    force = list(force_decoding_from or [])
    farr = (C.c_int64 * max(len(force), 1))(*force)
    none = lambda x: -1 if x is None else int(x)
    p = DecParams(int(num_beams), int(min_length if min_length is not None else -1), int(max_length),
                  float(length_penalty), int(eos_token_id), int(cfg.pad_token_id), int(cfg.decoder_start_token_id),
                  none(cfg.eos_token_id), none(getattr(cfg, "forced_eos_token_id", None)), none(forced_bos_token_id),
                  int(stop_at_count), int(bool(always_allow_eos)), int(bool(disable_fm_index)), 1, len(force), farr, SHIFT,
                  int(top_k))
    p._keepalive = farr
    return p


def _check_diverse_groups(num_beams, diverse_bs_groups, diverse_bs_penalty):
    """The argument checks fm_index_generate's diverse-beam path meets before any decoding (seal/beam_search.py:447-454,
    :597-601): transformers 4.13's HammingDiversityLogitsProcessor constructor when the penalty applies, then
    BeamSearchScorerWithMemory's group check.  Same exception type and message."""
    if diverse_bs_groups > 1 and diverse_bs_penalty > 0.0:
        if not isinstance(diverse_bs_penalty, float):
            raise ValueError("`diversity_penalty` should be a float strictly larger than 0.")
        if not isinstance(num_beams, int) or num_beams < 2:
            raise ValueError("`num_beams` should be an integer strictly larger than 1.")
        if diverse_bs_groups > num_beams:
            raise ValueError("`beam_groups` has to be smaller or equal to `num_beams`.")
    if (not isinstance(diverse_bs_groups, int) or diverse_bs_groups > num_beams or num_beams % diverse_bs_groups != 0
            or diverse_bs_groups < 1):
        raise ValueError(
            f"`num_beam_groups` has to be an integer smaller or equal than `num_beams` and `num_beams` "
            f"has to be divisible by `num_beam_groups`, but is {diverse_bs_groups} with `num_beams` being {num_beams}.")


def _check_topk(topk, diverse_bs_groups):
    """fm_index_generate's `topk` as the kernels take it (include/sealdec.h sealdec_params_t.top_k), checked the way the
    reference meets it before its first step (seal/beam_search.py:163-164, :249-250): a falsy value is off (None too,
    where the reference would raise a TypeError at `topk > 0`); a positive value goes through transformers'
    TopKLogitsWarper constructor (`True` is the int 1); a negative one leaves `topk_warper` unbound.  Diverse beam groups
    run group_beam_search, which never sees topk (:523-532): then it is neither checked nor used."""
    if diverse_bs_groups > 1 or not topk:
        return 0
    if topk > 0:
        if not isinstance(topk, int):
            raise ValueError(f"`top_k` has to be a strictly positive integer, but is {topk}")
        return int(topk)
    raise UnboundLocalError("cannot access local variable 'topk_warper' where it is not associated with a value")


def _group_params(num_beam_groups, diversity_penalty):
    # a penalty <= 0 means no Hamming processor (seal/beam_search.py:447)
    return GroupParams(int(num_beam_groups), float(diversity_penalty) if diversity_penalty > 0.0 else 0.0)


def generate_records(model, index, input_ids, attention_mask, min_length=3, max_length=25, length_penalty=1.0,
                     num_beams=3, eos_token_id=None, force_decoding_from=None, always_allow_eos=False,
                     disable_fm_index=False, stop_at_count=0, forced_bos_token_id="config", want_ranges=True,
                     num_beam_groups=1, diversity_penalty=0.0, top_k=0):
    """The C-ABI call with HOST buffers (sealdec_generate): returns the packed hypothesis records
    (scores [Q,H] f32, lens [Q,H] i32, tokens [Q,H,T] i32, valid [Q,H] u8, lo/hi [Q,H] u64).
    num_beam_groups > 1: diverse beam groups (include/sealdec.h sealdec_groups_t), records group by group per step.
    top_k > 0: the top-k logits warp on every step (sealdec_params_t.top_k; one group only)."""
    eng = _engine_for(model)
    _check_decoder_positions(eng, max_length)
    cfg = eng.config
    if forced_bos_token_id == "config":
        forced_bos_token_id = getattr(cfg, "forced_bos_token_id", None)
    if eos_token_id is None:
        eos_token_id = cfg.eos_token_id
    ids = np.ascontiguousarray(np.asarray(input_ids.cpu() if hasattr(input_ids, "cpu") else input_ids, dtype=np.int64))
    am = np.ascontiguousarray(np.asarray(attention_mask.cpu() if hasattr(attention_mask, "cpu") else attention_mask, dtype=np.int64))
    Q, S = ids.shape
    p = _make_params(cfg, num_beams, min_length, max_length, length_penalty, eos_token_id, force_decoding_from,
                     always_allow_eos, disable_fm_index, stop_at_count, forced_bos_token_id, top_k)
    H = int(lib.sealdec_hyps_per_query(C.byref(p)))
    T = int(max_length)
    scores = np.empty((Q, H), dtype=np.float32); lens = np.empty((Q, H), dtype=np.int32)
    toks = np.empty((Q, H, T), dtype=np.int32); valid = np.empty((Q, H), dtype=np.uint8)
    lo = np.zeros((Q, H), dtype=np.uint64) if want_ranges else None
    hi = np.zeros((Q, H), dtype=np.uint64) if want_ranges else None
    fm_h = None
    occ_ptr = None
    if not disable_fm_index:
        if index._device is None:
            index.to_device(eng.device)
        fm_h = index._dev()
        occ = _occurring_mask(index, int(cfg.vocab_size))
        occ_ptr = occ.ctypes.data
    grp = _group_params(num_beam_groups, diversity_penalty)
    check(lib.sealdec_generate(eng._h, fm_h, occ_ptr, C.byref(p), ids.ctypes.data, am.ctypes.data, Q, S,
                               scores.ctypes.data, lens.ctypes.data, toks.ctypes.data, valid.ctypes.data,
                               lo.ctypes.data if want_ranges else None, hi.ctypes.data if want_ranges else None,
                               C.byref(grp)))
    return {"scores": scores, "lens": lens, "tokens": toks, "valid": valid, "lo": lo, "hi": hi}


class DeviceRecords:
    """The hypothesis records of one generate call in ONE device buffer (sharding.RecordLayout): the decode
    kernels write into it, `sharding.gather_buffers` moves it (NCCL, device to device), `.host()` reads it."""

    def __init__(self, layout, device):
        torch = _torch()
        self.layout = layout
        self.buf = torch.zeros(layout.nbytes, dtype=torch.uint8, device=device)
        self._base = self.buf.data_ptr()

    def ptr(self, name):
        return self._base + self.layout.offsets[name][0]

    @property
    def err_ptr(self):
        return self._base + self.layout.err_offset

    def set_filled(self, n):
        torch = _torch()
        self.buf[:8] = torch.from_numpy(np.asarray([n], dtype=np.int64).view(np.uint8)).to(self.buf.device)

    def host(self):
        """Blocking read-back: dict of numpy arrays (first dim = the queries filled) + 'errors'."""
        from .sharding import merge_gathered
        return merge_gathered([self.buf], self.layout)


def _side_stream(device):
    """One non-default stream per device for the asynchronous entry points (CUDA graphs cannot be captured on the
    legacy default stream, which is what torch.cuda.current_stream() is unless the caller changed it)."""
    torch = _torch()
    cache = _side_stream.__dict__.setdefault("cache", {})
    key = torch.device(device).index if not isinstance(device, int) else device
    if key not in cache:
        cache[key] = torch.cuda.Stream(device=key)
    return cache[key]


def generate_records_device(model, index, input_ids_d, attention_mask_d, min_length=3, max_length=25, length_penalty=1.0,
                            num_beams=3, eos_token_id=None, force_decoding_from=None, always_allow_eos=False,
                            disable_fm_index=False, stop_at_count=0, forced_bos_token_id="config", out=None,
                            src_tokens=-1, stream=None, num_beam_groups=1, diversity_penalty=0.0, top_k=0,
                            check_positions=True):
    """sealdec_generate_dx on DEVICE tensors, asynchronous: input_ids / attention_mask are int64 CUDA tensors
    [Q, S]; the records land in `out` (a DeviceRecords, created if None) on `stream` (default: the current stream if
    it is not the legacy default stream, else a per-device side stream that first waits for the current one).
    `src_tokens`: number of non-zero mask entries if the caller knows it (right-padded masks) — then the call never
    touches the host; -1 = unknown.  Errors are flags inside the buffer (`out.host()["errors"]`, include/sealdec.h).
    `num_beam_groups` / `diversity_penalty` / `top_k`: diverse beam groups and the top-k warp, as in generate_records.
    `check_positions`: raise IndexError for a max_length whose decoder positions pass a bounded position table (Pegasus,
    mBART), as generate_records does; False leaves it to the caller (fm_index_generate with keep_history=False, whose
    stock scorer may stop before those steps)."""
    torch = _torch()
    from .sharding import RecordLayout
    eng = _engine_for(model)
    if check_positions:
        _check_decoder_positions(eng, max_length)
    cfg = eng.config
    if forced_bos_token_id == "config":
        forced_bos_token_id = getattr(cfg, "forced_bos_token_id", None)
    if eos_token_id is None:
        eos_token_id = cfg.eos_token_id
    if not (input_ids_d.is_cuda and attention_mask_d.is_cuda) or input_ids_d.dtype != torch.int64 or attention_mask_d.dtype != torch.int64:
        raise TypeError("generate_records_device takes int64 CUDA tensors (use generate_records for host arrays)")
    ids = input_ids_d.contiguous(); am = attention_mask_d.contiguous()
    Q, S = ids.shape
    p = _make_params(cfg, num_beams, min_length, max_length, length_penalty, eos_token_id, force_decoding_from,
                     always_allow_eos, disable_fm_index, stop_at_count, forced_bos_token_id, top_k)
    H = int(lib.sealdec_hyps_per_query(C.byref(p)))
    dev = ids.device
    if out is None:
        out = DeviceRecords(RecordLayout(Q, H, int(max_length)), dev)
    lay = out.layout
    if lay.H != H or lay.T != int(max_length) or lay.Q < Q:
        raise ValueError("record buffer layout does not fit this call")
    fm_h = None; occ_ptr = None
    if not disable_fm_index:
        if index._device is None:
            index.to_device(eng.device)
        fm_h = index._dev()
        occ = _occurring_mask(index, int(cfg.vocab_size), dev)
        occ_ptr = occ.data_ptr()
    with torch.cuda.device(dev):
        cur = torch.cuda.current_stream()
        if stream is None:
            stream = cur if cur.cuda_stream != 0 else _side_stream(dev)
        if stream.cuda_stream != cur.cuda_stream:
            stream.wait_stream(cur)
        grp = _group_params(num_beam_groups, diversity_penalty)
        with torch.cuda.stream(stream):
            out.set_filled(Q)
            check(lib.sealdec_generate_dx(eng._h, fm_h, occ_ptr, C.byref(p), ids.data_ptr(), am.data_ptr(), Q, S,
                                          stream.cuda_stream, out.ptr("scores"), out.ptr("lens"), out.ptr("tokens"),
                                          out.ptr("valid"), out.ptr("lo"), out.ptr("hi"), out.err_ptr, int(src_tokens),
                                          C.byref(grp)))
        for t in (ids, am, out.buf):
            t.record_stream(stream)
        if stream.cuda_stream != cur.cuda_stream:
            cur.wait_stream(stream)
    return out


def sharded_generate_records(model, index, input_ids, attention_mask, group=None, dst=0, **kw):
    """N-GPU generate: this rank decodes its contiguous block of the batch (host arrays in, as SEALSearcher holds
    them), the records stay on the device and ONE NCCL gather brings every rank's buffer to `dst`
    (SURVEY.md section 8e).  Returns the full-batch record arrays on `dst`, None elsewhere.  `kw` are
    generate_records_device's arguments, num_beam_groups / diversity_penalty / top_k included (same record layout)."""
    torch = _torch()
    from .sharding import sharded_generate
    eng = _engine_for(model)
    dev = torch.device("cuda", eng.device)
    ids_np = np.ascontiguousarray(np.asarray(input_ids, dtype=np.int64)); am_np = np.ascontiguousarray(np.asarray(attention_mask, dtype=np.int64))
    cfg = eng.config
    p = _make_params(cfg, kw.get("num_beams", 3), kw.get("min_length", 3), kw.get("max_length", 25), kw.get("length_penalty", 1.0),
                     kw.get("eos_token_id") or cfg.eos_token_id, kw.get("force_decoding_from"), False, False, 0, None)
    H = int(lib.sealdec_hyps_per_query(C.byref(p)))

    def fill(ids_blk, am_blk, layout):
        # per-engine staging: the same device buffers (inputs and record buffer) serve every call of a shape, so that
        # small shards replay the captured CUDA graph of the call instead of launching ~1 900 kernels eagerly
        cache = eng.__dict__.setdefault("_io_cache", {})
        n = len(ids_blk)
        key = (layout.Q, layout.H, layout.T, n, ids_blk.shape[1] if n else 0)
        if key not in cache:
            if len(cache) >= 8:
                cache.pop(next(iter(cache)))
            cache[key] = (DeviceRecords(layout, dev),
                          torch.empty((max(n, 1), ids_np.shape[1]), dtype=torch.int64, device=dev),
                          torch.empty((max(n, 1), ids_np.shape[1]), dtype=torch.int64, device=dev))
        rec, ids_d, am_d = cache[key]
        if n:
            right_padded = bool((np.diff(am_blk != 0, axis=1) <= 0).all()) and bool((am_blk[:, 0] != 0).all())
            ids_d.copy_(torch.from_numpy(ids_blk)); am_d.copy_(torch.from_numpy(am_blk))
            generate_records_device(eng, index, ids_d, am_d, out=rec,
                                    src_tokens=int((am_blk != 0).sum()) if right_padded else -2, **kw)
        else:
            rec.set_filled(0)
        return rec.buf

    return sharded_generate(fill, ids_np, am_np, H, int(kw.get("max_length", 25)), group=group, dst=dst)


def records_to_output(rec, length_penalty):
    """beam_search.py:555: [(score * len**lp, tokens) for every recorded hyp with score > -inf].
    The arithmetic is vectorised (float64, like the reference's Python floats; len**lp comes from a table filled
    with Python's own pow so that every bit matches); only the final tuples are built in a Python loop."""
    scores, lens, toks = rec["scores"], rec["lens"], rec["tokens"]
    Q = scores.shape[0]
    if scores.size == 0:
        return [[] for _ in range(Q)]
    pen_table = np.array([float(n) ** length_penalty if n > 0 else 1.0 for n in range(int(lens.max()) + 1)], dtype=np.float64)
    pen = pen_table[lens]
    hyp = scores.astype(np.float64) / pen                             # BeamHypothesesWithMemory.add, :752-755
    final = hyp * pen
    valid = hyp > float("-inf")
    # one flat list of the kept tokens (prefixes of the kept hypotheses), sliced per hypothesis
    n_kept = np.where(valid, lens, 0)
    keep_tok = valid[:, :, None] & (np.arange(toks.shape[2])[None, None, :] < lens[:, :, None])
    flat = toks[keep_tok].tolist()
    ends = np.cumsum(n_kept.reshape(-1)[valid.reshape(-1)]).tolist()
    fs = final[valid].tolist()
    per_query = valid.sum(axis=1).tolist()
    out = []
    i = 0; start = 0
    for cnt in per_query:
        row = []
        for j in range(i, i + cnt):
            e = ends[j]
            row.append((fs[j], flat[start:e]))
            start = e
        out.append(row)
        i += cnt
    return out


def _replay_beam_search_scorer(rec, num_beams, length_penalty, eos_token_id, pad_token_id, max_length, n_positions=None):
    """keep_history=False (seal/beam_search.py:505-515): the reference hands the loop transformers 4.13's stock
    `BeamSearchScorer` instead of BeamSearchScorerWithMemory.  Both choose the next beams the same way (the first
    num_beams non-EOS candidates of the top 2*num_beams), so the beams evolve identically until a query is `done`,
    after which the stock scorer freezes it (pads) and `finalize` skips it.  The device path therefore runs the very
    same kernels, and the stock scorer's bookkeeping -- BeamHypotheses.add / worst_score / is_done, process's
    "EOS only if ranked inside the top num_beams", finalize's best-num_beams selection with an appended EOS -- is
    replayed here, on the host, over the per-step candidate records (a few thousand scalar operations per query).
    Returns (beams per query [(score, tokens)] in BeamHypotheses order, sequences int64 [Q*num_beams, L],
    sequence_scores float32 [Q*num_beams]).  transformers 4.13 is not vendored: restated from its published algorithm.
    n_positions: the decoder's position table rows (None: unbounded).  The reference runs step `st` (decoder position
    st) while some query is not done, so a query still alive at step st >= n_positions means its forward read past the
    table: IndexError, unless a query failed the num_beams check at an earlier step, which the reference meets first."""
    scores, lens, toks = rec["scores"], rec["lens"], rec["tokens"]
    Q, H = scores.shape
    B, K = num_beams, 2 * num_beams
    n_steps = (H - B) // K
    all_beams, best, best_scores = [], [], []
    fail_step, past_table = None, False          # the first step that fails the num_beams check; a step past the table
    for q in range(Q):
        beams = []; worst = 1e9; done = False; stopped = False

        def add(tokens, sum_logprobs):
            nonlocal worst
            score = sum_logprobs / (len(tokens) ** length_penalty)
            if len(beams) < B or score > worst:
                beams.append((score, tokens))
                if len(beams) > B:
                    order = sorted((sc, i) for i, (sc, _) in enumerate(beams))
                    del beams[order[0][1]]
                    worst = order[1][0]
                else:
                    worst = min(score, worst)

        for st in range(n_steps):
            if done:
                break
            if n_positions is not None and st >= n_positions:
                past_table = stopped = True
                break
            cur_len = st + 1
            base = st * K
            cand_s = scores[q, base:base + K].tolist()
            nb = 0
            for rank in range(K):
                h = base + rank
                tok = int(toks[q, h, cur_len])
                if tok == eos_token_id:
                    if rank < B:
                        add(toks[q, h, :cur_len].tolist(), cand_s[rank])
                else:
                    nb += 1
                if nb == B:
                    break
            if nb < B:
                fail_step = st if fail_step is None else min(fail_step, st)
                stopped = True
                break
            if len(beams) >= B:
                done = worst >= max(cand_s) / cur_len ** length_penalty
        if stopped:
            continue
        if not done:
            fb = n_steps * K
            for j in range(B):
                add(toks[q, fb + j, :lens[q, fb + j]].tolist(), float(scores[q, fb + j]))
        all_beams.append(list(beams))
        order = sorted(beams, key=lambda x: x[0])
        for _ in range(B):
            sc, t = order.pop()
            best.append(t); best_scores.append(sc)
    if past_table and (fail_step is None or fail_step >= n_positions):
        raise _position_error()
    if fail_step is not None:
        raise ValueError(f"At most {B} tokens can be equal to `eos_token_id: {eos_token_id}`.")
    L = min(max(len(t) for t in best) + 1, max_length) if best else 0
    seq = np.full((len(best), L), pad_token_id, dtype=np.int64)
    for i, t in enumerate(best):
        seq[i, :len(t)] = t
        if len(t) < max_length:
            seq[i, len(t)] = eos_token_id
    return all_beams, seq, np.asarray(best_scores, dtype=np.float32)


def fm_index_generate(model, index: FMIndex, input_ids, attention_mask, min_length: int = 3, max_length: int = 25,
                      length_penalty: float = 1.0, num_beams: int = 3, diverse_bs_groups: int = 1,
                      diverse_bs_penalty: float = 0.0, eos_token_id: Optional[int] = None,
                      force_decoding_from: Optional[List[int]] = None, always_allow_eos: bool = False,
                      keep_history: bool = False, disable_fm_index: bool = False, sample: bool = False,
                      stop_at_count: int = 0, topk: int = 0, transformers_output: bool = False, **kwargs):
    """beam_search.py:391-557.  `model` is an HF BartForConditionalGeneration (its weights are
    mirrored on the GPU once and cached) or a SealBartEngine."""
    if sample:
        raise NotImplementedError("sampling is outside the constrained-decoding hot path")
    _check_diverse_groups(num_beams, diverse_bs_groups, diverse_bs_penalty)
    top_k = _check_topk(topk, diverse_bs_groups)
    if diverse_bs_groups > 1 and not keep_history:
        raise NotImplementedError("diverse_bs_groups > 1 with keep_history=False (transformers' stock grouped BeamSearchScorer) "
                                  "is not implemented; keep_history=True, the path SEALSearcher uses, is")
    forced_bos = kwargs.pop("forced_bos_token_id", "config")                     # :415-418
    torch = _torch()
    if keep_history:
        rec = generate_records(model, index, input_ids, attention_mask, min_length, max_length, length_penalty,
                               num_beams, eos_token_id, force_decoding_from, always_allow_eos, disable_fm_index,
                               stop_at_count, forced_bos, want_ranges=False, num_beam_groups=diverse_bs_groups,
                               diversity_penalty=diverse_bs_penalty, top_k=top_k)
        if transformers_output:
            # BeamSearchScorerWithMemory.finalize returns an UNINITIALISED [Q*num_beams, 3] tensor as `sequences`
            # (:727); zeros of that shape here
            return torch.zeros((rec["scores"].shape[0] * num_beams, 3), dtype=torch.long,
                               device=input_ids.device if hasattr(input_ids, "device") else "cpu")
        return records_to_output(rec, length_penalty)
    # ---- keep_history=False: transformers' stock BeamSearchScorer (:505-515), the reference's default --------------
    eng = _engine_for(model)
    cfg = eng.config
    eos = cfg.eos_token_id if eos_token_id is None else eos_token_id
    dev = torch.device("cuda", eng.device)
    ids_np = np.ascontiguousarray(np.asarray(input_ids.cpu() if hasattr(input_ids, "cpu") else input_ids, dtype=np.int64))
    am_np = np.ascontiguousarray(np.asarray(attention_mask.cpu() if hasattr(attention_mask, "cpu") else attention_mask, dtype=np.int64))
    out = generate_records_device(eng, index, torch.from_numpy(ids_np).to(dev), torch.from_numpy(am_np).to(dev), min_length,
                                  max_length, length_penalty, num_beams, eos_token_id, force_decoding_from, always_allow_eos,
                                  disable_fm_index, stop_at_count, forced_bos, src_tokens=-2, top_k=top_k, check_positions=False)
    rec = out.host()
    if rec["errors"][1] and eng.gemm_mode in (3, 5):   # fp16 range exceeded: redo with the 3xTF32 kernels (sealdec.h)
        check(lib.sealbart_set_option(eng._h, b"gemm_mode", 2))
        try:
            rec = generate_records_device(eng, index, torch.from_numpy(ids_np).to(dev), torch.from_numpy(am_np).to(dev), min_length,
                                          max_length, length_penalty, num_beams, eos_token_id, force_decoding_from, always_allow_eos,
                                          disable_fm_index, stop_at_count, forced_bos, src_tokens=-2, top_k=top_k,
                                          check_positions=False).host()
        finally:
            check(lib.sealbart_set_option(eng._h, b"gemm_mode", eng.gemm_mode))
    # the device's "fewer than num_beams non-EOS candidates" flag also fires for queries the stock scorer had already
    # frozen; the replay re-derives the condition per query and step and raises exactly where the reference does
    # with a bounded position table (Pegasus, mBART) the replay raises IndexError where the reference's forward would
    # first read past it; the steps the kernels ran there (on the table's last row) are never read
    beams, seq, _ = _replay_beam_search_scorer(rec, num_beams, length_penalty, eos, cfg.pad_token_id, int(max_length),
                                               n_positions=getattr(eng, "max_positions", None))
    if transformers_output:
        return torch.from_numpy(seq).to(input_ids.device if hasattr(input_ids, "device") else "cpu")     # :388
    return [[(sc * (len(t) ** length_penalty), t) for sc, t in b if sc > float("-inf")] for b in beams]    # :555
