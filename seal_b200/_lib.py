"""ctypes loader for the C-ABI shared library (include/sealfm.h, include/sealdec.h).

The library is the product; there is NO Python/CPU fallback.  If libsealb200.so is missing or a
symbol cannot be resolved, importing this module raises — loudly, on purpose.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsealb200.so")

u64 = C.c_uint64
u32 = C.c_uint32
i32 = C.c_int
vp = C.c_void_p
cp = C.c_char_p


class SealB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[sealb200 {code}] {msg}")
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C seal_b200/csrc`. seal_b200 has no CPU fallback.")
    return C.CDLL(LIB_PATH)


lib = _load()


class BuildOpts(C.Structure):             # sealfm_build_opts_t
    _fields_ = [("device_budget_bytes", C.c_uint64), ("chunk_elems", C.c_uint64), ("force_wide", C.c_int32),
                ("reserved", C.c_int32 * 7)]


class BuildStats(C.Structure):            # sealfm_build_stats_t
    _fields_ = [("chunk_elems", C.c_uint64), ("windows", C.c_uint64), ("max_windows_per_round", C.c_uint64),
                ("spanning_groups", C.c_uint64), ("giant_groups", C.c_uint64), ("key_partitions", C.c_uint64),
                ("single_key_buckets", C.c_uint64), ("device_peak_bytes", C.c_uint64), ("host_pinned_bytes", C.c_uint64),
                ("wide", C.c_uint32), ("text_bytes", C.c_uint32), ("rounds", C.c_uint32), ("reserved", C.c_uint32),
                ("phase_s", C.c_double * 4), ("round_unsorted", C.c_uint64 * 48), ("round_s", C.c_double * 48)]


# name -> (restype, argtypes); mirrors include/sealfm.h one to one
_FM_SIGS = {
    "sealfm_last_error": (cp, []),
    "sealfm_abi_version": (i32, []),
    "sealfm_build": (i32, [vp, u64, C.POINTER(vp)]),
    "sealfm_build_gpu": (i32, [vp, u64, i32, C.POINTER(vp)]),
    "sealfm_build_gpu_ex": (i32, [vp, u64, i32, i32, C.POINTER(BuildOpts), C.POINTER(vp)]),
    "sealfm_build_gpu_ex_stats": (i32, [C.POINTER(BuildStats)]),
    "sealfm_save_sdsl": (i32, [vp, cp]),
    "sealfm_from_sections": (i32, [u64, u32, u64, vp, u64, vp, vp, vp, u64, vp, u64, C.POINTER(vp)]),
    "sealfm_build_from_file": (i32, [cp, i32, C.POINTER(vp)]),
    "sealfm_load": (i32, [cp, C.POINTER(vp)]),
    "sealfm_save": (i32, [vp, cp]),
    "sealfm_free": (None, [vp]),
    "sealfm_size": (u64, [vp]),
    "sealfm_sigma": (u64, [vp]),
    "sealfm_max_level": (u32, [vp]),
    "sealfm_section": (i32, [vp, i32, C.POINTER(C.POINTER(u64)), C.POINTER(u64)]),
    "sealfm_to_device": (i32, [vp, i32]),
    "sealfm_device": (i32, [vp]),
    "sealfm_device_bytes": (u64, [vp]),
    "sealfm_set_beginnings": (i32, [vp, vp, u64]),
    "sealfm_backward_search_step": (i32, [vp, u64, vp, vp, vp, vp, vp]),
    "sealfm_backward_search_multi": (i32, [vp, u64, vp, vp, vp, vp]),
    "sealfm_distinct_count_multi": (i32, [vp, u64, vp, vp, vp, vp, u64]),
    "sealfm_locate": (i32, [vp, u64, vp, vp]),
    "sealfm_doc_index_from_rows": (i32, [vp, u64, vp, vp]),
    "sealfm_extract_text": (i32, [vp, u64, vp, vp, vp, vp, u64]),
    "sealfm_backward_search_step_d": (i32, [vp, vp, u64, vp, vp, vp, vp, vp]),
    "sealfm_expand_mask_d": (i32, [vp, vp, u64, vp, vp, vp, u32, u32, u32]),
    "sealfm_debug_sector_probe": (i32, [u64, u64, i32, C.POINTER(C.c_double)]),
}


f32p = C.POINTER(C.c_float)


class ProcessorCfg(C.Structure):          # sealdec_processor_cfg_t
    _fields_ = [("num_beams", C.c_int32), ("pad_token_id", C.c_int32), ("eos_token_id", C.c_int32),
                ("stop_at_count", C.c_int32), ("always_allow_eos", C.c_int32), ("forced_bos_token_id", C.c_int32),
                ("n_force_decoding_from", C.c_int32), ("force_decoding_from", C.POINTER(C.c_int64)),
                ("shift", C.c_int32)]


class BartConfig(C.Structure):            # sealbart_config_t
    _fields_ = [("vocab_size", C.c_int32), ("d_model", C.c_int32), ("encoder_layers", C.c_int32),
                ("decoder_layers", C.c_int32), ("heads", C.c_int32), ("ffn_dim", C.c_int32),
                ("max_positions", C.c_int32), ("scale_embedding", C.c_int32), ("gemm_mode", C.c_int32)]


class BartVariant(C.Structure):           # sealbart_variant_t
    _fields_ = [("pre_layer_norm", C.c_int32), ("position_offset", C.c_int32), ("layernorm_embedding", C.c_int32),
                ("activation", C.c_int32)]


class T5Config(C.Structure):              # sealt5_config_t
    _fields_ = [("vocab_size", C.c_int32), ("d_model", C.c_int32), ("num_layers", C.c_int32),
                ("num_decoder_layers", C.c_int32), ("num_heads", C.c_int32), ("d_kv", C.c_int32), ("d_ff", C.c_int32),
                ("ffn_kind", C.c_int32), ("relative_attention_num_buckets", C.c_int32),
                ("relative_attention_max_distance", C.c_int32), ("layer_norm_epsilon", C.c_float),
                ("scale_decoder_outputs", C.c_int32), ("gemm_mode", C.c_int32)]


class DecParams(C.Structure):             # sealdec_params_t
    _fields_ = [("num_beams", C.c_int32), ("min_length", C.c_int32), ("max_length", C.c_int32),
                ("length_penalty", C.c_float), ("eos_token_id", C.c_int32), ("pad_token_id", C.c_int32),
                ("decoder_start_token_id", C.c_int32), ("model_eos_token_id", C.c_int32),
                ("forced_eos_token_id", C.c_int32), ("forced_bos_token_id", C.c_int32),
                ("stop_at_count", C.c_int32), ("always_allow_eos", C.c_int32), ("disable_fm_index", C.c_int32),
                ("remove_invalid_values", C.c_int32), ("n_force_decoding_from", C.c_int32),
                ("force_decoding_from", C.POINTER(C.c_int64)), ("shift", C.c_int32), ("top_k", C.c_int32)]


class GroupParams(C.Structure):           # sealdec_groups_t
    _fields_ = [("num_beam_groups", C.c_int32), ("diversity_penalty", C.c_float)]


class AttnCase(C.Structure):              # sealdec_attn_case_t
    _fields_ = [("kind", C.c_int32), ("arch", C.c_int32), ("d", C.c_int32), ("heads", C.c_int32),
                ("Q", C.c_int64), ("S", C.c_int64),
                ("B", C.c_int32), ("pos", C.c_int32), ("T", C.c_int32), ("compact", C.c_int32),
                ("qkv", vp), ("q", vp), ("ckv", vp), ("kc", vp), ("vc", vp), ("anc", vp),
                ("src_mask", vp), ("src_off", vp),
                ("G", C.c_int64), ("grp_query", vp), ("grp_start", vp),
                ("rel_bias", vp), ("num_buckets", C.c_int32), ("max_distance", C.c_int32),
                ("split_part", vp), ("split_ks", C.c_int32), ("split_unscale", C.c_float), ("split_bias", vp),
                ("out_split", C.c_int32)]


class NormCase(C.Structure):              # sealdec_norm_case_t
    _fields_ = [("kind", C.c_int32), ("d", C.c_int32), ("rows", C.c_int64),
                ("tok", vp), ("tok_stride", C.c_int64), ("V", C.c_int32), ("embed", vp), ("scale", C.c_float),
                ("pos", vp), ("pos_const", C.c_int32), ("pos_offset", C.c_int32), ("pos_rows", C.c_int32), ("pos_table", vp),
                ("ln_emb_g", vp), ("ln_emb_b", vp),
                ("a", vp), ("b", vp),
                ("split_part", vp), ("split_ks", C.c_int32), ("split_unscale", C.c_float), ("split_bias", vp),
                ("gamma", vp), ("beta", vp), ("eps", C.c_float), ("out_scale", C.c_float),
                ("h", vp),
                ("out_split", C.c_int32)]


_DEC_SIGS = {
    "sealdec_apply_index_mask_d": (i32, [vp, vp, C.POINTER(ProcessorCfg), vp, C.c_int64, C.c_int64, vp, vp, vp,
                                         C.c_int64, C.c_int64]),
    "sealbart_create": (i32, [C.POINTER(BartConfig), C.POINTER(BartVariant), i32, C.POINTER(vp)]),
    "sealbart_free": (None, [vp]),
    "sealt5_create": (i32, [C.POINTER(T5Config), i32, C.POINTER(vp)]),
    "sealt5_relative_buckets": (i32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, vp]),
    "sealbart_set_tensor": (i32, [vp, cp, vp, u64]),
    "sealbart_finalize": (i32, [vp]),
    "sealbart_device_bytes": (u64, [vp]),
    "sealdec_hyps_per_query": (C.c_int64, [C.POINTER(DecParams)]),
    "sealdec_generate": (i32, [vp, vp, vp, C.POINTER(DecParams), vp, vp, C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp,
                               C.POINTER(GroupParams)]),
    "sealdec_generate_dx": (i32, [vp, vp, vp, C.POINTER(DecParams), vp, vp, C.c_int64, C.c_int64, vp, vp, vp, vp, vp,
                                  vp, vp, vp, C.c_int64, C.POINTER(GroupParams)]),
    "sealbart_set_option": (i32, [vp, cp, C.c_int64]),
    "sealbart_get_stat": (C.c_int64, [vp, cp]),
    "sealdec_teacher_forced": (i32, [vp, vp, vp, C.c_int64, C.c_int64, vp, vp, C.c_int64, C.c_int64, C.c_float, vp,
                                     C.c_int64, vp]),
    "sealdec_debug_step_logits": (i32, [vp, vp, vp, C.c_int64, C.c_int64, C.c_int32, vp, C.c_int64, vp, C.c_int64, vp]),
    "sealdec_debug_gemm": (i32, [i32, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32,
                                 C.POINTER(C.c_double)]),
    "sealdec_debug_gemm_ex": (i32, [i32, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32,
                                    C.POINTER(C.c_double), C.c_int32, C.c_int32]),
    "sealdec_debug_gemm_split": (i32, [i32, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp,
                                       vp, vp, C.c_int64, vp, vp, vp, vp]),
    "sealdec_debug_head": (i32, [C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    "sealdec_debug_head_ex": (i32, [i32, C.c_int64, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp]),
    "sealdec_debug_select_step": (i32, [vp, C.POINTER(DecParams), C.POINTER(GroupParams), C.c_int64, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32] + [vp] * 30),
    "sealdec_debug_target_logprob": (i32, [C.c_int64, C.c_int32, C.c_int64, vp, vp, C.c_int64, C.c_float, vp, C.c_int64,
                                           vp, C.c_int64]),
    "sealdec_debug_attention": (i32, [C.POINTER(AttnCase), vp, vp, vp, vp, vp, vp, vp, vp]),
    "sealdec_debug_rownorm": (i32, [C.POINTER(NormCase), vp, vp, vp, vp, vp, vp]),
    "sealdec_debug_topk_threshold": (i32, [C.c_int64, C.c_int32, C.c_int64, vp, C.c_int32, vp, vp, vp]),
    "sealdec_debug_topk_threshold_cluster": (i32, [C.c_int64, C.c_int32, C.c_int64, vp, C.c_int32, vp, vp, vp]),
    "sealdec_debug_topk_rows":(i32, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double)]),
    "sealdec_debug_gemm_trace": (i32, [i32, C.POINTER(C.c_int64)]),
    "sealdec_debug_gemm_units": (i32, [C.POINTER(C.c_int64), C.c_int32]),
    "sealev_first_stage": (i32, [C.c_int64, vp, vp, vp, vp, C.c_int64, vp, vp, vp, i32, i32, C.c_double, C.c_double, C.c_int64, vp, vp]),
    "sealev_score_docs": (i32, [C.c_int64, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, vp, C.c_int64, i32, i32, i32, i32,
                                C.c_double, C.c_double, vp, vp, vp, vp, vp, vp, C.c_int64]),
    "sealev_last_error": (C.c_char_p, []),
    "sealev_set_sum_mode": (None, [i32]),
    # include/sealev_batch.h
    "sealev_key_scores": (i32, [C.c_int64, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, i32, vp]),
    "sealev_unigram_topk": (i32, [C.c_int64, C.c_int64, vp, C.c_int64, vp, vp, vp, vp]),
    "sealev_unigram_scores": (i32, [C.c_int64, vp, vp, vp, C.c_double, C.c_double, C.c_double, i32, vp]),
    "sealev_best_unigrams": (i32, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int64]),
    "sealev_set_device_budget": (None, [u64]),
    "sealev_batch_first_stage": (i32, [vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, i32, i32, C.c_double, C.c_double,
                                       C.c_int64, vp, vp, C.c_int64]),
    "sealev_batch_score_docs": (i32, [vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int64, i32, i32,
                                      i32, i32, C.c_double, C.c_double, vp, vp, C.c_int64, vp, vp, vp, vp, vp, vp,
                                      C.c_int64, vp]),
    "sealev_batch_phase_us": (None, [vp]),
    "sealdec_profile_gemm": (i32, [vp, i32, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "sealdec_last_phase_us": (i32, [vp, C.POINTER(C.c_double)]),
}


def _bind(sigs):
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing: intended
        fn.restype = res
        fn.argtypes = args


_bind(_FM_SIGS)
_bind(_DEC_SIGS)


def check(code):
    if code != 0:
        raise SealB200Error(code, lib.sealfm_last_error().decode(errors="replace"))


def fm_symbols():
    return list(_FM_SIGS)
