/* sealdec.h — C ABI of the H100-native constrained beam-search decode for SEAL.
 *
 * Replaces, behind the reference's own Python surface (seal_b200/beam_search.py mirrors
 * /root/reference/seal/beam_search.py), the per-step work of
 *   - IndexBasedLogitsProcessor.__call__            seal/beam_search.py:62-140
 *   - constrained_beam_search's step                seal/beam_search.py:219-345
 *   - BeamSearchScorerWithMemory.process/finalize   seal/beam_search.py:614-735
 *   - the BART-large forward the reference gets from transformers 4.13 (call sites
 *     seal/beam_search.py:231-238,481-483; model = BartForConditionalGeneration), or the T5 forward
 *     (T5ForConditionalGeneration, SEALSearcher's 't5' backbone) behind the same handle (sealt5_create), or the
 *     pre-LayerNorm BART-family forward of Pegasus and mBART (sealbart_create with a variant)
 * Plain pointers and sizes only.  Status codes and sealfm_last_error() as in sealfm.h.
 * Everything runs on the GPU; there is no CPU path.
 * This header is ABI version 3 (sealfm_abi_version()); the prototypes that changed in it say so.
 */
#ifndef SEALDEC_H
#define SEALDEC_H
#include <stdint.h>
#include "sealfm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- stateless logits-processor hook (HF LogitsProcessor protocol) ------------------------------ */

typedef struct {
    int32_t num_beams;
    int32_t pad_token_id;              /* IndexBasedLogitsProcessor defaults: 0          (:43) */
    int32_t eos_token_id;              /*                                     2          (:44) */
    int32_t stop_at_count;             /* 0 = off                                        (:46) */
    int32_t always_allow_eos;          /*                                                (:47) */
    int32_t forced_bos_token_id;       /* -1 = None                                      (:48) */
    int32_t n_force_decoding_from;     /* length of force_decoding_from, 0 = None        (:45) */
    const int64_t* force_decoding_from;/* host pointer                                         */
    int32_t shift;                     /* seal/index.py:16 SHIFT = 10                           */
} sealdec_processor_cfg_t;

/* scores_out[r][v] = scores_in[r][v] + (allowed(r,v) ? 0 : -inf)  — seal/beam_search.py:62-140.
 * input_ids_d: int64 [R][t] (device), scores: float32 [R][ld] (device; in == out allowed).
 * occurring_mask_d: uint32 [ceil(V/32)] bitmask of index.occurring_distinct (first-step rule :73-77).
 * No host synchronisation. */
int sealdec_apply_index_mask_d(const sealfm_t* fm, sealfm_stream_t stream,
                               const sealdec_processor_cfg_t* cfg,
                               const int64_t* input_ids_d, int64_t R, int64_t t,
                               const uint32_t* occurring_mask_d,
                               const float* scores_in_d, float* scores_out_d, int64_t V, int64_t ld);

/* ---- BART-family weights (bart-large; Pegasus and mBART, the pre-LayerNorm family) ------------------ */

typedef struct sealbart sealbart_t;

typedef struct {
    int32_t vocab_size;        /* 50265 after resize (seal/retrieval.py:570)   */
    int32_t d_model;           /* 1024                                         */
    int32_t encoder_layers;    /* 12                                           */
    int32_t decoder_layers;    /* 12                                           */
    int32_t heads;             /* 16 (head_dim must be 64)                     */
    int32_t ffn_dim;           /* 4096                                         */
    int32_t max_positions;     /* 1024 (+2 learned offset)                     */
    int32_t scale_embedding;   /* 0 for bart-large                             */
    int32_t gemm_mode;         /* 3 = 3xFP16, one CTA per 128x128 tile (split-K for small problems; default), 5 = 3xFP16 in clusters of 2 CTAs sharing the W tile (TMA multicast), 2 = 3xTF32 (fp32 range),
                                  6 = 3xBF16 with bf16 weights (see below).  All wgmma + TMA. */
} sealbart_config_t;

#define SEALBART_ACT_GELU 0            /* exact-erf GELU (bart-large, mBART, PegasusConfig() defaults) */
#define SEALBART_ACT_RELU 1            /* ReLU (released Pegasus checkpoints)                          */

typedef struct {
    int32_t pre_layer_norm;            /* 1: h += SelfAttn(LN_self(h)); h += CrossAttn(LN_cross(h)); h += fc2(act(fc1(LN_final(h))))
                                          and the stacks' final "model.{encoder,decoder}.layer_norm" (Pegasus, mBART);
                                          0: bart-large's post-LayerNorm layer (then only {0, 2, 1, SEALBART_ACT_GELU}) */
    int32_t position_offset;           /* 0: position p reads table row p (Pegasus's sinusoidal table); 2: row p + 2 (mBART, BART) */
    int32_t layernorm_embedding;       /* 1: "model.{encoder,decoder}.layernorm_embedding" after the embedding (mBART); 0: none */
    int32_t activation;                /* SEALBART_ACT_GELU or SEALBART_ACT_RELU, the fc1 epilogue                           */
} sealbart_variant_t;

/* Creates a BART-family model; every entry point below takes the handle.  variant NULL is bart-large's post-LayerNorm
 * layer, as is {0, 2, 1, SEALBART_ACT_GELU}, the only variant with pre_layer_norm = 0.  cfg: d_model a multiple of 128
 * up to 1024, 64-wide heads, ffn_dim % 64 == 0; for a pre-LayerNorm variant max_positions >= 1 is the number of
 * positions the tables cover: each of "model.{encoder,decoder}.embed_positions.weight" has max_positions +
 * position_offset rows (Pegasus's max_position_embeddings rows; mBART's max_position_embeddings + 2).  A pre-LayerNorm
 * model's sealbart_set_tensor takes BART's keys plus "model.{encoder,decoder}.layer_norm.{weight,bias}";
 * "model.{encoder,decoder}.layernorm_embedding.*" only with layernorm_embedding = 1.  Every other key is SEALFM_EINVAL.
 * An unsupported variant or shape is SEALFM_EINVAL before any allocation.
 * Position table (BART's learned table of max_positions + 2 rows too): sources longer than max_positions are refused,
 * and sealdec_teacher_forced / sealdec_debug_step_logits refuse decoder inputs longer than max_positions.  A generate
 * may reach decoder positions past the table (max_length - 2 >= max_positions); those steps read the table's last
 * row, so the records of a beam that is still alive there are not the model's -- whether such a call may run is the
 * caller's decision (seal_b200.beam_search raises the reference's IndexError exactly where the reference's forward
 * would read past the table).
 * ABI version 3 added the variant argument. */
int  sealbart_create(const sealbart_config_t* cfg, const sealbart_variant_t* variant, int device, sealbart_t** out);
void sealbart_free(sealbart_t* m);
/* Copies one tensor of an HF BartForConditionalGeneration state_dict (float32, host pointer,
 * row-major, `numel` elements) by its state_dict key, e.g.
 * "model.decoder.layers.3.encoder_attn.q_proj.weight".  Unknown keys return SEALFM_EINVAL.
 * gemm_mode 6 (bf16 weights, for bf16 checkpoints; any handle kind): every GEMM weight matrix, the token-embedding
 * table and an untied lm_head are stored once, in bf16, rounded to nearest-even here -- exact for values that are
 * bf16 already.  Biases, LayerNorm / RMSNorm weights, position tables, T5 relative-attention tables and
 * final_logits_bias stay fp32.  The GEMMs multiply the bf16 W by the activation split into three bf16 pieces
 * (exact for 2^-100 <= |x| < (2 - 2^-8) 2^127), so each product is exact and only the fp32 accumulation rounds; bf16 has fp32's
 * exponent range, so error_flag [1] is never raised, sealdec_generate never re-runs ("overflow_fallbacks" stays 0) and
 * the GEMM sets last_paths bit 24, never 12 or 14.  The mode is fixed at creation: sealbart_set_option "gemm_mode"
 * refuses to switch into or out of 6 (SEALFM_EINVAL).
 * sealbart_device_bytes: the bytes of the weights on the device -- in gemm_mode 6, 2 per matrix element plus 4 per
 * element of every fp32 vector and table; in the other modes 4 per element of everything plus the modes' split
 * copies (2 x 2 bytes per matrix element for 3 / 5, and 2 x 4 more once 3xTF32 has run). */
int  sealbart_set_tensor(sealbart_t* m, const char* key, const float* host, uint64_t numel);
/* After all tensors are set: checks completeness, ties lm_head to model.shared if it was not
 * given, derives fused/pre-split copies. */
int  sealbart_finalize(sealbart_t* m);
uint64_t sealbart_device_bytes(const sealbart_t* m);

/* ---- T5 weights ------------------------------------------------------------------------------- */

typedef struct {
    int32_t vocab_size;                      /* 32128 for the released t5 checkpoints                          */
    int32_t d_model;                         /* a multiple of 128 up to 1024 (t5-small 512, t5-base 768, t5-large 1024),
                                                or 2048, 3072 or 4096 (the XL / XXL members of T5 v1.1, Flan-T5, mT5) */
    int32_t num_layers;                      /* encoder blocks                                                 */
    int32_t num_decoder_layers;              /* decoder blocks (may differ from num_layers)                    */
    int32_t num_heads;                       /* num_heads * 64 == d_model                                      */
    int32_t d_kv;                            /* must be 64 (t5-3b / t5-11b use 128: not covered)               */
    int32_t d_ff;                            /* multiple of 64                                                 */
    int32_t ffn_kind;                        /* 0 = relu (DenseReluDense.wi / wo); 1 = gated-gelu (wi_0, wi_1, wo; gelu_new, the tanh form) */
    int32_t relative_attention_num_buckets;  /* 32; in [4, 1024]                                               */
    int32_t relative_attention_max_distance; /* 128; > num_buckets / 2                                         */
    float   layer_norm_epsilon;              /* 1e-6                                                           */
    int32_t scale_decoder_outputs;           /* 1: the last decoder state is multiplied by d_model^-0.5 before the lm_head */
    int32_t gemm_mode;                       /* as sealbart_config_t                                           */
} sealt5_config_t;

/* Creates a T5 model behind the same opaque handle: sealbart_set_tensor / sealbart_finalize / sealbart_free and every
 * entry point below take it and behave as documented for BART.  A shape the kernels do not cover is rejected with
 * SEALFM_EINVAL before any allocation (d_kv != 64, num_heads * 64 != d_model, d_model neither a multiple of 128 up to
 * 1024 nor a multiple of 1024 up to 4096, d_ff % 64 != 0, an unknown ffn_kind, a bucket count / max distance outside the ranges above).
 * sealbart_set_tensor takes HF T5ForConditionalGeneration state_dict keys: "shared.weight" (aliases
 * "encoder.embed_tokens.weight", "decoder.embed_tokens.weight"), "encoder.block.{i}.layer.0.SelfAttention.{q,k,v,o}.weight",
 * "encoder.block.{i}.layer.{0,1}.layer_norm.weight", "encoder.block.{i}.layer.1.DenseReluDense.{wi | wi_0, wi_1, wo}.weight",
 * "decoder.block.{i}.layer.0.SelfAttention.*", "decoder.block.{i}.layer.1.EncDecAttention.{q,k,v,o}.weight",
 * "decoder.block.{i}.layer.{0,1,2}.layer_norm.weight", "decoder.block.{i}.layer.2.DenseReluDense.*",
 * "{encoder,decoder}.block.0.layer.0.SelfAttention.relative_attention_bias.weight" (the only bias tables: every layer
 * reuses layer 0's, as in HF), "{encoder,decoder}.final_layer_norm.weight" and "lm_head.weight" (tied to shared.weight if
 * not given).  Every other key -- the keys of the other ffn_kind included -- is SEALFM_EINVAL.
 * Sources are limited to 1024 positions (T5 has no position table; the encoder's bucket table covers distances
 * -1023 .. 1023): a longer source is rejected where BART's max_positions is enforced.  Relative position buckets are
 * computed on the host once per model, in the float32 arithmetic of transformers' _relative_position_bucket. */
int  sealt5_create(const sealt5_config_t* cfg, int device, sealbart_t** out);
/* The host bucket table (no device needed): bidirectional (encoder) out[2n-1], out[i] = bucket of key - query = i - (n-1);
 * unidirectional (decoder) out[n], out[i] = bucket of key - query = -i.  SEALFM_EINVAL for n < 1 or bucket settings
 * sealt5_create rejects. */
int  sealt5_relative_buckets(int32_t num_buckets, int32_t max_distance, int32_t bidirectional, int32_t n, int32_t* out);

/* ---- fused generate --------------------------------------------------------------------------- */

typedef struct {
    int32_t num_beams;
    int32_t min_length;
    int32_t max_length;
    float   length_penalty;
    int32_t eos_token_id;            /* scorer / processor eos (fm_index_generate kwarg, :403)        */
    int32_t pad_token_id;            /* model.config.pad_token_id (1)                                */
    int32_t decoder_start_token_id;  /* model.config.decoder_start_token_id (2)                      */
    int32_t model_eos_token_id;      /* model.config.eos_token_id: MinLength processor (SURVEY §H3)  */
    int32_t forced_eos_token_id;     /* model.config.forced_eos_token_id, -1 = None (§H3)            */
    int32_t forced_bos_token_id;     /* -1 = None                                                    */
    int32_t stop_at_count;
    int32_t always_allow_eos;
    int32_t disable_fm_index;
    int32_t remove_invalid_values;   /* InfNanRemoveLogitsProcessor (:445)                           */
    int32_t n_force_decoding_from;
    const int64_t* force_decoding_from;   /* host pointer */
    int32_t shift;                   /* 10 */
    int32_t top_k;                   /* 0 = off; > 0: TopKLogitsWarper(top_k) on every step's raw logits, see below */
} sealdec_params_t;
/* top_k (constrained_beam_search's topk, seal/beam_search.py:163-164,249-253): before the log-softmax, every logit below
 * tau, the min(top_k, V)-th largest of its fp32 row, becomes -inf (ties at tau are kept, -0.0 == +0.0, -inf entries count
 * as values).  The row max is unchanged; the log-softmax denominator sums exp(x - max) over x >= tau only, and a -inf
 * fill-in pick (a masked candidate, SURVEY.md H4) records -inf when its logit is below tau.  The forcing steps (forced
 * BOS, forced EOS) overwrite every score and are unaffected.  top_k >= V is no warp at all and takes the top_k = 0 path
 * (bit-identical records).  A top_k > 0 step stores the lm_head's logits densely (no statistics epilogue) and runs one
 * more kernel per step whose logits are read: one CTA per logits row for vocab_size <= 53 248 (bart-large's 50 265),
 * one cluster of ceil(vocab_size / 53 248) CTAs per row above (mT5's 250 112: 5).  SEALFM_EINVAL for top_k < 0, for
 * top_k > 0 with num_beam_groups > 1 (group_beam_search has no warper) and for top_k > 0 with vocab_size > 425 984
 * (the row is staged in the shared memory of at most 8 CTAs).  The member sits in the struct's former tail padding: a
 * caller that zero-initialises the struct keeps the previous behaviour. */

/* Number of hypothesis records per query that sealdec_generate writes:
 * (max_length-1) * 2*num_beams + num_beams   (process :662-668 every step + finalize :717-725). */
int64_t sealdec_hyps_per_query(const sealdec_params_t* p);

/* ---- diverse beam groups (fm_index_generate's diverse_bs_groups / diverse_bs_penalty, seal/beam_search.py:447-532) ----
 * With num_beam_groups = G > 1 the decode follows transformers 4.13's group_beam_search: the beams of a query form G
 * groups of num_beams / G, chosen one group after the other at every step; the index mask is an ordinary logits
 * processor there, so recorded scores are the constrained ones (tie-filled picks record -inf), and a positive
 * diversity_penalty subtracts penalty * count(v) from group g's log-probability of token v, count(v) = how often the
 * groups before g chose v at this step (HammingDiversityLogitsProcessor).  The record count and layout are those of
 * one group: sealdec_hyps_per_query per query, each step's 2*num_beams records group by group, in rank order.
 * The generate calls take this struct; NULL and {1, 0} are both the single-group decode, with bit-identical records.
 * 1 <= num_beam_groups <= num_beams with num_beams % num_beam_groups == 0, else SEALFM_EINVAL. */
typedef struct {
    int32_t num_beam_groups;         /* G, 1 = one group                                             */
    float   diversity_penalty;       /* <= 0: no Hamming penalty (only used with G > 1); finite      */
} sealdec_groups_t;

/* fm_index_generate(model, index, input_ids, attention_mask, ..., keep_history=True)
 * seal/beam_search.py:391-557, with the beam groups of `groups` (NULL = one group).  HOST buffers in and out (copies
 * are part of the call):
 *   input_ids, attention_mask  int64 [Q][S]
 *   out_scores   float32 [Q][H]      sum_logprobs of each recorded hypothesis (:667); caller applies
 *                                    score/len**lp * len**lp (:754,:555) — identity for lp = 0
 *   out_len      int32   [Q][H]      tokens in the hypothesis (incl. decoder_start)
 *   out_tokens   int32   [Q][H][max_length]
 *   out_valid    uint8   [Q][H]      1 iff the pick's CONSTRAINED score was finite (SURVEY §H4);
 *                                    finalize records carry 2
 *   out_lo/out_hi uint64 [Q][H]      SA range [lo,hi) of the hypothesis' tokens[1:] (0,0 if invalid
 *                                    or FM index disabled); may be NULL
 * Every source must attend to at least one position, and every token id must lie in [0, vocab_size): an
 * attention_mask row that is all zero or an id outside that range is rejected with SEALFM_EINVAL (here, by
 * sealdec_teacher_forced and by the debug entry points); sealdec_generate_dx does not check either, and its results
 * for such a source are undefined.
 * H = sealdec_hyps_per_query(p).  Returns SEALFM_EINVAL("beam") if some query had fewer than
 * num_beams non-EOS candidates (the reference raises ValueError, :687-690).  If an activation leaves the fp16
 * range of the default GEMM mode the pass is repeated with the 3xTF32 kernels (sealbart_get_stat "overflow_fallbacks").
 * ABI version 3 added `groups`. */
int sealdec_generate(sealbart_t* model, const sealfm_t* fm, const uint32_t* occurring_mask_host,
                     const sealdec_params_t* p, const int64_t* input_ids, const int64_t* attention_mask,
                     int64_t Q, int64_t S, float* out_scores, int32_t* out_len, int32_t* out_tokens,
                     uint8_t* out_valid, uint64_t* out_lo, uint64_t* out_hi, const sealdec_groups_t* groups);

/* fm_index_generate as sealdec_generate computes it, on inputs and outputs already resident on the model's device:
 * the arguments and outputs of sealdec_generate, as device pointers (*_d), and these:
 *   stream          the call is asynchronous on it, except for workspace (re)allocation and -- with
 *                   src_tokens_hint = -1 -- one 16-byte read-back of the real source-token count.
 *   src_tokens_hint what the caller knows about the sources:
 *                   >= 1  the number of non-zero attention_mask entries, masks right-padded (the only kind SEAL
 *                         builds): the encoder runs on the real tokens only and the call never touches the host;
 *                         a wrong count raises error_flag_d[2];
 *                   -1    unknown: one 16-byte device->host read to learn it;
 *                   -2    compute the padded positions too (no host access either).
 *   error_flag_d    int32[4] on the device, zeroed by the call and raised by its kernels:
 *                   [0] some query had fewer than num_beams non-EOS candidates (the reference raises ValueError,
 *                       :687-690)
 *                   [1] an activation left the fp16 range of the 3xFP16 GEMM modes (|x| > 65504; operands were
 *                       saturated): the results are NOT to be used -- re-run after sealbart_set_option(model,
 *                       "gemm_mode", 2) (3xTF32, fp32 range).  sealdec_generate (host buffers) does that by itself.
 *                   [2] src_tokens_hint did not match the attention mask
 *                   [3] reserved
 * On a non-default stream, batches of at most 4096 rows (queries x beams) are replayed from a CUDA graph of the
 * whole call from the third call with the same shapes, parameters and buffer addresses on (a generate of 20
 * queries is ~1 900 short kernels: launch-bound); sealbart_set_option(model, "cuda_graph", 0 / 1 / -1) forces it
 * off / on / back to automatic.  ABI version 3 added `groups`. */
int sealdec_generate_dx(sealbart_t* model, const sealfm_t* fm, const uint32_t* occurring_mask_d,
                        const sealdec_params_t* p, const int64_t* input_ids_d,
                        const int64_t* attention_mask_d, int64_t Q, int64_t S, sealfm_stream_t stream,
                        float* out_scores_d, int32_t* out_len_d, int32_t* out_tokens_d,
                        uint8_t* out_valid_d, uint64_t* out_lo_d, uint64_t* out_hi_d,
                        int32_t* error_flag_d, int64_t src_tokens_hint, const sealdec_groups_t* groups);

/* Options: "cuda_graph" (-1 auto, 0 off, 1 on), "gemm_mode" (switch between the 3xFP16 modes 3/5 and 2 = 3xTF32;
 * the TF32 operand copies are made on first use; never into or out of 6), "fused_head" (-1 = $SEALB200_FUSED_HEAD, default on; 0 = the
 * lm_head stores every logit and the select kernel streams them for the log-softmax statistics; 1 = where the select
 * kernels read only the row's allowed tokens, the lm_head emits per-tile statistics and stores only those logits),
 * "poison_logits" (testing: 1 fills the logits buffer with NaN before every such lm_head), "query_slices" (-1 =
 * $SEALB200_QUERY_SLICES, default on; 1 = after the first decode step a generate whose two halves of the batch have
 * more than 2 048 rows (queries x beams) each runs the two halves on two streams -- the caller's and one the model
 * owns, forked and joined with events on the caller's stream, so a CUDA graph captures both -- with bit-identical
 * records; never while GEMM profiling is on).  Stats: "last_used_graph",
 * "overflow_fallbacks", "gemm_mode", "cached_graphs", "fused_head_steps" (decode steps of the last generate run
 * eagerly that used the statistics epilogue), "topk_cluster_steps" (decode steps of the last generate whose top-k
 * threshold ran one cluster per logits row, vocab_size > 53 248; a CUDA-graph replay reports the captured call's
 * count), "launches" (kernel launches issued by the last generate / teacher-forced / debug-step call, own kernels
 * only; a CUDA-graph replay reports the captured call's count; a stat since ABI version 3), "last_paths" (-1 for an
 * unknown name).
 * "last_paths" is the OR, over the last generate / teacher-forced / debug-step call (a CUDA-graph replay reports
 * the call it was captured from), of one bit per kernel branch of the BART forward:
 *   0 encoder on the real tokens only (packed)         1 encoder on the padded rows (mask per key)
 *   2 decoder self-attention, beams of a query together (dec_self_attn_query_kernel)
 *   3 ... one row per CTA, <= 12 keys                  4 ... <= 32 keys                5 ... > 32 keys
 *   6 cross-attention, source <= 32 positions          7 cross-attention, longer sources
 *   8 add + LayerNorm, one CTA per row (<= 2048 rows)  9 add + LayerNorm, one warp per row
 *  10 split-K GEMM summed by its consumer kernel      11 split-K GEMM + finish pass
 *  12 3xFP16 GEMM on whole tiles                      13 3xFP16 GEMM on 2-CTA clusters (gemm_mode 5)
 *  14 3xTF32 GEMM (gemm_mode 2)                      15 generate run as two query slices ("query_slices")
 * and of the T5 forward (a T5 call also sets 6, 7, 10 .. 15 as above; 0 / 1 name its encoder packing):
 *  16 T5 encoder self-attention with the relative position bias
 *  17 T5 decoder self-attention with the relative position bias (one warp per row and head, any position)
 *  18 embedding / add + RMSNorm (one CTA per row; folds a pending split-K GEMM), d_model <= 1024
 *  19 ReLU feed-forward (ReLU GEMM epilogue)          20 gated-gelu feed-forward (gelu_new(wi_0 x) * wi_1 x kernel)
 *  21 embedding / add + RMSNorm as 18, d_model 2048 .. 4096 ("t5_rms_wide"; such a model never sets 18)
 * and of the pre-LayerNorm forward (a sealbart_create variant; it also sets 0 .. 7 and 10 .. 15 as BART does, never 8 / 9;
 * bit 19 names its ReLU feed-forward, e.g. Pegasus's):
 *  22 embedding / add + LayerNorm, one CTA per row (preln_row_kernel; folds a pending split-K GEMM)
 *  23 the embedding form of 22 with layernorm_embedding (mBART: two LayerNorms in one launch)
 * and, for any handle kind:
 *  24 3xBF16 GEMM (gemm_mode 6; such a call never sets 12, 13 or 14) */
int     sealbart_set_option(sealbart_t* model, const char* name, int64_t value);
int64_t sealbart_get_stat(const sealbart_t* model, const char* name);

/* ---- teacher-forced scoring: SURVEY.md section 8(f) rank 1 ------------------------------------------
 * The decoder pass behind rescore_keys (seal/keys.py:64-141) and compute_unigram_scores (:145-176).
 * dec_ids: int64 [N][T] decoder inputs (row r = decoder_start + key tokens, right-padded), row r is
 * scored against encoder input row_query[r] (sorted ascending).  HOST pointers.
 *   out_logprob [N][T-1]: log_softmax(logits_p / temperature)[dec_ids[r][p+1]] for p = 0..T-2
 *                         (full-vocabulary normalisation; the caller masks padding and sums, :131-135)
 *   out_full    [N][V]  : if non-NULL, the whole log-prob vector of position out_full_pos (:167-172)
 * Rows are decoded in passes of 4096; T <= 128.  Returns SEALFM_EINVAL, before anything runs, for an all-zero
 * attention_mask row, a token id of input_ids or dec_ids outside [0, vocab_size) (the reference raises IndexError),
 * row_query unsorted or outside [0, Q), and out_full with out_full_pos outside [0, T).  It also returns SEALFM_EINVAL
 * ("fp16 range exceeded") when an activation of the encoder or the decoder left the fp16 range of the 3xFP16 GEMM
 * modes: unlike sealdec_generate there is no automatic re-run, the outputs are not to be used, and the caller may
 * switch to gemm_mode 2 (3xTF32) and call again. */
int sealdec_teacher_forced(sealbart_t* model, const int64_t* input_ids, const int64_t* attention_mask,
                           int64_t Q, int64_t S, const int64_t* dec_ids, const int32_t* row_query,
                           int64_t N, int64_t T, float temperature, float* out_logprob,
                           int64_t out_full_pos, float* out_full);

/* Test / profiling hooks: one decoder step's logits for explicit decoder inputs (teacher forcing).  Host pointers:
 *   decoder_input_ids int64 [R][t], R = Q*num_beams rows laid out query-major like the reference's expanded batch
 *            (:517-521);
 *   ancestry int32 [R][t], or NULL for every row its own ancestor: row r reads the decoder cache of position s
 *            from row ancestry[r][s] (in [0, R)), as a generate does after beams were reordered; entries at
 *            position t-1 are not read.  The caller keeps it consistent (equal decoder_input_ids[:s+1]).
 *   src_tokens_hint as in sealdec_generate_dx: -1 pack right-padded masks, -2 never pack, >= 1 the count of
 *            non-zero mask entries of right-padded masks (checked here);
 *   out_logits float32 [R][V], the logits of the last position.
 * ABI version 3 added ancestry and src_tokens_hint. */
int sealdec_debug_step_logits(sealbart_t* model, const int64_t* input_ids, const int64_t* attention_mask,
                              int64_t Q, int64_t S, int32_t num_beams, const int64_t* decoder_input_ids,
                              int64_t t, const int32_t* ancestry, int64_t src_tokens_hint, float* out_logits);
/* Stand-alone GEMM C[M,N] = A[M,K] W[N,K]^T + bias (+ the epilogue activation) through the model's GEMM kernels
 * (mode 2 = 3xTF32, 3 = 3xFP16, 5 = 3xFP16 on CTA pairs, 6 = 3xBF16 with W rounded to bf16 as sealbart_set_tensor
 * rounds it), host pointers; gelu: 0 = no activation, 1 = exact-erf GELU, 2 = ReLU.  If iters > 0 also reports the
 * average device time per call (CUDA events, includes the activation split). */
int sealdec_debug_gemm(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W,
                       const float* bias, float* C, int32_t gelu, int32_t iters, double* avg_us);
/* the same with the tile order (mode 3 without split-K; other paths ignore band) and the store as variables
 * (tools/head_bench.py): band -1 = the order the decoder
 * uses, 0 = no bands (m fastest over all rows when N > M), > 0 = bands of that many 128-row tiles; store 0 = the
 * epilogue writes nothing (C may be NULL, and is not written).  Modes 3 / 5 split A into halves (mode 6 into three
 * bf16 pieces) once, outside the timed calls, as the decoder's producers do. */
int sealdec_debug_gemm_ex(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W,
                          const float* bias, float* C, int32_t gelu, int32_t iters, double* avg_us, int32_t band,
                          int32_t store);
/* The GEMM's other outputs, as the forward uses them (tests/test_gemm_split_out_gpu.py): one sealdec_debug_gemm_ex call
 * (A split once beforehand; bias may be NULL) with
 *   act       0 = no activation, 1 = exact-erf GELU, 2 = ReLU;
 *   outputs   bit 0: the fp32 C [M][N]; bit 1: the operand split of the next GEMM, row stride N, in the mode's format:
 *             mode 2 float s1 / s2 (TF32 hi / lo), modes 3 / 5 fp16 s1 / s2 (h1 / h2, saturated at +-65504), mode 6
 *             bf16 s1 / s2 / s3 (the three pieces).  1, 2 or 3; s3 is only read in mode 6.  Whatever the GEMM does
 *             not write comes back as NaN;
 *   *overflow the GEMM's own fp16 range flag (1 if its epilogue or finish pass saturated a value; the flag the input
 *             split may raise is cleared before the GEMM runs);
 *   defer_rows as the forward passes it: a split-K result of at most this many rows, without activation or split
 *             output, with a bias and N a multiple of 4, is left unsummed for its consumer.  If the call deferred,
 *             *k_slices > 1, slices [k_slices][M][N] receives the raw slices (room for 8 is needed) and *unscale the
 *             factor the consumer applies before the bias (finished = (sum of the slices in index order) * unscale +
 *             bias); otherwise *k_slices = 0.  slices and unscale may be NULL when defer_rows is 0;
 *   *paths    the "last_paths" bits of the call (10 .. 14, 24; 19 for ReLU). */
int sealdec_debug_gemm_split(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W,
                             const float* bias, int32_t act, int32_t outputs, float* C, void* s1, void* s2, void* s3,
                             int32_t* overflow, int64_t defer_rows, float* slices, int32_t* k_slices, float* unscale,
                             uint32_t* paths);
/* The lm_head GEMM of a decode step with the statistics epilogue requested (gemm_mode 3, through the same GEMM
 * dispatch as the decoder; tests/test_select_step_gpu.py): C[M,N] = A W^T + bias with the row masks
 * mask uint32 [M][ceil(N/32)] and eos / pad defining each row's read set.  Host pointers.  With Mpad = M rounded up
 * to 128 rows, C is float32 [Mpad][N] and stats float32 [Mpad][ceil(N/128)][2] = per (row, 128-column tile)
 * (max, sum exp(x - max)); both are filled with NaN on the device before the call, so whatever the GEMM does not
 * write comes back as NaN.  *fused = 1 if the statistics epilogue ran (then C holds only the read set: the whole
 * first tile, the mask bits, eos and pad); 0 if the shape took the split-K path, which stores C densely and no
 * statistics, as the decoder then does. */
int sealdec_debug_head(int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias,
                       const uint32_t* mask, int32_t eos, int32_t pad, float* C, float* stats, int32_t* fused);
/* sealdec_debug_head in gemm_mode 3 or 6 (W rounded to bf16); any other mode is SEALFM_EINVAL. */
int sealdec_debug_head_ex(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias,
                          const uint32_t* mask, int32_t eos, int32_t pad, float* C, float* stats, int32_t* fused);
/* One decode step's selection (log-softmax statistics or the top-k warp of p->top_k, processors, index mask, top-2*beam, the scorer bookkeeping,
 * the records and the LF step) on caller-supplied inputs, through the same kernel dispatch as the generate entry
 * points.  Host pointers; B = p->num_beams, T = p->max_length, R = Q*B, W = ceil(V/32), G from `groups` (NULL = 1).
 * Configurations a generate never produces are rejected with SEALFM_EINVAL (B > 32, cur_len outside
 * [1, max_length-1], logits_shared away from cur_len 1, logits_ignored away from the forced-EOS step, head statistics
 * on a step where the lm_head would not write them or with p->top_k > 0, ...).
 * Inputs:  logits float32 [logits_shared ? Q : R][V] (NULL with logits_ignored; padded to the generate's stride with
 *          NaN), head_stats float32 [R][ceil(V/128)][2] from the lm_head epilogue or NULL (statistics streamed from
 *          the logits), masks uint32 [R][W] (may be NULL where not read), occurring_mask uint32 [W] (the first
 *          step's mask), beam_scores float32 [R], tokens and ancestry int32 [R][T], lo, hi, pw uint64 [R]; fm is
 *          needed unless p->disable_fm_index.
 * Outputs: row_max, row_logsum float32 [R], row_rule uint8 [R]; the candidate lists cand_val float32 / cand_idx
 *          int32 [R][2B] and cand_cnt int32 [R], of which the first Q * (*lists) are the step's lists; the next beams
 *          beam_scores_out [R], tokens_out / ancestry_out [R][T], lo_out, hi_out, pw_out [R]; the step's records
 *          rec_score, rec_len, rec_tokens [Q][2B][T], rec_valid, rec_lo, rec_hi, [Q][2B] each; error_flag int32 [1]
 *          (fewer than num_beams non-EOS candidates).  Every output and scratch buffer is filled with NaN / all-ones
 *          bits on the device first, so an element the step does not write comes back that way. */
int sealdec_debug_select_step(const sealfm_t* fm, const sealdec_params_t* p, const sealdec_groups_t* groups, int64_t Q,
                              int32_t V, int32_t cur_len, int32_t logits_shared, int32_t logits_ignored,
                              const float* logits, const float* head_stats, const uint32_t* masks,
                              const uint32_t* occurring_mask, const float* beam_scores, const int32_t* tokens,
                              const int32_t* ancestry, const uint64_t* lo, const uint64_t* hi, const uint64_t* pw,
                              float* row_max, float* row_logsum, uint8_t* row_rule, float* cand_val, int32_t* cand_idx,
                              int32_t* cand_cnt, int32_t* lists, float* beam_scores_out, int32_t* tokens_out,
                              int32_t* ancestry_out, uint64_t* lo_out, uint64_t* hi_out, uint64_t* pw_out,
                              float* rec_score, int32_t* rec_len, int32_t* rec_tokens, uint8_t* rec_valid,
                              uint64_t* rec_lo, uint64_t* rec_hi, int32_t* error_flag);
/* The teacher-forced log-prob kernel of sealdec_teacher_forced on caller-supplied logits, through the same launch.
 * Host pointers: logits float32 [R][ld] (ld >= V; columns V .. ld-1 are not read), targets int64 read at
 * r * tgt_stride, out float32 [(R-1)*out_stride + 1] with out[r * out_stride] = log_softmax(logits[r][:V] /
 * temperature)[target] (fp32 division, as the reference; exactly 0 for a target outside [0, V)), full float32
 * [(R-1)*full_ld + V] with the whole log-prob row at full[r * full_ld].  out or full may be NULL, not both.  Both are
 * filled with NaN on the device first, so an element the kernel does not write comes back as NaN.  Arguments the
 * teacher-forced path never passes (ld < V, temperature <= 0 or not finite, strides < 1, full_ld < V) give
 * SEALFM_EINVAL. */
int sealdec_debug_target_logprob(int64_t R, int32_t V, int64_t ld, const float* logits, const int64_t* targets,
                                 int64_t tgt_stride, float temperature, float* out, int64_t out_stride, float* full,
                                 int64_t full_ld);
/* One attention block of the model on caller-supplied activations (sealdec_debug_attention), through the same kernel
 * choice as the layer loops.  Host pointers throughout; heads = d / 64.
 *   kind 0 encoder self-attention: Q sources of S positions; qkv [N][3d] with N = Q*S (src_mask int32 [Q][S], 0 = pad)
 *          or, packed (src_off int32 [Q+1], prefix sums of lengths in [1, S]), N = src_off[Q] rows of real tokens.
 *   kind 1 decoder self-attention at position pos (keys 0 .. pos) of B beams per query: qkv [R][3d] of this step's rows,
 *          R = Q*B, or R = Q with compact (the first step, pos 0: row r stands for cache rows r*B .. r*B + B-1); the
 *          layer's cache kc, vc float32 [T][Q*B][d], key s < pos of row r read from cache row anc[r][s] (int32
 *          [Q*B][T], entries in [0, Q*B)).  The rows at position pos are filled with NaN on the device first.
 *   kind 2 cross-attention: q [rows][d] over ckv [N][2d] (k | v of the encoder states, N as for kind 0, src_mask or
 *          src_off as there); groups of B rows per query (rows = Q*B; compact: 1 row per query), or ragged groups
 *          (G > 0): group g = rows grp_start[g] .. grp_start[g+1]-1 (grp_start[0] = 0, non-decreasing) of query
 *          grp_query[g] (in [0, Q)), rows = grp_start[G].
 *   arch 0 BART (scores q.k / 8), 1 T5 (kinds 0 and 1 add rel_bias [num_buckets][heads] at the bucket of key - query,
 *          bidirectional for kind 0; scores unscaled; kind 2 runs the BART kernel, as the model does).
 *   split_ks > 1: qkv (kind 1) or q (kind 2) as split-K GEMM slices split_part [split_ks][rows][cols], element =
 *          (sum of slices in order) * split_unscale + split_bias[col]; only for the two kernels that sum them (the
 *          decoder's per-query kernel and the short-source cross kernel); the plain qkv / q is then not read.
 *   out_split 0 none, 1 TF32 pieces (float32 hi, lo), 2 fp16 halves (h1, h2; overflow raised past 65504), 3 bf16 x3.
 * Outputs (each filled with NaN on the device first): out float32 [rows][d] (the T5 kernels write only the split; out
 * then stays NaN, and out_split 0 is refused), split1..3 [rows][d] of the split's element type, *overflow,
 * kc_out / vc_out [T][Q*B][d] (kind 1), *path = the sealbart_get_stat "last_paths" bit of the kernel that ran (0 for
 * the BART encoder kernel).  Arguments the model never passes are SEALFM_EINVAL before any device work: a head width
 * other than 64, d above 1024 (BART) / 4096 (T5), S outside [1, 1024], T outside [pos+1, 128], an ancestry entry out of
 * range, a query without a valid key, split-K slices for a kernel that does not sum them. */
typedef struct {
    int32_t kind, arch, d, heads;
    int64_t Q, S;
    int32_t B, pos, T, compact;
    const float* qkv; const float* q; const float* ckv;
    const float* kc; const float* vc; const int32_t* anc;
    const int32_t* src_mask; const int32_t* src_off;
    int64_t G; const int32_t* grp_query; const int32_t* grp_start;
    const float* rel_bias; int32_t num_buckets, max_distance;
    const float* split_part; int32_t split_ks; float split_unscale; const float* split_bias;
    int32_t out_split;
} sealdec_attn_case_t;
int sealdec_debug_attention(const sealdec_attn_case_t* c, float* out, void* split1, void* split2, void* split3,
                            int32_t* overflow, float* kc_out, float* vc_out, uint32_t* path);
/* One row-norm or gate producer of the model on caller-supplied rows (sealdec_debug_rownorm), through the same
 * launchers as the layer loops: the kernels that write every GEMM operand that is not an attention output.  Host
 * pointers throughout; `rows` rows of width d.
 *   kind 0 BART embedding + layernorm_embedding: out[r] = LN(embed[tok[r * tok_stride]] * scale
 *          + pos_table[min(p + 2, pos_rows - 1)]; gamma, beta), p = pos[r] or pos_const (pos NULL).
 *   kind 1 BART add + LayerNorm: out[r] = LN(a[r] + b[r]; gamma, beta), run in place as the layers run it (out == a);
 *          a CTA per row up to 2 048 rows, a warp per row above.
 *   kind 2 T5 RMSNorm: the residual x_out[r] = embed[tok[r * tok_stride]] (tok given) or a[r] + b[r] (a given), and
 *          the split of (gamma * (x_out * rsqrt(mean(x_out^2) + eps))) * out_scale.
 *   kind 3 pre-LayerNorm row: the residual x_out[r] = embed[tok] * scale + pos_table[min(p + pos_offset, pos_rows - 1)],
 *          then LN(.; ln_emb_g, ln_emb_b) if ln_emb_g is given (tok given), or a[r] + b[r] (a given); and the split of
 *          LN(x_out; gamma, beta).
 *   kind 4 T5 gated-gelu: h [rows][2d] (d = d_ff) -> the split of gelu_new(h[:, :d]) * h[:, d:].
 * embed float32 [V][d] (rounded to bf16 as sealbart_set_tensor rounds it for out_split 3), pos_table float32
 * [pos_rows][d], gamma / beta / ln_emb_g / ln_emb_b float32 [d].  b may be given as split-K slices instead (split_ks in
 * 2 .. 8): split_part [split_ks][rows][d], element = (sum of slices in index order) * split_unscale + split_bias[col];
 * only where the kernel sums them (kind 1 up to 2 048 rows, the add forms of kinds 2 and 3).
 * out_split 0 none (kinds 0, 1 only), 1 TF32 pieces (float32 hi, lo), 2 fp16 halves (h1, h2; overflow raised past
 * 65504), 3 bf16 x3 (the splits of gemm_mode 2 / 3 / 6).
 * Outputs, each filled with NaN on the device first: out float32 [rows][d] (the LayerNorm of kinds 0 and 1, the
 * residual x_out of kinds 2 and 3; not written for kind 4, may be NULL there), split1..3 [rows][d] of the split's
 * element type, *overflow, *path = the sealbart_get_stat "last_paths" bit(s) of the kernel that ran (0 for kind 0).
 * The position table is followed on the device by NaN rows up to row 1 026, so a read past its last row shows as NaN.
 * Arguments the model never passes are SEALFM_EINVAL before any device work: d outside the family's widths (kinds 0,
 * 1, 3: multiples of 128 up to 1 024; kind 2: also 2 048, 3 072, 4 096; kind 4: multiples of 64 up to 65 536), rows
 * outside [1, 2^20], split_ks outside 2 .. 8 (0 and 1: no slices), slices where the kernel does not sum them, a token id
 * outside [0, V), a position outside [0, 1 024], pos_rows outside [pos_offset + 1, 1 026], pos_offset other than 0 or 2
 * (kind 0 always uses 2), out_split 0 for kinds 2 .. 4, both tok and a (kinds 2, 3), or a missing input or output. */
typedef struct {
    int32_t kind, d;
    int64_t rows;
    const int32_t* tok; int64_t tok_stride; int32_t V; const float* embed; float scale;
    const int32_t* pos; int32_t pos_const, pos_offset, pos_rows; const float* pos_table;
    const float* ln_emb_g; const float* ln_emb_b;
    const float* a; const float* b;
    const float* split_part; int32_t split_ks; float split_unscale; const float* split_bias;
    const float* gamma; const float* beta; float eps, out_scale;
    const float* h;
    int32_t out_split;
} sealdec_norm_case_t;
int sealdec_debug_rownorm(const sealdec_norm_case_t* c, float* out, void* split1, void* split2, void* split3,
                          int32_t* overflow, uint32_t* path);
/* The top-k warp's threshold kernel of the generate (one CTA per row) on caller-supplied rows, through the same launch.
 * Host pointers: logits float32 [R][ld] (ld >= V; columns V .. ld-1 are not read), V <= 53 248, top_k >= 1 (values above
 * V select the smallest value).  Per row: out_thr = tau, the min(top_k, V)-th largest value (-0.0 returned as +0.0),
 * out_max = the row max, out_logsum = log(sum over x >= tau of exp(x - max)). */
int sealdec_debug_topk_threshold(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k, float* out_thr,
                                 float* out_max, float* out_logsum);
/* The same outputs from the threshold kernel the generate runs above V = 53 248: one cluster of ceil(V / 53 248) CTAs
 * per row, each staging a contiguous slice of the row, with histograms merged over distributed shared memory.  Any
 * 1 <= V <= 425 984 (so it can be checked at small V too); other arguments as above.  out_logsum is summed in a fixed
 * order: per CTA as the one-CTA kernel sums a row, then the CTA sums in rank order (decode_kernels.cuh). */
int sealdec_debug_topk_threshold_cluster(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k,
                                         float* out_thr, float* out_max, float* out_logsum);
/* average device time of the decoder's per-row statistics + top-2*beam kernel over R rows of V pseudo-random logits
 * (a later step of constrained beam search, per_row allowed tokens per row) */
int sealdec_debug_topk_rows(int64_t R, int32_t V, int32_t num_beams, int32_t per_row, int32_t iters, double* avg_us);
/* in-kernel timeline of CTA 0 of the GEMM kernel, in every gemm_mode (development aid): out20 (may be NULL) receives
 * the stamps of the last traced launch -- SM cycles at 0 entry, 1 prologue done, 2 first operands landed,
 * 3 last MMA issued, 4 last chunk complete, 5 tile stored, 6 exit; 7/8 globaltimer ns at entry / exit --
 * 9..16 the epilogue's four store passes (staged / stored) -- then tracing is switched on (enable != 0) or off. */
int sealdec_debug_gemm_trace(int enable, int64_t out20[20]);
/* per-unit timeline of CTA 0 of the last launches traced by sealdec_debug_gemm_trace (development aid): out[4i + e] for
 * the CTA's i-th work unit (i < 256) = SM cycles at e = 0 its first k-block of MMAs committed, 1 its K loop done,
 * 2 epilogue start, 3 epilogue end (0 where nothing was stamped).  Copies the first n <= 1 024 entries, then clears
 * the record.  Only in a library built with GEMM_UNIT_TRACE=1 (seal_b200/csrc/Makefile); otherwise SEALFM_EINVAL. */
int sealdec_debug_gemm_units(int64_t* out, int32_t n);
/* GEMM profiling: enable != 0 makes every following GEMM launch of this model be bracketed by CUDA
 * events on its stream.  When total_us/launches/flops are non-NULL the call first drains the device
 * and returns the summed device time, launch count and 2MNK flops recorded since the previous call,
 * then clears the record. */
int sealdec_profile_gemm(sealbart_t* model, int enable, double* total_us, int64_t* launches, double* flops);
/* microseconds spent (CUDA events) in the last generate, split by phase:
 * 0 encoder, 1 decoder layers, 2 lm_head, 3 select+expand (FM index), 4 total.  0 and 4 are taken on the caller's
 * stream; when the generate ran as two query slices, 1..3 of every step after the first are those of the first
 * slice (the second runs beside it on another stream). */
int sealdec_last_phase_us(const sealbart_t* model, double out5[5]);

#ifdef __cplusplus
}
#endif
#endif /* SEALDEC_H */
