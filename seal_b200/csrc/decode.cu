// Host orchestration + C ABI (include/sealdec.h) of the constrained beam-search decode:
// BART, pre-LayerNorm BART-family (Pegasus, mBART) and T5 weights, workspace, encoder pass, per-step decoder forward, fused select step.
#include "../../include/sealdec.h"
#include "bart_kernels.cuh"
#include "common.cuh"
#include "decode_kernels.cuh"
#include "fm_handle.hpp"
#include "preln_kernels.cuh"
#include "t5_kernels.cuh"
#include "wgmma_gemm.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <iterator>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <type_traits>
#include <vector>

using namespace sealb200;

namespace {

struct Lin {
    float* w = nullptr; float* b = nullptr; int out = 0, in = 0;
    float* w_hi = nullptr; float* w_lo = nullptr;          // TF32 split copies (gemm_mode 2)
    __half* w_h1 = nullptr; __half* w_h2 = nullptr;        // FP16 split copies of W * 2^s (gemm_mode 3)
    __nv_bfloat16* w_bf = nullptr;                         // gemm_mode 6: the only copy of W (w is null)
    float w_unscale = 1.f;                                 // 2^-s
    CUtensorMap map_hi{}, map_lo{}; bool maps_ready = false;
    CUtensorMap map2_hi{}, map2_lo{}; bool maps2_ready = false;   // 64-row boxes: one CTA's half of a cluster's W tile (gemm_mode 5)
};
struct LNp { float* g = nullptr; float* b = nullptr; };
struct EncLayerW { Lin qkv, o, fc1, fc2; LNp ln_attn, ln_final; };
struct DecLayerW { Lin qkv, o, cq, ckv, co, fc1, fc2; LNp ln_self, ln_cross, ln_final; };

// Every (re)allocation of a workspace buffer bumps this; a captured CUDA graph bakes buffer addresses in, so
// graphs captured under an older epoch are discarded.
uint64_t g_ws_epoch = 0;

// A device buffer that owns its memory: freed when the Buf goes out of scope.
struct Buf {
    void* p = nullptr; size_t bytes = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    void ensure(size_t need) {
        if (need <= bytes) return;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        ++g_ws_epoch;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

}  // namespace

struct sealbart {
    sealbart_config_t cfg{};          // a T5 handle fills it from its sealt5_config_t (max_positions = kT5MaxSource)
    // architecture: 0 BART (sealbart_create), 1 T5 (sealt5_create).  For T5 the Lin biases stay zero, LNp::g holds the
    // T5LayerNorm weights (EncLayerW: ln_attn = layer.0, ln_final = layer.1; DecLayerW: ln_self / ln_cross / ln_final =
    // layer.0 / 1 / 2), enc_ln_emb / dec_ln_emb the final_layer_norm of each stack, and fc1 is wi or [wi_0; wi_1].
    // 2 pre-LayerNorm BART family (sealbart_create_ex): BART's keys and biases; enc_ln_emb / dec_ln_emb hold
    // layernorm_embedding (allocated only if variant.layernorm_embedding), enc_ln_out / dec_ln_out the stacks' final
    // layer_norm; the position tables have max_positions + variant.position_offset rows.
    int arch = 0;
    sealbart_variant_t variant{};
    LNp enc_ln_out, dec_ln_out;
    sealt5_config_t t5{};
    float* t5_rel_enc = nullptr; float* t5_rel_dec = nullptr;          // layer-0 relative_attention_bias [buckets][heads]
    int32_t* t5_bkt_enc = nullptr; int32_t* t5_bkt_dec = nullptr;      // bucket of distance k - q, see t5_bucket_tables
    int device = 0;
    float* shared = nullptr; float* enc_pos = nullptr; float* dec_pos = nullptr;
    float* lm_head = nullptr; float* final_bias = nullptr;
    bool lm_head_given = false;
    // gemm_mode 6: the token-embedding / tied lm_head table and an untied lm_head in bf16 (shared / lm_head stay null)
    __nv_bfloat16* shared_bf = nullptr; __nv_bfloat16* lm_head_bf = nullptr;
    LNp enc_ln_emb, dec_ln_emb;
    Lin head;
    std::vector<EncLayerW> enc;
    std::vector<DecLayerW> dec;
    struct Slot { void* dst; uint64_t numel; bool bf16 = false; };     // bf16: rounded (RNE) into a bf16 matrix (gemm_mode 6)
    std::map<std::string, Slot> slots;
    std::set<std::string> loaded;
    std::vector<void*> allocs;
    uint64_t weight_bytes = 0;
    bool finalized = false;
    // workspace
    Buf enc_tok, enc_mask, ex, eqkv, etmp, ckv, src_off;
    bool enc_packed = false;          // the last encoder_forward ran on the real tokens only (src_off valid)
    Buf dx, dqkv, dtmp, dcq, logits, kc, vc;
    Buf ex_hi, ex_lo, eattn_hi, eattn_lo, effn_hi, effn_lo, dx_hi, dx_lo, dattn_hi, dattn_lo, dffn_hi, dffn_lo;   // activation splits (halves or TF32)
    Buf st_scores, st_tokens, st_lo, st_hi, st_pw, st_anc, st_mask;
    Buf st_rowmax, st_rowls, st_rule, st_cval, st_cidx, st_ccnt, st_wide;     // scratch between the kernels of a step
    Buf st_hstat;                     // [R][V / 128] lm_head tile statistics (HeadEpi)
    Buf st_thr;                       // [R][3] top-k warp statistics of each logits row (topk_threshold_kernel)
    Buf hy_score, hy_len, hy_tok, hy_valid, hy_lo, hy_hi, err, dbg_ids, a_hi, a_lo, splitk;
    std::vector<void*> split_allocs;
    int64_t launches = 0;
    uint32_t last_paths = 0;          // OR of the kPath* bits of every kernel branch the last model call took
    int* ovf = nullptr;              // where the producers raise "fp16 range exceeded" (set by every entry point)
    double phase_us[5] = {0, 0, 0, 0, 0};
    bool profile_gemm = false;
    int fused_head = -1;              // -1 $SEALB200_FUSED_HEAD (default on), 0 dense lm_head logits, 1 statistics epilogue
    bool poison_logits = false;
    int fused_head_steps = 0;         // steps of the last enqueued generate whose lm_head used the statistics epilogue       // testing: the logits buffer is filled with NaN before every statistics-epilogue head
    int topk_cluster_steps = 0;       // steps of the last generate whose top-k threshold ran topk_threshold_cluster_kernel
    int gemm_band = -1;               // sealdec_debug_gemm_ex: -1 tile order chosen by gemm_impl, 0 no bands, > 0 band size
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> gemm_events;
    double gemm_flops = 0;
    std::vector<cudaEvent_t> events;
    // host-buffer entry point: persistent device staging of the inputs (stable addresses -> CUDA graph reuse)
    Buf in_ids, in_mask, in_occ;
    // CUDA graphs of whole generate calls (small batches are launch-latency-bound: ~1 900 kernels per generate)
    struct GraphEntry { std::vector<uint8_t> key; uint64_t epoch = 0; cudaGraphExec_t exec = nullptr; int64_t launches = 0; uint32_t paths = 0; uint64_t stamp = 0;
                        int topk_cluster_steps = 0; };
    std::vector<GraphEntry> graphs;
    std::vector<std::vector<uint8_t>> seen_keys;     // shapes run once already (their buffers are sized): capture next time
    uint64_t graph_stamp = 0;
    int graph_policy = -1;            // -1 auto (small batches), 0 never, 1 whenever possible
    int last_used_graph = 0;
    bool tf32_ready = false;          // 3xTF32 weight splits exist (gemm_mode 2 fallback after an fp16 range overflow)
    int64_t overflow_fallbacks = 0;
    cudaStream_t stream = nullptr;    // the host-buffer entry point's own (non-blocking) stream
    // query slices (generate_enqueue): the second slice runs on slice_stream, forked from and joined back into the
    // caller's stream with two events, and has GEMM / mask-expansion scratch of its own
    int query_slices = -1;            // -1 $SEALB200_QUERY_SLICES (default on), 0 off, 1 on
    cudaStream_t slice_stream = nullptr;
    cudaEvent_t slice_fork = nullptr, slice_join = nullptr;
    Buf a_hi1, a_lo1, splitk1, st_wide1;
    Buf effn2, dffn2;                 // T5 gated-gelu: [rows][2 d_ff] output of the [wi_0; wi_1] GEMM
    ~sealbart() { for (void* p : allocs) cudaFree(p); for (void* p : split_allocs) cudaFree(p); }
};

namespace {

float* dalloc(sealbart* m, uint64_t numel) {
    void* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, std::max<uint64_t>(numel, 1) * sizeof(float)));
    CUDA_CHECK(cudaMemset(p, 0, std::max<uint64_t>(numel, 1) * sizeof(float)));
    m->allocs.push_back(p);
    m->weight_bytes += numel * sizeof(float);
    return static_cast<float*>(p);
}

__nv_bfloat16* dalloc_bf16(sealbart* m, uint64_t numel) {
    void* p = nullptr;
    CUDA_CHECK(cudaMalloc(&p, std::max<uint64_t>(numel, 1) * 2));
    CUDA_CHECK(cudaMemset(p, 0, std::max<uint64_t>(numel, 1) * 2));
    m->allocs.push_back(p);
    m->weight_bytes += numel * 2;
    return static_cast<__nv_bfloat16*>(p);
}

// sealbart_config_t::gemm_mode (include/sealdec.h)
enum GemmMode : int { kGemmTf32 = 2, kGemmFp16 = 3, kGemmFp16Cluster = 5, kGemmBf16 = 6 };
// 3xFP16 (one CTA per tile, or 2-CTA clusters): activations in fp16 halves, which an activation can overflow
bool is_3xfp16(int64_t mode) { return mode == kGemmFp16 || mode == kGemmFp16Cluster; }
// the modes whose lm_head may take the statistics epilogue (HeadEpi)
bool head_stats_mode(int mode) { return mode == kGemmFp16 || mode == kGemmBf16; }
// gemm_mode 6 stores every GEMM weight matrix (and the embedding table) once, in bf16; the other modes keep the fp32
// master and derive their splits from it at finalize
bool bf16_weights(const sealbart* m) { return m->cfg.gemm_mode == kGemmBf16; }

void make_lin(sealbart* m, Lin& l, int out, int in) {
    l.out = out; l.in = in;
    if (bf16_weights(m)) l.w_bf = dalloc_bf16(m, (uint64_t)out * in);
    else l.w = dalloc(m, (uint64_t)out * in);
    l.b = dalloc(m, out);
}
void make_ln(sealbart* m, LNp& l, int d) { l.g = dalloc(m, d); l.b = dalloc(m, d); }

void reg(sealbart* m, const std::string& key, float* dst, uint64_t numel) { m->slots[key] = {dst, numel}; }
void reg_mat(sealbart* m, const std::string& key, Lin& l, int row0, int rows) {
    const uint64_t off = (uint64_t)row0 * l.in, n = (uint64_t)rows * l.in;
    if (l.w_bf) m->slots[key] = {l.w_bf + off, n, true};
    else reg(m, key, l.w + off, n);
}
void reg_lin(sealbart* m, const std::string& prefix, Lin& l, int row0, int rows) {
    reg_mat(m, prefix + ".weight", l, row0, rows);
    reg(m, prefix + ".bias", l.b + row0, rows);
}
// the [V][d] token-embedding table under `key`
void make_shared(sealbart* m, const std::string& key) {
    const uint64_t n = (uint64_t)m->cfg.vocab_size * m->cfg.d_model;
    if (bf16_weights(m)) { m->shared_bf = dalloc_bf16(m, n); m->slots[key] = {m->shared_bf, n, true}; }
    else { m->shared = dalloc(m, n); reg(m, key, m->shared, n); }
}
void reg_ln(sealbart* m, const std::string& prefix, LNp& l, int d) {
    reg(m, prefix + ".weight", l.g, d);
    reg(m, prefix + ".bias", l.b, d);
}

// HF T5ForConditionalGeneration state_dict keys.  No biases and no position tables; the bucket tables are not weights.
void build_slots_t5(sealbart* m) {
    const auto& c = m->cfg;
    const int d = c.d_model, f = c.ffn_dim, V = c.vocab_size, nb = m->t5.relative_attention_num_buckets, H = c.heads;
    const bool gated = m->t5.ffn_kind == 1;
    make_shared(m, "shared.weight");
    m->final_bias = dalloc(m, V);                                          // zero: T5's lm_head has no bias
    m->enc_ln_emb.g = dalloc(m, d); reg(m, "encoder.final_layer_norm.weight", m->enc_ln_emb.g, d);
    m->dec_ln_emb.g = dalloc(m, d); reg(m, "decoder.final_layer_norm.weight", m->dec_ln_emb.g, d);
    m->t5_rel_enc = dalloc(m, (uint64_t)nb * H);
    reg(m, "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", m->t5_rel_enc, (uint64_t)nb * H);
    m->t5_rel_dec = dalloc(m, (uint64_t)nb * H);
    reg(m, "decoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", m->t5_rel_dec, (uint64_t)nb * H);
    auto reg_w = [&](const std::string& key, Lin& l, int row0, int rows) { reg_mat(m, key + ".weight", l, row0, rows); };
    auto ffn = [&](const std::string& p, Lin& fc1, Lin& fc2) {
        make_lin(m, fc1, gated ? 2 * f : f, d);
        if (gated) { reg_w(p + "DenseReluDense.wi_0", fc1, 0, f); reg_w(p + "DenseReluDense.wi_1", fc1, f, f); }
        else reg_w(p + "DenseReluDense.wi", fc1, 0, f);
        make_lin(m, fc2, d, f); reg_w(p + "DenseReluDense.wo", fc2, 0, d);
    };
    auto attn = [&](const std::string& p, Lin& qkv, Lin& o) {
        make_lin(m, qkv, 3 * d, d);
        reg_w(p + "q", qkv, 0, d); reg_w(p + "k", qkv, d, d); reg_w(p + "v", qkv, 2 * d, d);
        make_lin(m, o, d, d); reg_w(p + "o", o, 0, d);
    };
    auto norm = [&](const std::string& key, LNp& l) { l.g = dalloc(m, d); reg(m, key + ".layer_norm.weight", l.g, d); };
    m->enc.resize(c.encoder_layers);
    for (int i = 0; i < c.encoder_layers; ++i) {
        EncLayerW& L = m->enc[i];
        const std::string p = "encoder.block." + std::to_string(i) + ".layer.";
        attn(p + "0.SelfAttention.", L.qkv, L.o); norm(p + "0", L.ln_attn);
        ffn(p + "1.", L.fc1, L.fc2); norm(p + "1", L.ln_final);
    }
    m->dec.resize(c.decoder_layers);
    for (int i = 0; i < c.decoder_layers; ++i) {
        DecLayerW& L = m->dec[i];
        const std::string p = "decoder.block." + std::to_string(i) + ".layer.";
        attn(p + "0.SelfAttention.", L.qkv, L.o); norm(p + "0", L.ln_self);
        make_lin(m, L.cq, d, d); reg_w(p + "1.EncDecAttention.q", L.cq, 0, d);
        make_lin(m, L.ckv, 2 * d, d); reg_w(p + "1.EncDecAttention.k", L.ckv, 0, d); reg_w(p + "1.EncDecAttention.v", L.ckv, d, d);
        make_lin(m, L.co, d, d); reg_w(p + "1.EncDecAttention.o", L.co, 0, d);
        norm(p + "1", L.ln_cross);
        ffn(p + "2.", L.fc1, L.fc2); norm(p + "2", L.ln_final);
    }
}

// HF BartForConditionalGeneration state_dict keys; a pre-LayerNorm handle (arch 2) registers layernorm_embedding only
// for a variant that has it, the stacks' final layer_norm, and position tables of max_positions + position_offset rows.
void build_slots(sealbart* m) {
    const auto& c = m->cfg;
    const bool preln = m->arch == 2;
    const int d = c.d_model, f = c.ffn_dim, V = c.vocab_size, P = c.max_positions + (preln ? m->variant.position_offset : 2);
    make_shared(m, "model.shared.weight");
    m->enc_pos = dalloc(m, (uint64_t)P * d); reg(m, "model.encoder.embed_positions.weight", m->enc_pos, (uint64_t)P * d);
    m->dec_pos = dalloc(m, (uint64_t)P * d); reg(m, "model.decoder.embed_positions.weight", m->dec_pos, (uint64_t)P * d);
    m->final_bias = dalloc(m, V); reg(m, "final_logits_bias", m->final_bias, V);
    if (!preln || m->variant.layernorm_embedding) {
        make_ln(m, m->enc_ln_emb, d); reg_ln(m, "model.encoder.layernorm_embedding", m->enc_ln_emb, d);
        make_ln(m, m->dec_ln_emb, d); reg_ln(m, "model.decoder.layernorm_embedding", m->dec_ln_emb, d);
    }
    if (preln) {
        make_ln(m, m->enc_ln_out, d); reg_ln(m, "model.encoder.layer_norm", m->enc_ln_out, d);
        make_ln(m, m->dec_ln_out, d); reg_ln(m, "model.decoder.layer_norm", m->dec_ln_out, d);
    }
    m->enc.resize(c.encoder_layers);
    for (int i = 0; i < c.encoder_layers; ++i) {
        EncLayerW& L = m->enc[i];
        const std::string p = "model.encoder.layers." + std::to_string(i) + ".";
        make_lin(m, L.qkv, 3 * d, d);
        reg_lin(m, p + "self_attn.q_proj", L.qkv, 0, d); reg_lin(m, p + "self_attn.k_proj", L.qkv, d, d);
        reg_lin(m, p + "self_attn.v_proj", L.qkv, 2 * d, d);
        make_lin(m, L.o, d, d); reg_lin(m, p + "self_attn.out_proj", L.o, 0, d);
        make_ln(m, L.ln_attn, d); reg_ln(m, p + "self_attn_layer_norm", L.ln_attn, d);
        make_lin(m, L.fc1, f, d); reg_lin(m, p + "fc1", L.fc1, 0, f);
        make_lin(m, L.fc2, d, f); reg_lin(m, p + "fc2", L.fc2, 0, d);
        make_ln(m, L.ln_final, d); reg_ln(m, p + "final_layer_norm", L.ln_final, d);
    }
    m->dec.resize(c.decoder_layers);
    for (int i = 0; i < c.decoder_layers; ++i) {
        DecLayerW& L = m->dec[i];
        const std::string p = "model.decoder.layers." + std::to_string(i) + ".";
        make_lin(m, L.qkv, 3 * d, d);
        reg_lin(m, p + "self_attn.q_proj", L.qkv, 0, d); reg_lin(m, p + "self_attn.k_proj", L.qkv, d, d);
        reg_lin(m, p + "self_attn.v_proj", L.qkv, 2 * d, d);
        make_lin(m, L.o, d, d); reg_lin(m, p + "self_attn.out_proj", L.o, 0, d);
        make_ln(m, L.ln_self, d); reg_ln(m, p + "self_attn_layer_norm", L.ln_self, d);
        make_lin(m, L.cq, d, d); reg_lin(m, p + "encoder_attn.q_proj", L.cq, 0, d);
        make_lin(m, L.ckv, 2 * d, d);
        reg_lin(m, p + "encoder_attn.k_proj", L.ckv, 0, d); reg_lin(m, p + "encoder_attn.v_proj", L.ckv, d, d);
        make_lin(m, L.co, d, d); reg_lin(m, p + "encoder_attn.out_proj", L.co, 0, d);
        make_ln(m, L.ln_cross, d); reg_ln(m, p + "encoder_attn_layer_norm", L.ln_cross, d);
        make_lin(m, L.fc1, f, d); reg_lin(m, p + "fc1", L.fc1, 0, f);
        make_lin(m, L.fc2, d, f); reg_lin(m, p + "fc2", L.fc2, 0, d);
        make_ln(m, L.ln_final, d); reg_ln(m, p + "final_layer_norm", L.ln_final, d);
    }
}

// ---- launch helpers ----------------------------------------------------------------------------
// pending: a split-K GEMM whose slices are still unsummed -- its consumer (add+LN on small batches, the attention kernels)
// folds the finish pass in; defer_rows = how many rows that consumer accepts (0: the GEMM must finish itself)
// head: the lm_head GEMM may use the statistics epilogue (HeadEpi); head_fused reports that it did
// slice: 1 = the second query slice of a generate, which has its own GEMM scratch (a_hi1, a_lo1, splitk1)
struct Ctx { sealbart* m; cudaStream_t s; SplitSrc pending{}; int64_t defer_rows = 0; HeadEpi head{}; bool head_fused = false; int slice = 0; };

// ---- TMA descriptors ------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        if (!p || q != cudaDriverEntryPointSuccess) throw ApiError(SEALFM_ECUDA, "cuTensorMapEncodeTiled unavailable");
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// row-major [rows][K] of T (fp32, fp16 or bf16), box = 128 bytes of K x box_rows, 128B swizzle, zero fill out of bounds
template <typename T> void make_map(CUtensorMap* map, const T* ptr, uint64_t rows, uint64_t K, uint64_t ld, uint32_t box_rows) {
    cuuint64_t dims[2] = {K, rows};
    cuuint64_t strides[1] = {ld * sizeof(T)};
    cuuint32_t box[2] = {(cuuint32_t)(128 / sizeof(T)), box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                   : std::is_same<T, __half>::value      ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                                                          : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUresult r = encode_tiled()(map, dt, 2, const_cast<T*>(ptr), dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) throw ApiError(SEALFM_ECUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

constexpr int64_t kAddLnRowMax = 2048;      // up to this many rows add+LN runs one CTA per row

// sealbart_get_stat(model, "last_paths"): one bit per kernel branch of the BART forward (include/sealdec.h), set on
// the host next to the launch it names
enum : uint32_t {
    kPathEncPacked = 1u << 0, kPathEncUnpacked = 1u << 1,
    kPathSelfQuery = 1u << 2, kPathSelfRounds3 = 1u << 3, kPathSelfRounds8 = 1u << 4, kPathSelfLong = 1u << 5,
    kPathCrossSmall = 1u << 6, kPathCrossGrouped = 1u << 7,
    kPathAddLnRow = 1u << 8, kPathAddLnWarp = 1u << 9,
    kPathSplitKDeferred = 1u << 10, kPathSplitKFinish = 1u << 11, kPathGemmFullTile = 1u << 12, kPathGemmCluster = 1u << 13,
    kPathGemmTf32 = 1u << 14, kPathQuerySlices = 1u << 15,
    kPathT5EncAttn = 1u << 16, kPathT5DecAttn = 1u << 17, kPathT5Rms = 1u << 18, kPathT5Relu = 1u << 19, kPathT5Gate = 1u << 20,
    kPathT5RmsWide = 1u << 21, kPathPreLn = 1u << 22, kPathPreLnEmbedLn = 1u << 23, kPathGemmBf16 = 1u << 24,
};

void split_into(cudaStream_t s, const float* x, float* hi, float* lo, uint64_t numel) {
    const int64_t n4 = (int64_t)(numel / 4);
    const int blocks = (int)std::min<int64_t>((n4 + 255) / 256, (int64_t)sm_count() * 8);
    split_tf32_kernel<<<std::max(blocks, 1), 256, 0, s>>>(n4, reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(hi),
                                                          reinterpret_cast<float4*>(lo));
    CUDA_CHECK(cudaGetLastError());
}

// An activation tensor as the GEMMs see it: plain fp32 and/or its split in the gemm_mode's format (X3Format).
struct Act {
    float* x = nullptr; float* hi = nullptr; float* lo = nullptr;   // fp32 / TF32 split
    __half* h1 = nullptr; __half* h2 = nullptr;                     // FP16 split
    __nv_bfloat16* b1 = nullptr; __nv_bfloat16* b2 = nullptr; __nv_bfloat16* b3 = nullptr;   // 3xBF16 split
};

SplitOut split_of(const Act& a, int* overflow) {
    SplitOut so;
    if (a.hi) { so.a = a.hi; so.b = a.lo; so.kind = 1; }
    else if (a.h1) { so.a = a.h1; so.b = a.h2; so.kind = 2; so.overflow = overflow; }
    return so;
}

// f(so) with the split output a producer of activation a writes: SplitBf16 in gemm_mode 6, SplitOut (split_of)
// otherwise.  The producer kernels are instantiated per split type, so f launches kernel<decltype(so)>.
template <typename F> void with_split(const sealbart* m, const Act& a, F&& f) {
    if (bf16_weights(m)) f(SplitBf16{a.b1, a.b2, a.b3});
    else f(split_of(a, m->ovf));
}
// the embedding table a producer with split type SO gathers from
template <class SO> const EmbT<SO>* embed_table(const sealbart* m) {
    if constexpr (std::is_same<SO, SplitBf16>::value) return m->shared_bf;
    else return m->shared;
}

// Buffers hi / lo (and plain, if not null) as an Act from element off on: the TF32 split in gemm_mode 2, the fp16
// split in the 3xFP16 modes, the three bf16 pieces in gemm_mode 6 (b1 and b3 in the two halves of hi -- every split
// buffer holds 4 bytes per element -- b2 in lo).  plain is null for activations whose producers write the split only.
Act act_view(int gemm_mode, float* plain, const Buf& hi, const Buf& lo, int64_t off = 0) {
    Act a;
    if (plain) a.x = plain + off;
    if (gemm_mode == kGemmTf32) { a.hi = hi.as<float>() + off; a.lo = lo.as<float>() + off; }
    else if (gemm_mode == kGemmBf16) { a.b1 = hi.as<__nv_bfloat16>() + off; a.b2 = lo.as<__nv_bfloat16>() + off; a.b3 = hi.as<__nv_bfloat16>() + hi.bytes / 4 + off; }
    else if (is_3xfp16(gemm_mode)) { a.h1 = hi.as<__half>() + off; a.h2 = lo.as<__half>() + off; }
    return a;
}

template <typename T, int ACT, int CL, bool HEAD = false>
void gemm_launch(cudaStream_t s, int ctas, const CUtensorMap& ahi, const CUtensorMap& alo, const CUtensorMap& whi, const CUtensorMap& wlo,
                 int64_t M, int N, int K, const float* bias, float w_unscale, float* C, T* C1, T* C2, int ldc, int n_fastest, int m_band,
                 int* ovf, int k_slices, int64_t slice_stride, const HeadEpi& he = HeadEpi{}, T* C3 = nullptr) {
    auto kern = wgmma_gemm_x3_kernel<T, ACT, CL, HEAD>;
    CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM));
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)ctas); cfg.blockDim = dim3(GTHREADS); cfg.dynamicSmemBytes = G_SMEM; cfg.stream = s;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, ahi, alo, whi, wlo, (int)M, N, K, bias, w_unscale, C, C1, C2, ldc, n_fastest, m_band, ovf,
                                  k_slices, slice_stride, he, C3));
}

// f(std::integral_constant<int, ACT>{}) for the epilogue activation act: kernels are instantiated per activation
template <typename F> void with_act(int act, F&& f) {
    if (act == kActGelu) f(std::integral_constant<int, kActGelu>{});
    else if (act == kActRelu) f(std::integral_constant<int, kActRelu>{});
    else f(std::integral_constant<int, kActNone>{});
}

// C = A W^T + b (+ the epilogue activation act: kActNone / kActGelu / kActRelu, wgmma_gemm.cuh) on the tensor cores:
// gemm_mode 3 / 5 = 3xFP16 (one CTA per tile / clusters of 2 sharing W), 6 = 3xBF16 (bf16 weights), 2 = 3xTF32 (fp32
// range: the fallback when an activation leaves the fp16 range).  Operands arrive pre-split from the producing kernel
// (A.h1/A.h2, A.b1/A.b2/A.b3 or A.hi/A.lo); they are split here only if the producer did not.
void gemm_impl(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act);

void gemm(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act) {
    sealbart* m = cx.m;
    if (!m->profile_gemm || M == 0) { gemm_impl(cx, M, N, K, A, lda, l, C, ldc, act); return; }
    cudaEvent_t a, b;
    CUDA_CHECK(cudaEventCreate(&a)); CUDA_CHECK(cudaEventCreate(&b));
    CUDA_CHECK(cudaEventRecord(a, cx.s));
    gemm_impl(cx, M, N, K, A, lda, l, C, ldc, act);
    CUDA_CHECK(cudaEventRecord(b, cx.s));
    m->gemm_events.emplace_back(a, b);
    m->gemm_flops += 2.0 * (double)M * N * K;
}

// K slices of a 3xFP16 / 3xBF16 GEMM of `tiles` output tiles: skinny problems (a few tiles for the whole GPU) split K
// so that the serial K loop of a tile is spread over up to 8 CTAs, then sum the partial tiles in a fixed order
int split_k_slices(int tiles, int kblocks) {
    int k_slices = 1;
    static const int force_slices = [] { const char* e = std::getenv("SEALB200_KSLICES"); return e ? std::atoi(e) : 0; }();
    if (tiles * 2 <= sm_count() && kblocks >= 4) {
        k_slices = std::min(8, std::min(kblocks / 2, sm_count() / tiles));
        if (force_slices > 0) k_slices = std::min(force_slices, kblocks);     // experiments only
        while (k_slices > 1 && kblocks % k_slices) --k_slices;
    }
    return k_slices;
}

// m fastest with more A than a band holds (the lm_head at thousands of rows): bands of m tiles whose A pieces (a_bytes
// per element: 4 for the two halves, 6 for three bf16 pieces) take <= 8 MB of the 50 MB L2, so A is read from HBM once
// and W once per band (wgmma_gemm.cuh, tile_coords).  8 MB (16 tiles at K = 1 024 in 3xFP16) measured fastest of
// 4 / 8 / 16 / 32 MB bands for the lm_head at 15 000 rows (tools/head_bench.py); the band shares the L2 with the
// streaming W tiles and the logits stores.
int band_tiles(const sealbart* m, int n_fastest, int64_t M, int K, int a_bytes) {
    const int64_t a_tile_bytes = (int64_t)GM * K * a_bytes, band_bytes = 8ll << 20;
    const int band = (!n_fastest && M * K * a_bytes > band_bytes) ? (int)std::max<int64_t>(1, band_bytes / a_tile_bytes) : 0;
    return m->gemm_band >= 0 ? m->gemm_band : band;
}

// The x3 GEMM's operand formats, by element type T: the Act fields of A's pieces (C's split outputs use the same
// fields), the Lin fields of W's pieces, whether the epilogue unscales W by l.w_unscale, whether split-K, L2 bands and
// the lm_head statistics epilogue apply (tuned), and the last_paths bits of every call and of the whole-tile launch.
// 3xBF16's W is one piece; its kernel reads A's third piece in the W lo slot.
template <typename T> using ActField = T* Act::*;
template <typename T> using LinField = T* Lin::*;
template <typename T> struct X3Format;
template <> struct X3Format<__half> {                 // 3xFP16 (modes 3, 5): A = h1 + h2, W * 2^s = w_h1 + w_h2
    static constexpr ActField<__half> piece[] = {&Act::h1, &Act::h2};
    static constexpr LinField<__half> w = &Lin::w_h1, w2 = &Lin::w_h2;
    static constexpr bool scaled_w = true, tuned = true;
    static constexpr uint32_t path_call = 0, path_tile = kPathGemmFullTile;
};
template <> struct X3Format<__nv_bfloat16> {          // 3xBF16 (mode 6): A = b1 + b2 + b3, W once in bf16
    static constexpr ActField<__nv_bfloat16> piece[] = {&Act::b1, &Act::b2, &Act::b3};
    static constexpr LinField<__nv_bfloat16> w = &Lin::w_bf;
    static constexpr bool scaled_w = false, tuned = true;
    static constexpr uint32_t path_call = kPathGemmBf16, path_tile = 0;
};
template <> struct X3Format<float> {                  // 3xTF32 (mode 2): A = hi + lo, W = w_hi + w_lo; band 0, gemm_band ignored
    static constexpr ActField<float> piece[] = {&Act::hi, &Act::lo};
    static constexpr LinField<float> w = &Lin::w_hi, w2 = &Lin::w_lo;
    static constexpr bool scaled_w = false, tuned = false;    // unscaled: after an overflow fallback l.w_unscale is 3xFP16's
    static constexpr uint32_t path_call = 0, path_tile = kPathGemmTf32;
};

// f(T()) with the element type T of gemm_mode's operand format
template <typename F> void with_format(int mode, F&& f) {
    if (mode == kGemmBf16) f(__nv_bfloat16());
    else if (is_3xfp16(mode)) f(__half());
    else f(0.f);
}

// x (n fp32 values) split into format T's pieces in hi / lo (grown to fit) on stream s, in act_view's layout but with
// bf16's third piece n elements into hi.  3xFP16 raises *ovf for a value past the fp16 range.
template <typename T> Act split_act(cudaStream_t s, float* x, int64_t n, Buf& hi, Buf& lo, int* ovf) {
    Act a{x};
    const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8);
    if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        hi.ensure((size_t)n * 4); lo.ensure((size_t)n * 2);
        a.b1 = hi.as<T>(); a.b2 = lo.as<T>(); a.b3 = a.b1 + n;
        split_bf16x3_kernel<<<blocks, 256, 0, s>>>(n, x, a.b1, a.b2, a.b3);
    } else if constexpr (std::is_same<T, __half>::value) {
        hi.ensure((size_t)n * 2); lo.ensure((size_t)n * 2);
        a.h1 = hi.as<T>(); a.h2 = lo.as<T>();
        split_half_kernel<<<blocks, 256, 0, s>>>(n, x, 1.0f, a.h1, a.h2, ovf);
    } else {
        hi.ensure((size_t)n * 4); lo.ensure((size_t)n * 4);
        a.hi = hi.as<T>(); a.lo = lo.as<T>();
        split_into(s, x, a.hi, a.lo, (uint64_t)n);
    }
    CUDA_CHECK(cudaGetLastError());
    return a;
}

template <typename T> void gemm_x3(Ctx& cx, int64_t M, int N, int K, const Act& A, Lin& l, const Act& C, int ldc, int act) {
    using F = X3Format<T>;
    constexpr int pieces = (int)std::size(F::piece);
    sealbart* m = cx.m;
    const int tiles = (int)(((N + GN - 1) / GN) * ((M + GM - 1) / GM));
    const int n_fastest = ((int64_t)M >= (int64_t)N) ? 1 : 0;     // stream the larger operand once
    Act a = A;
    if (!(a.*F::piece[0])) {
        a = split_act<T>(cx.s, A.x, M * K, cx.slice ? m->a_hi1 : m->a_hi, cx.slice ? m->a_lo1 : m->a_lo, m->ovf);
        m->launches++;
    }
    CUtensorMap ma[3];
    for (int i = 0; i < pieces; ++i) make_map(&ma[i], a.*F::piece[i], M, K, K, GM);
    if (!l.maps_ready) {
        make_map(&l.map_hi, l.*F::w, N, K, K, GN);
        if constexpr (pieces == 2) make_map(&l.map_lo, l.*F::w2, N, K, K, GN);
        l.maps_ready = true;
    }
    const CUtensorMap& w_lo = pieces == 3 ? ma[2] : l.map_lo;
    T* const c1 = C.*F::piece[0]; T* const c2 = C.*F::piece[1]; T* c3 = nullptr;
    if constexpr (pieces == 3) c3 = C.*F::piece[2];
    const float unscale = F::scaled_w ? l.w_unscale : 1.0f;
    m->last_paths |= F::path_call;
    const int k_slices = F::tuned ? split_k_slices(tiles, K / UK16) : 1;
    if constexpr (std::is_same<T, __half>::value) {
        if (m->cfg.gemm_mode == kGemmFp16Cluster && k_slices == 1 && M > GM) {
            // clusters of 2 CTAs on vertically adjacent tiles: the W tile is loaded once (TMA multicast) for both
            if (!l.maps2_ready) { make_map(&l.map2_hi, l.w_h1, N, K, K, GN / 2); make_map(&l.map2_lo, l.w_h2, N, K, K, GN / 2); l.maps2_ready = true; }
            const int groups = (int)((M + 2 * GM - 1) / (2 * GM)) * ((N + GN - 1) / GN);
            const int ctas = 2 * std::min(groups, sm_count() / 2);
            with_act(act, [&](auto Ac) {
                gemm_launch<__half, decltype(Ac)::value, 2>(cx.s, ctas, ma[0], ma[1], l.map2_hi, l.map2_lo, M, N, K, l.b, unscale, C.x, c1, c2, ldc, n_fastest, 0, m->ovf, 1, 0);
            });
            m->launches++; m->last_paths |= kPathGemmCluster;
            return;
        }
    }
    if constexpr (F::tuned) {
        if (k_slices > 1) {
            Buf& splitk = cx.slice ? m->splitk1 : m->splitk;
            const int64_t slice_stride = (int64_t)M * ldc;
            splitk.ensure((size_t)k_slices * slice_stride * 4);
            float* part = splitk.as<float>();
            const int ctas2 = std::min(tiles * k_slices, sm_count());
            gemm_launch<T, kActNone, 1>(cx.s, ctas2, ma[0], ma[1], l.map_hi, w_lo, M, N, K, nullptr, 1.0f, part, nullptr, nullptr, ldc, n_fastest, 0,
                                        m->ovf, k_slices, slice_stride);
            m->launches++;
            if (M <= cx.defer_rows && act == kActNone && !C.hi && !C.h1 && !C.b1 && ldc == N && l.b) {     // C has no split output: summed by the consumer kernel
                cx.pending = SplitSrc{part, k_slices, slice_stride, l.b, unscale};
                m->last_paths |= kPathSplitKDeferred;
                return;
            }
            const int fblocks = (int)std::min<int64_t>((M * (ldc / 4) + 255) / 256, (int64_t)sm_count() * 8);
            with_act(act, [&](auto Ac) {
                launch_k(gemm_splitk_finish_kernel<decltype(Ac)::value, T>, fblocks, 256, 0, cx.s, M, N, ldc, k_slices, slice_stride, part, l.b, unscale,
                         C.x, c1, c2, m->ovf, c3);
            });
            CUDA_CHECK(cudaGetLastError()); m->launches++; m->last_paths |= kPathSplitKFinish;
            return;
        }
    }
    const int band = F::tuned ? band_tiles(m, n_fastest, M, K, pieces * (int)sizeof(T)) : 0;
    const int ctas = std::min(tiles, sm_count());
    if (F::tuned && cx.head.stats && act == kActNone) {
        if constexpr (F::tuned)
            gemm_launch<T, kActNone, 1, true>(cx.s, ctas, ma[0], ma[1], l.map_hi, w_lo, M, N, K, l.b, unscale, C.x, nullptr, nullptr, ldc, n_fastest, band,
                                              m->ovf, 1, 0, cx.head);
        cx.head_fused = true;
    } else
        with_act(act, [&](auto Ac) {
            gemm_launch<T, decltype(Ac)::value, 1>(cx.s, ctas, ma[0], ma[1], l.map_hi, w_lo, M, N, K, l.b, unscale, C.x, c1, c2, ldc, n_fastest, band,
                                                   m->ovf, 1, 0, HeadEpi{}, c3);
        });
    m->launches++; m->last_paths |= F::path_tile;
}

void gemm_impl(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act) {
    if (M == 0) return;
    if (act == kActRelu) cx.m->last_paths |= kPathT5Relu;
    with_format(cx.m->cfg.gemm_mode, [&](auto t) {
        using T = decltype(t);
        if (K % GemmElem<T>::KE || lda != K || !(l.*X3Format<T>::w))
            throw ApiError(SEALFM_EINVAL, "GEMM: K must be a multiple of 64 (3xFP16, 3xBF16) / 32 (3xTF32) with contiguous operands");
        gemm_x3<T>(cx, M, N, K, A, l, C, ldc, act);
    });
}

void add_ln(Ctx& cx, int64_t rows, int d, const float* a, const float* b, const LNp& ln, const Act& out) {
    const SplitSrc ps = cx.pending;
    cx.pending = SplitSrc{};
    with_split(cx.m, out, [&](auto so) {
        using SO = decltype(so);
        if (rows <= kAddLnRowMax)          // small batches: a CTA per row (and the split-K finish of the GEMM before it, if pending)
            launch_k(add_ln_row_kernel<SO>, (unsigned)rows, 128, 0, cx.s, rows, d, a, b, (const float*)ln.g, (const float*)ln.b, out.x, so, ps);
        else
            launch_k(add_ln_kernel<SO>, (unsigned)((rows + 3) / 4), 128, 0, cx.s, rows, d, a, b, (const float*)ln.g, (const float*)ln.b, out.x, so);
    });
    cx.m->launches++;
    cx.m->last_paths |= rows <= kAddLnRowMax ? kPathAddLnRow : kPathAddLnWarp;
}

__global__ void prep_enc_kernel(int64_t n, int S, const int64_t* __restrict__ ids, const int64_t* __restrict__ mask,
                                int32_t* __restrict__ tok, int32_t* __restrict__ m32, int32_t* __restrict__ pos) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    tok[i] = (int32_t)ids[i];
    m32[i] = mask[i] != 0;
    pos[i] = (int32_t)(i % S);
}

// Source lengths, their exclusive prefix sum (src_off[Q+1]) and whether every mask row is "ones then zeros"
// (right padding) -- the precondition for running the encoder on the real tokens only.  One block.
__global__ void __launch_bounds__(1024) pack_lengths_kernel(int64_t Q, int S, const int64_t* __restrict__ mask,
                                                            int32_t* __restrict__ src_off, int64_t* __restrict__ info,
                                                            int64_t hint, int32_t* __restrict__ hint_err) {
    __shared__ int64_t part[1024];
    __shared__ int bad;
    const int t = threadIdx.x;
    if (t == 0) bad = 0;
    __syncthreads();
    const int64_t per = (Q + 1023) / 1024, q0 = t * per, q1 = q0 + per < Q ? q0 + per : Q;
    int64_t sum = 0; int notprefix = 0;
    for (int64_t q = q0; q < q1; ++q) {
        int len = 0;
        for (int s2 = 0; s2 < S; ++s2) { const int on = mask[q * S + s2] != 0; if (on && s2 != len) notprefix = 1; len += on; }
        sum += len;
    }
    part[t] = sum;
    if (notprefix) atomicExch(&bad, 1);
    __syncthreads();
    if (t == 0) {
        int64_t run = 0;
        for (int i = 0; i < 1024; ++i) { const int64_t v = part[i]; part[i] = run; run += v; }
        info[0] = run; info[1] = bad;
        if (hint >= 0 && hint_err && (run != hint || bad)) *hint_err = 1;      // the caller's token count was wrong
    }
    __syncthreads();
    int64_t run = part[t];
    for (int64_t q = q0; q < q1; ++q) {
        src_off[q] = (int32_t)run;
        int len = 0;
        for (int s2 = 0; s2 < S; ++s2) len += mask[q * S + s2] != 0;
        run += len;
    }
    if (t == 0) src_off[Q] = (int32_t)info[0];
}

__global__ void prep_enc_packed_kernel(int64_t n, int S, const int64_t* __restrict__ ids, const int32_t* __restrict__ src_off,
                                       int32_t* __restrict__ tok, int32_t* __restrict__ pos) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t q = i / S; const int s2 = (int)(i % S);
    if (s2 < src_off[q + 1] - src_off[q]) { const int64_t dst = src_off[q] + s2; tok[dst] = (int32_t)ids[i]; pos[dst] = s2; }
}

// gs = beams per group: the first beam of every group starts at 0, the others at -1e9 (seal/beam_search.py:214-216;
// with diverse beam groups 4.13's group_beam_search sets beam_scores[:, ::gs] = 0)
__global__ void init_state_kernel(int64_t R, int gs, int T, int start_tok, int pad, uint64_t lo0, uint64_t hi0,
                                  float* __restrict__ scores, int32_t* __restrict__ tokens, uint64_t* __restrict__ lo,
                                  uint64_t* __restrict__ hi, uint64_t* __restrict__ pw, int32_t* __restrict__ anc) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= R) return;
    scores[r] = (r % gs) == 0 ? 0.f : -1e9f;
    for (int t = 0; t < T; ++t) { tokens[r * T + t] = t == 0 ? start_tok : pad; anc[r * T + t] = (int32_t)r; }
    lo[r] = lo0; hi[r] = hi0; pw[r] = hi0 - lo0;
}

__global__ void ids_to_tokens_kernel(int64_t R, int t, int T, const int64_t* __restrict__ ids, int32_t* __restrict__ tokens,
                                     int32_t* __restrict__ anc) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= R) return;
    for (int i = 0; i < T; ++i) { tokens[r * T + i] = i < t ? (int32_t)ids[r * t + i] : 0; anc[r * T + i] = (int32_t)r; }
}

struct Dims {
    int64_t Q, S, R; int B, T, d, f, V, ld, W;
    int64_t G = 0; const int32_t* grp_query = nullptr; const int32_t* grp_start = nullptr;   // ragged row groups (re-scoring)
    // A query slice (generate_enqueue): queries [q0, q0 + Q) of a batch of Qb queries and Rb rows.  Its rows start at
    // r0 = q0 * B in every row-indexed buffer; the KV cache keeps the batch's row stride Rb, its ancestor indices are
    // relative to r0.  Qb = Rb = 0: not a slice.
    int64_t q0 = 0, r0 = 0, Qb = 0, Rb = 0;
};

void ensure_workspace(sealbart* m, const Dims& D) {
    const int64_t Tk = D.Q * D.S;
    const int Ld = m->cfg.decoder_layers;
    m->enc_tok.ensure(Tk * 4 * 2); m->enc_mask.ensure(Tk * 4); m->src_off.ensure((D.Q + 1) * 4 + 16 + 16);
    m->ex.ensure(Tk * D.d * 4); m->eqkv.ensure(Tk * 3 * D.d * 4); m->etmp.ensure(Tk * D.d * 4);
    m->ckv.ensure((size_t)Ld * Tk * 2 * D.d * 4);
    m->dx.ensure(D.R * D.d * 4); m->dqkv.ensure(D.R * 3 * D.d * 4); m->dtmp.ensure(D.R * D.d * 4); m->dcq.ensure(D.R * D.d * 4);
    m->logits.ensure((size_t)D.R * D.ld * 4);
    m->kc.ensure((size_t)Ld * D.T * D.R * D.d * 4); m->vc.ensure((size_t)Ld * D.T * D.R * D.d * 4);
    m->st_scores.ensure(2 * D.R * 4); m->st_tokens.ensure(2 * D.R * D.T * 4);
    m->st_lo.ensure(2 * D.R * 8); m->st_hi.ensure(2 * D.R * 8); m->st_pw.ensure(2 * D.R * 8);
    m->st_anc.ensure(2 * D.R * D.T * 4); m->st_mask.ensure((size_t)2 * D.R * D.W * 4);
    m->st_rowmax.ensure(D.R * 4); m->st_rowls.ensure(D.R * 4); m->st_rule.ensure(D.R);
    m->st_hstat.ensure((size_t)D.R * ((D.V + GN - 1) / GN) * 8);
    m->st_thr.ensure((size_t)D.R * 3 * 4);
    m->st_cval.ensure((size_t)D.R * 2 * D.B * 4); m->st_cidx.ensure((size_t)D.R * 2 * D.B * 4); m->st_ccnt.ensure(D.R * 4);
    if (m->arch == 1 && m->t5.ffn_kind == 1) { m->effn2.ensure(Tk * 2 * D.f * 4); m->dffn2.ensure(D.R * 2 * D.f * 4); }
    {
        m->ex_hi.ensure(Tk * D.d * 4); m->ex_lo.ensure(Tk * D.d * 4);
        m->eattn_hi.ensure(Tk * D.d * 4); m->eattn_lo.ensure(Tk * D.d * 4);
        m->effn_hi.ensure(Tk * D.f * 4); m->effn_lo.ensure(Tk * D.f * 4);
        m->dx_hi.ensure(D.R * D.d * 4); m->dx_lo.ensure(D.R * D.d * 4);
        m->dattn_hi.ensure(D.R * D.d * 4); m->dattn_lo.ensure(D.R * D.d * 4);
        m->dffn_hi.ensure(D.R * D.f * 4); m->dffn_lo.ensure(D.R * D.f * 4);
    }
    m->err.ensure(16);
}

// ---- T5 forward --------------------------------------------------------------------------------------
// Pre-norm layers: x (fp32, the residual stream) += sublayer(RMSNorm(x)).  The plain half of the Act x holds the
// residual, its split half the normed operand of the next GEMM: every t5_rms launch adds the previous sublayer's output
// (or gathers the embedding), stores the residual and writes RMSNorm(x) with the next sublayer's weight -- after the
// last layer the stack's final_layer_norm (and, in the decoder, the d_model^-0.5 output scale).
void t5_rms(Ctx& cx, int64_t rows, int d, const int32_t* tok, int64_t tok_stride, const Act& x, const float* b, const float* w,
            float out_scale) {
    const SplitSrc ps = cx.pending;
    cx.pending = SplitSrc{};
    const bool wide = d > 4 * 128 * kT5RmsVec;
    with_split(cx.m, x, [&](auto so) {
        using SO = decltype(so);
        launch_k(wide ? t5_rms_row_kernel<kT5RmsVecWide, SO> : t5_rms_row_kernel<kT5RmsVec, SO>, (unsigned)rows, 128, 0, cx.s, rows, d, tok, tok_stride,
                 embed_table<SO>(cx.m), x.x, b, ps, w, cx.m->t5.layer_norm_epsilon, out_scale, so);
    });
    cx.m->launches++;
    cx.m->last_paths |= wide ? kPathT5RmsWide : kPathT5Rms;
}

// wi (ReLU epilogue) or [wi_0; wi_1] + gate, then wo into tmp (split-K slices left to the next t5_rms)
void t5_ffn(Ctx& cx, int64_t rows, int d, int f, const Act& x, Lin& fc1, Lin& fc2, const Act& ffn, float* ffn2, const Act& tmp) {
    sealbart* m = cx.m;
    if (m->t5.ffn_kind == 1) {
        gemm(cx, rows, 2 * f, d, x, d, fc1, Act{ffn2}, 2 * f, kActNone);
        const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((rows * (f / 4) + 255) / 256, (int64_t)sm_count() * 8));
        with_split(m, ffn, [&](auto so) { launch_k(t5_gate_kernel<decltype(so)>, (unsigned)blocks, 256, 0, cx.s, rows, f, (const float*)ffn2, so); });
        m->launches++; m->last_paths |= kPathT5Gate;
    } else
        gemm(cx, rows, f, d, x, d, fc1, ffn, f, kActRelu);
    cx.defer_rows = INT64_MAX;
    gemm(cx, rows, d, f, ffn, f, fc2, tmp, d, kActNone);
    cx.defer_rows = 0;
}

// The activations of one stack's layers as the GEMMs see them.  x: the residual stream (plain) and the next GEMM's
// operand (split); qkv, tmp, cq: plain GEMM outputs; attn, ffn: the split operands of the o / co and fc2 GEMMs, whose
// producers write no plain copy; ffn2: the [rows][2 d_ff] output of T5's gated [wi_0; wi_1] GEMM.
struct Acts { Act x, qkv, attn, tmp, cq, ffn; float* ffn2 = nullptr; };

// One decoder step: rows r0 .. r0 + R of the activation buffers; at the compact first step a row stands for row_mul
// beams.  Rc: the KV cache's row stride; Tk, ckv_q0, m32, soff_x: the encoder side of the step's queries (packed,
// src_off holds absolute ckv rows; unpacked, query q's rows are q * S).
struct DecStep : Acts {
    int64_t R = 0, Rc = 0, Tk = 0, ckv_q0 = 0; int row_mul = 1, pos = 0; bool compact = false;
    const int32_t* tokens = nullptr; const int32_t* anc = nullptr; const int32_t* m32 = nullptr; const int32_t* soff_x = nullptr;
};

// ---- attention dispatch -----------------------------------------------------------------------------------------
// Which kernel runs each attention block.  The layer loops and sealdec_debug_attention both go through these, so the
// debug entry point exercises the model's own choice; each launcher enqueues one kernel and returns its kPath* bit.

// dec_self_attn_query_kernel (the beams of a query together, distinct ancestors staged once): not at the compact first
// step, where a row stands for all beams, nor for ragged re-scoring groups, and only while the staged K / V of P = pos + 1
// positions fit in 112 KB of shared memory.  It sums a split-K qkv itself.
bool use_self_attn_query(int pos, int B, bool compact, bool ragged) {
    static const bool sa_query = [] { const char* e = std::getenv("SEALB200_SELF_ATTN_QUERY"); return !e || std::atoi(e) != 0; }();
    const size_t saq_smem = self_attn_query_smem(pos + 1, B);
    return sa_query && !compact && !ragged && pos >= 1 && B >= 2 && B <= 32 && pos + 1 <= 128 && saq_smem <= 112 * 1024;
}

// cross_attn_small_kernel for sources of at most kXKeys positions; it sums a split-K cq itself
bool use_cross_attn_small(int64_t S) { return S <= kXKeys; }

// Decoder self-attention of one step and layer: qkv [R][3d] of the step's rows (at the compact first step row r stands
// for cache rows r * row_mul .. r * row_mul + row_mul - 1), the layer's cache kc / vc [T][Rc][d] and ancestry anc [Rc][T].
struct SelfAttnArgs {
    int64_t Q, R, Rc; int B, d, heads, pos, T, row_mul;
    const float* qkv; float* kc; float* vc; const int32_t* anc; float* out;
};

template <class SO>
uint32_t launch_bart_self_attn(cudaStream_t s, const SelfAttnArgs& a, bool use_saq, const SO& so, const SplitSrc& qkv_src) {
    const unsigned sa_threads = 32 * std::min(a.heads, 16);
    if (use_saq) {
        static size_t saq_set = 0;                     // per instantiation
        const size_t saq_smem = self_attn_query_smem(a.pos + 1, a.B);
        if (saq_smem > saq_set) { CUDA_CHECK(cudaFuncSetAttribute(dec_self_attn_query_kernel<SO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024)); saq_set = 112 * 1024; }
        launch_k(dec_self_attn_query_kernel<SO>, dim3((unsigned)a.Q, a.heads), 32 * a.B, saq_smem, s, a.Rc, a.B, a.d, a.pos, a.T, a.qkv, a.kc, a.vc, a.anc,
                 a.out, so, qkv_src);
        return kPathSelfQuery;
    }
    if (a.pos + 1 <= 12) {
        launch_k(dec_self_attn_kernel<3, SO>, (unsigned)a.R, sa_threads, 0, s, a.Rc, a.d, a.heads, a.pos, a.T, a.qkv, a.kc, a.vc, a.anc, a.out, so, a.row_mul, a.row_mul);
        return kPathSelfRounds3;
    }
    if (a.pos + 1 <= 32) {
        launch_k(dec_self_attn_kernel<8, SO>, (unsigned)a.R, sa_threads, 0, s, a.Rc, a.d, a.heads, a.pos, a.T, a.qkv, a.kc, a.vc, a.anc, a.out, so, a.row_mul, a.row_mul);
        return kPathSelfRounds8;
    }
    launch_k(dec_self_attn_long_kernel<SO>, (unsigned)a.R, sa_threads, 0, s, a.Rc, a.d, a.heads, a.pos, a.T, a.qkv, a.kc, a.vc, a.anc, a.out, so);
    return kPathSelfLong;
}

template <class SO>
uint32_t launch_t5_dec_self_attn(cudaStream_t s, const SelfAttnArgs& a, const RelBias& rb, const SO& so) {
    launch_k(t5_dec_self_attn_kernel<SO>, (unsigned)a.R, 32 * std::min(a.heads, 16), 0, s, a.Rc, a.d, a.heads, a.pos, a.T, a.qkv, a.kc, a.vc,
             a.anc, rb, so, a.row_mul, a.row_mul);
    return kPathT5DecAttn;
}

// Cross-attention of `groups` row groups (beams rows each, or ragged grp_query / grp_start) over ckv [Q*S or packed][2d].
struct CrossAttnArgs {
    int64_t groups; int d, heads, beams, S;
    const float* q; const float* ckv; const int32_t* mask; const int32_t* grp_query; const int32_t* grp_start; float* out;
    const int32_t* src_off;
};

template <class SO>
uint32_t launch_cross_attn(cudaStream_t s, const CrossAttnArgs& a, const SO& so, const SplitSrc& q_src) {
    if (use_cross_attn_small(a.S)) {
        launch_k(cross_attn_small_kernel<SO>, dim3((unsigned)a.groups, a.heads), 128, 0, s, a.groups, a.d, a.heads, a.beams, a.S, a.q,
                 a.ckv, a.mask, a.grp_query, a.grp_start, a.out, so, a.src_off, q_src);
        return kPathCrossSmall;
    }
    launch_k(cross_attn_kernel<SO>, dim3((unsigned)a.groups, a.heads), kGAttnWarps * 32, 0, s, a.groups, a.d, a.heads, a.beams, a.S, a.q,
             a.ckv, a.mask, a.grp_query, a.grp_start, a.out, so, a.src_off);
    return kPathCrossGrouped;
}

// Encoder self-attention of Q sources of S positions: qkv [Q*S or packed][3d]; rb != nullptr: T5 (relative position bias,
// unscaled scores, no fp32 copy of the output), else the BART kernel.  Returns kPathT5EncAttn or 0 (the BART encoder's
// attention has no bit of its own: kPathEncPacked / kPathEncUnpacked name its two forms).
template <class SO>
uint32_t launch_enc_self_attn(cudaStream_t s, int64_t Q, int d, int heads, int S, const float* qkv, const int32_t* mask,
                              const RelBias* rb, float* out, const SO& so, const int32_t* src_off) {
    if (rb) {
        launch_k(t5_enc_self_attn_kernel<kGAttnWarps, kGAttnPasses, SO>, dim3((unsigned)Q, heads), kGAttnWarps * 32, 0, s, Q, d, S, qkv, mask, *rb,
                 so, src_off);
        return kPathT5EncAttn;
    }
    launch_k(enc_self_attn_kernel<SO>, dim3((unsigned)Q, heads), kGAttnWarps * 32, 0, s, Q, d, heads, S, qkv, mask, out, so, src_off);
    return 0;
}

// The cross-attention block of decoder layer l: cq = x Wq, attention over the layer's encoder K / V into attn, then
// co into tmp.  defer_rows: how many rows the norm after the block accepts with co's split-K slices unsummed.
void cross_attention(Ctx& cx, const Dims& D, const DecStep& S, int l, int64_t defer_rows) {
    sealbart* m = cx.m;
    const int d = D.d, heads = m->cfg.heads;
    DecLayerW& L = m->dec[l];
    cx.defer_rows = use_cross_attn_small(D.S) ? INT64_MAX : 0;
    gemm(cx, S.R, d, d, S.x, d, L.cq, S.cq, d, kActNone);
    cx.defer_rows = 0;
    const SplitSrc cq_src = cx.pending;
    cx.pending = SplitSrc{};
    const CrossAttnArgs a{D.grp_start ? D.G : D.Q, d, heads, S.compact ? 1 : D.B, (int)D.S, S.cq.x,
                          m->ckv.as<float>() + (size_t)l * S.Tk * 2 * d + S.ckv_q0, S.m32, D.grp_query, D.grp_start, S.attn.x, S.soff_x};
    with_split(m, S.attn, [&](auto so) { m->last_paths |= launch_cross_attn(cx.s, a, so, cq_src); });
    m->launches++;
    cx.defer_rows = defer_rows;
    gemm(cx, S.R, d, d, S.attn, d, L.co, S.tmp, d, kActNone);
    cx.defer_rows = 0;
}

void t5_encoder_layers(Ctx& cx, const Dims& D, int64_t Te, const Acts& A, const int32_t* tok, const int32_t* m32, const int32_t* soff) {
    sealbart* m = cx.m;
    const int d = D.d;
    const RelBias rb{m->t5_rel_enc, m->t5_bkt_enc, kT5MaxSource - 1, m->cfg.heads};
    const int n = (int)m->enc.size();
    t5_rms(cx, Te, d, tok, 1, A.x, nullptr, m->enc[0].ln_attn.g, 1.f);
    for (int i = 0; i < n; ++i) {
        EncLayerW& L = m->enc[i];
        gemm(cx, Te, 3 * d, d, A.x, d, L.qkv, A.qkv, 3 * d, kActNone);
        with_split(m, A.attn, [&](auto so) {
            m->last_paths |= launch_enc_self_attn(cx.s, D.Q, d, m->cfg.heads, (int)D.S, A.qkv.x, m32, &rb, A.attn.x, so, soff);
        });
        m->launches++;
        cx.defer_rows = INT64_MAX;
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone);
        cx.defer_rows = 0;
        t5_rms(cx, Te, d, nullptr, 0, A.x, A.tmp.x, L.ln_final.g, 1.f);
        t5_ffn(cx, Te, d, D.f, A.x, L.fc1, L.fc2, A.ffn, A.ffn2, A.tmp);
        t5_rms(cx, Te, d, nullptr, 0, A.x, A.tmp.x, i + 1 < n ? m->enc[i + 1].ln_attn.g : m->enc_ln_emb.g, 1.f);
    }
}

// The T5 decoder layers: the self-attention adds the relative position bias, the cross-attention runs the BART kernels
// on the query projection pre-multiplied by 8 (their 0.125 undoes it exactly).
void t5_decoder_layers(Ctx& cx, const Dims& D, const DecStep& S) {
    sealbart* m = cx.m;
    const int d = D.d, heads = m->cfg.heads;
    const RelBias rb{m->t5_rel_dec, m->t5_bkt_dec, kMaxLen - 1, heads};
    const int n = (int)m->dec.size();
    const float out_scale = m->t5.scale_decoder_outputs ? 1.0f / sqrtf((float)d) : 1.0f;
    t5_rms(cx, S.R, d, S.tokens + S.pos, (int64_t)(D.T * S.row_mul), S.x, nullptr, m->dec[0].ln_self.g, 1.f);
    for (int l = 0; l < n; ++l) {
        DecLayerW& L = m->dec[l];
        float* kc = m->kc.as<float>() + (size_t)l * D.T * S.Rc * d + D.r0 * d;
        float* vc = m->vc.as<float>() + (size_t)l * D.T * S.Rc * d + D.r0 * d;
        gemm(cx, S.R, 3 * d, d, S.x, d, L.qkv, S.qkv, 3 * d, kActNone);
        const SelfAttnArgs a{D.Q, S.R, S.Rc, D.B, d, heads, S.pos, D.T, S.row_mul, S.qkv.x, kc, vc, S.anc, S.attn.x};
        with_split(m, S.attn, [&](auto so) { m->last_paths |= launch_t5_dec_self_attn(cx.s, a, rb, so); });
        m->launches++;
        cx.defer_rows = INT64_MAX;
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone);
        cx.defer_rows = 0;
        t5_rms(cx, S.R, d, nullptr, 0, S.x, S.tmp.x, L.ln_cross.g, 1.f);
        cross_attention(cx, D, S, l, INT64_MAX);
        t5_rms(cx, S.R, d, nullptr, 0, S.x, S.tmp.x, L.ln_final.g, 1.f);
        t5_ffn(cx, S.R, d, D.f, S.x, L.fc1, L.fc2, S.ffn, S.ffn2, S.tmp);
        t5_rms(cx, S.R, d, nullptr, 0, S.x, S.tmp.x, l + 1 < n ? m->dec[l + 1].ln_self.g : m->dec_ln_emb.g, l + 1 < n ? 1.f : out_scale);
    }
}

void bart_encoder_layers(Ctx& cx, const Dims& D, int64_t Te, const Acts& A, const int32_t* tok, const int32_t* pos, const int32_t* m32,
                         const int32_t* soff) {
    sealbart* m = cx.m;
    const int d = D.d, heads = m->cfg.heads;
    const float scale = m->cfg.scale_embedding ? sqrtf((float)d) : 1.0f;
    with_split(m, A.x, [&](auto so) {
        using SO = decltype(so);
        embed_ln_kernel<SO><<<(unsigned)((Te + 3) / 4), 128, 0, cx.s>>>(Te, d, tok, 1, pos, 0, embed_table<SO>(m), scale, m->enc_pos,
                                                                        m->enc_ln_emb.g, m->enc_ln_emb.b, A.x.x, so);
    });
    CUDA_CHECK(cudaGetLastError()); m->launches++;
    for (auto& L : m->enc) {
        gemm(cx, Te, 3 * d, d, A.x, d, L.qkv, A.qkv, 3 * d, kActNone);
        with_split(m, A.attn, [&](auto so) { launch_enc_self_attn(cx.s, D.Q, d, heads, (int)D.S, A.qkv.x, m32, nullptr, A.attn.x, so, soff); });
        m->launches++;
        cx.defer_rows = kAddLnRowMax;
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone);
        cx.defer_rows = 0;
        add_ln(cx, Te, d, A.x.x, A.tmp.x, L.ln_attn, A.x);
        gemm(cx, Te, D.f, d, A.x, d, L.fc1, A.ffn, D.f, kActGelu);
        cx.defer_rows = kAddLnRowMax;
        gemm(cx, Te, d, D.f, A.ffn, D.f, L.fc2, A.tmp, d, kActNone);
        cx.defer_rows = 0;
        add_ln(cx, Te, d, A.x.x, A.tmp.x, L.ln_final, A.x);
    }
}

// The BART decoder self-attention of layer l (BART and the pre-LayerNorm variants): qkv = x Wqkv, then attention over
// the layer's KV cache (beam ancestry) into attn; the current k / v are persisted to the cache.
void bart_self_attention(Ctx& cx, const Dims& D, const DecStep& S, int l) {
    sealbart* m = cx.m;
    const int d = D.d, heads = m->cfg.heads, pos = S.pos;
    DecLayerW& L = m->dec[l];
    float* kc = m->kc.as<float>() + (size_t)l * D.T * S.Rc * d + D.r0 * d;
    float* vc = m->vc.as<float>() + (size_t)l * D.T * S.Rc * d + D.r0 * d;
    const bool use_saq = use_self_attn_query(pos, D.B, S.compact, D.grp_start != nullptr);
    cx.defer_rows = use_saq ? INT64_MAX : 0;
    gemm(cx, S.R, 3 * d, d, S.x, d, L.qkv, S.qkv, 3 * d, kActNone);
    cx.defer_rows = 0;
    const SplitSrc qkv_src = cx.pending;
    cx.pending = SplitSrc{};
    const SelfAttnArgs a{D.Q, S.R, S.Rc, D.B, d, heads, pos, D.T, S.row_mul, S.qkv.x, kc, vc, S.anc, S.attn.x};
    with_split(m, S.attn, [&](auto so) { m->last_paths |= launch_bart_self_attn(cx.s, a, use_saq, so, qkv_src); });
    m->launches++;
}

void bart_decoder_layers(Ctx& cx, const Dims& D, const DecStep& S) {
    sealbart* m = cx.m;
    const int d = D.d, pos = S.pos;
    const float scale = m->cfg.scale_embedding ? sqrtf((float)d) : 1.0f;
    with_split(m, S.x, [&](auto so) {
        using SO = decltype(so);
        launch_k(embed_ln_kernel<SO>, (unsigned)((S.R + 3) / 4), 128, 0, cx.s, S.R, d, S.tokens + pos, (int64_t)(D.T * S.row_mul), (const int32_t*)nullptr, pos,
                 embed_table<SO>(m), scale, (const float*)m->dec_pos, (const float*)m->dec_ln_emb.g, (const float*)m->dec_ln_emb.b, S.x.x, so);
    });
    m->launches++;
    for (int l = 0; l < m->cfg.decoder_layers; ++l) {
        DecLayerW& L = m->dec[l];
        bart_self_attention(cx, D, S, l);
        cx.defer_rows = kAddLnRowMax;
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone);
        cx.defer_rows = 0;
        add_ln(cx, S.R, d, S.x.x, S.tmp.x, L.ln_self, S.x);
        cross_attention(cx, D, S, l, kAddLnRowMax);
        add_ln(cx, S.R, d, S.x.x, S.tmp.x, L.ln_cross, S.x);
        gemm(cx, S.R, D.f, d, S.x, d, L.fc1, S.ffn, D.f, kActGelu);
        cx.defer_rows = kAddLnRowMax;
        gemm(cx, S.R, d, D.f, S.ffn, D.f, L.fc2, S.tmp, d, kActNone);
        cx.defer_rows = 0;
        add_ln(cx, S.R, d, S.x.x, S.tmp.x, L.ln_final, S.x);
    }
}

// ---- pre-LayerNorm BART family (Pegasus, mBART) ---------------------------------------------------------------
// The T5 loops' structure with BART's weights and kernels: x (fp32, the residual stream) += sublayer(LN(x)).  The
// plain half of the Act x holds the residual, its split half the normed operand of the next GEMM: every preln_norm
// launch adds the previous sublayer's output (or gathers the embedding), stores the residual and writes LN(x) with the
// next sublayer's norm -- after the last layer the stack's final layer_norm.
PreLnEmbed preln_embed(const sealbart* m, const int32_t* tok, int64_t tok_stride, const int32_t* pos, int pos_const,
                       const float* table, const LNp& ln_emb) {
    PreLnEmbed em;
    em.tok = tok; em.tok_stride = tok_stride; em.pos = pos; em.pos_const = pos_const;
    em.pos_offset = m->variant.position_offset; em.pos_rows = m->cfg.max_positions + m->variant.position_offset;
    em.embed = m->shared; em.scale = m->cfg.scale_embedding ? sqrtf((float)m->cfg.d_model) : 1.0f; em.pos_table = table;
    em.ln_g = ln_emb.g; em.ln_b = ln_emb.b;
    return em;
}

void preln_norm(Ctx& cx, int64_t rows, int d, const PreLnEmbed& em, const Act& x, const float* b, const LNp& ln) {
    const SplitSrc ps = cx.pending;
    cx.pending = SplitSrc{};
    with_split(cx.m, x, [&](auto so) {
        using SO = decltype(so);
        PreLnEmbedT<EmbT<SO>> e;                           // em with the table in the mode's element type
        e.tok = em.tok; e.tok_stride = em.tok_stride; e.pos = em.pos; e.pos_const = em.pos_const; e.pos_offset = em.pos_offset;
        e.pos_rows = em.pos_rows; e.embed = em.tok ? embed_table<SO>(cx.m) : nullptr; e.scale = em.scale; e.pos_table = em.pos_table;
        e.ln_g = em.ln_g; e.ln_b = em.ln_b;
        launch_k(preln_row_kernel<SO>, (unsigned)rows, 128, 0, cx.s, rows, d, e, x.x, b, ps, (const float*)ln.g, (const float*)ln.b, so);
    });
    cx.m->launches++;
    cx.m->last_paths |= kPathPreLn | (em.tok && em.ln_g ? kPathPreLnEmbedLn : 0u);
}

// fc1 with the variant's activation epilogue, then fc2 into tmp (split-K slices left to the next preln_norm)
void preln_ffn(Ctx& cx, int64_t rows, const Dims& D, const Act& x, Lin& fc1, Lin& fc2, const Act& ffn, const Act& tmp) {
    const int act = cx.m->variant.activation == SEALBART_ACT_RELU ? kActRelu : kActGelu;
    gemm(cx, rows, D.f, D.d, x, D.d, fc1, ffn, D.f, act);
    cx.defer_rows = INT64_MAX;
    gemm(cx, rows, D.d, D.f, ffn, D.f, fc2, tmp, D.d, kActNone);
    cx.defer_rows = 0;
}

void preln_encoder_layers(Ctx& cx, const Dims& D, int64_t Te, const Acts& A, const int32_t* tok, const int32_t* pos,
                          const int32_t* m32, const int32_t* soff) {
    sealbart* m = cx.m;
    const int d = D.d, heads = m->cfg.heads;
    const int n = (int)m->enc.size();
    preln_norm(cx, Te, d, preln_embed(m, tok, 1, pos, 0, m->enc_pos, m->enc_ln_emb), A.x, nullptr, m->enc[0].ln_attn);
    for (int i = 0; i < n; ++i) {
        EncLayerW& L = m->enc[i];
        gemm(cx, Te, 3 * d, d, A.x, d, L.qkv, A.qkv, 3 * d, kActNone);
        with_split(m, A.attn, [&](auto so) { launch_enc_self_attn(cx.s, D.Q, d, heads, (int)D.S, A.qkv.x, m32, nullptr, A.attn.x, so, soff); });
        m->launches++;
        cx.defer_rows = INT64_MAX;
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone);
        cx.defer_rows = 0;
        preln_norm(cx, Te, d, PreLnEmbed{}, A.x, A.tmp.x, L.ln_final);
        preln_ffn(cx, Te, D, A.x, L.fc1, L.fc2, A.ffn, A.tmp);
        preln_norm(cx, Te, d, PreLnEmbed{}, A.x, A.tmp.x, i + 1 < n ? m->enc[i + 1].ln_attn : m->enc_ln_out);
    }
}

void preln_decoder_layers(Ctx& cx, const Dims& D, const DecStep& S) {
    sealbart* m = cx.m;
    const int d = D.d;
    const int n = (int)m->dec.size();
    preln_norm(cx, S.R, d, preln_embed(m, S.tokens + S.pos, (int64_t)(D.T * S.row_mul), nullptr, S.pos, m->dec_pos, m->dec_ln_emb),
               S.x, nullptr, m->dec[0].ln_self);
    for (int l = 0; l < n; ++l) {
        DecLayerW& L = m->dec[l];
        bart_self_attention(cx, D, S, l);
        cx.defer_rows = INT64_MAX;
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone);
        cx.defer_rows = 0;
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, L.ln_cross);
        cross_attention(cx, D, S, l, INT64_MAX);
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, L.ln_final);
        preln_ffn(cx, S.R, D, S.x, L.fc1, L.fc2, S.ffn, S.tmp);
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, l + 1 < n ? m->dec[l + 1].ln_self : m->dec_ln_out);
    }
}

// src_tokens_hint: >= 0 the caller's count of real source tokens (right-padded masks): no host synchronisation, the
// kernel that derives the offsets checks it and raises err_d[2] on a mismatch; -1 unknown: one 16-byte read-back;
// -2 do not pack (padded rows are computed; also no synchronisation).
void encoder_forward(Ctx& cx, const Dims& D, const int64_t* ids_d, const int64_t* mask_d, int64_t src_tokens_hint = -1,
                     int32_t* hint_err = nullptr) {
    sealbart* m = cx.m;
    const int64_t Tk = D.Q * D.S;
    const int d = D.d;
    int32_t* tok = m->enc_tok.as<int32_t>(); int32_t* pos = tok + Tk; int32_t* m32 = m->enc_mask.as<int32_t>();
    // Padding is not computed: with right-padded sources (the only kind SEAL produces) the encoder and the
    // cross-attention K/V projections run on the sum of the real lengths P instead of Q * S_max rows
    // (29 % fewer at S ~ U[12, 28]); query q's states are rows src_off[q] .. src_off[q+1] everywhere downstream.
    static const bool pack_enabled = [] { const char* e = std::getenv("SEALB200_PACK_ENCODER"); return !e || std::atoi(e) != 0; }();
    int32_t* src_off = m->src_off.as<int32_t>();
    int64_t* info_d = reinterpret_cast<int64_t*>(reinterpret_cast<char*>(m->src_off.p) + ((D.Q + 1) * 4 + 15) / 16 * 16);
    int64_t rows_enc = Tk;
    m->enc_packed = false;
    if (pack_enabled && src_tokens_hint != -2) {
        pack_lengths_kernel<<<1, 1024, 0, cx.s>>>(D.Q, (int)D.S, mask_d, src_off, info_d, src_tokens_hint, hint_err);
        CUDA_CHECK(cudaGetLastError()); m->launches++;
        if (src_tokens_hint > 0) { m->enc_packed = true; rows_enc = src_tokens_hint; }
        else {
            int64_t info[2] = {0, 1};
            CUDA_CHECK(cudaMemcpyAsync(info, info_d, 16, cudaMemcpyDeviceToHost, cx.s));
            CUDA_CHECK(cudaStreamSynchronize(cx.s));
            if (info[1] == 0 && info[0] > 0) { m->enc_packed = true; rows_enc = info[0]; }
        }
    }
    const int32_t* soff = m->enc_packed ? src_off : nullptr;
    if (m->enc_packed) prep_enc_packed_kernel<<<(unsigned)((Tk + 255) / 256), 256, 0, cx.s>>>(Tk, (int)D.S, ids_d, src_off, tok, pos);
    else prep_enc_kernel<<<(unsigned)((Tk + 255) / 256), 256, 0, cx.s>>>(Tk, (int)D.S, ids_d, mask_d, tok, m32, pos);
    CUDA_CHECK(cudaGetLastError()); m->launches++;
    m->last_paths |= m->enc_packed ? kPathEncPacked : kPathEncUnpacked;
    const int64_t Te = rows_enc;                    // encoder rows actually computed
    const int gm = m->cfg.gemm_mode;
    Acts A;
    A.x = act_view(gm, m->ex.as<float>(), m->ex_hi, m->ex_lo);
    A.qkv = Act{m->eqkv.as<float>()};
    A.attn = act_view(gm, nullptr, m->eattn_hi, m->eattn_lo);
    A.tmp = Act{m->etmp.as<float>()};
    A.ffn = act_view(gm, nullptr, m->effn_hi, m->effn_lo);
    A.ffn2 = m->effn2.as<float>();
    if (m->arch == 1) t5_encoder_layers(cx, D, Te, A, tok, m32, soff);
    else if (m->arch == 2) preln_encoder_layers(cx, D, Te, A, tok, pos, m32, soff);
    else bart_encoder_layers(cx, D, Te, A, tok, pos, m32, soff);
    // per-query cross-attention K/V of every decoder layer, once, from the encoder's output (T5 and the pre-LayerNorm
    // variants: its final layer norm);
    // the reference recomputes nothing either: HF caches them after the first step
    for (int l = 0; l < m->cfg.decoder_layers; ++l)
        gemm(cx, Te, 2 * d, d, A.x, d, m->dec[l].ckv, Act{m->ckv.as<float>() + (size_t)l * Tk * 2 * d}, 2 * d, kActNone);
}

// one decoder step for all R rows: token at position pos = cur_len-1 -> logits [R][ld]
// `compact` (first step of a generate only): every beam of a query is the same row there (same start token, same
// source), so the step runs on one row per query -- Q rows instead of Q*B -- and the select kernel reads that
// row's logits for all of the query's beams (StepCfg::logits_shared); the k / v of position 0 are written to the
// cache entries of all B beams.  1/T of the decoder + lm_head work disappears (~8 % of a 9-step generate).
void decoder_step(Ctx& cx, const Dims& D, const int32_t* tokens, int cur_len, const int32_t* anc, bool want_logits,
                  cudaEvent_t ev_layers_done, bool compact = false, const HeadEpi& head = HeadEpi{}) {
    sealbart* m = cx.m;
    if (compact && (cur_len != 1 || D.grp_start || D.Qb)) throw ApiError(SEALFM_EINVAL, "internal: compact step only at position 0 of a generate");
    const int d = D.d, gm = m->cfg.gemm_mode;
    DecStep S;
    S.x = act_view(gm, m->dx.as<float>(), m->dx_hi, m->dx_lo, D.r0 * d);
    S.qkv = Act{m->dqkv.as<float>() + D.r0 * 3 * d};
    S.attn = act_view(gm, nullptr, m->dattn_hi, m->dattn_lo, D.r0 * d);
    S.tmp = Act{m->dtmp.as<float>() + D.r0 * d};
    S.cq = Act{m->dcq.as<float>() + D.r0 * d};
    S.ffn = act_view(gm, nullptr, m->dffn_hi, m->dffn_lo, D.r0 * D.f);
    S.ffn2 = m->dffn2.as<float>() ? m->dffn2.as<float>() + D.r0 * 2 * D.f : nullptr;
    S.R = compact ? D.Q : D.R; S.row_mul = compact ? D.B : 1; S.compact = compact;
    S.Rc = D.Rb ? D.Rb : D.R; S.pos = cur_len - 1; S.tokens = tokens; S.anc = anc;
    S.Tk = (D.Qb ? D.Qb : D.Q) * D.S; S.ckv_q0 = m->enc_packed ? 0 : D.q0 * D.S * 2 * d;
    S.m32 = m->enc_mask.as<int32_t>() + D.q0 * D.S; S.soff_x = m->enc_packed ? m->src_off.as<int32_t>() + D.q0 : nullptr;
    if (m->arch == 1) t5_decoder_layers(cx, D, S);
    else if (m->arch == 2) preln_decoder_layers(cx, D, S);
    else bart_decoder_layers(cx, D, S);
    if (ev_layers_done) CUDA_CHECK(cudaEventRecord(ev_layers_done, cx.s));
    cx.head = head;                 // only the lm_head may take the statistics epilogue
    if (want_logits) gemm(cx, S.R, D.V, d, S.x, d, m->head, Act{m->logits.as<float>() + D.r0 * D.ld}, D.ld, kActNone);
    cx.head = HeadEpi{};
}

void check_model(const sealbart* m) {
    if (!m) throw ApiError(SEALFM_EINVAL, "null model");
    if (!m->finalized) throw ApiError(SEALFM_EINVAL, "sealbart_finalize not called");
    CUDA_CHECK(cudaSetDevice(m->device));
}

Dims make_dims(const sealbart* m, int64_t Q, int64_t S, int B, int T) {
    Dims D;
    D.Q = Q; D.S = S; D.B = B; D.R = Q * B; D.T = T;
    D.d = m->cfg.d_model; D.f = m->cfg.ffn_dim; D.V = m->cfg.vocab_size;
    D.ld = (D.V + 3) / 4 * 4; D.W = (D.V + 31) / 32;
    return D;
}

cudaEvent_t new_event(sealbart* m) {
    cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); m->events.push_back(e); return e;
}


template <typename Fn> void for_each_lin(sealbart* m, Fn&& fn) {
    for (auto& L : m->enc) { fn(L.qkv); fn(L.o); fn(L.fc1); fn(L.fc2); }
    for (auto& L : m->dec) { fn(L.qkv); fn(L.o); fn(L.cq); fn(L.ckv); fn(L.co); fn(L.fc1); fn(L.fc2); }
    fn(m->head);
}

// 3xTF32 operand copies of l (gemm_mode 2): W = w_hi + w_lo, allocated here and owned by m (split_allocs)
void split_lin_tf32(sealbart* m, Lin& l) {
    const uint64_t n = (uint64_t)l.out * l.in;
    CUDA_CHECK(cudaMalloc(&l.w_hi, n * 4)); m->split_allocs.push_back(l.w_hi);
    CUDA_CHECK(cudaMalloc(&l.w_lo, n * 4)); m->split_allocs.push_back(l.w_lo);
    split_into(nullptr, l.w, l.w_hi, l.w_lo, n);
    m->weight_bytes += 2 * n * 4;
}

// 3xFP16 operand copies of l (gemm_mode 3 / 5): W * 2^s = w_h1 + w_h2 with max|W| * 2^s in [2^13, 2^14), w_unscale =
// 2^-s, allocated here and owned by m (split_allocs); a weight outside the halves' range raises m->err[1].  d_max: one
// device word of scratch.
void split_lin_half(sealbart* m, Lin& l, unsigned int* d_max) {
    const uint64_t n = (uint64_t)l.out * l.in;
    CUDA_CHECK(cudaMemset(d_max, 0, 4));
    absmax_kernel<<<sm_count() * 4, 256>>>((int64_t)n, l.w, d_max);
    unsigned int bits = 0; CUDA_CHECK(cudaMemcpy(&bits, d_max, 4, cudaMemcpyDeviceToHost));
    float mx; std::memcpy(&mx, &bits, 4);
    int sexp = 0;
    if (mx > 0.f) { int e; std::frexp(mx, &e); sexp = 14 - e; }
    l.w_unscale = std::ldexp(1.0f, -sexp);
    CUDA_CHECK(cudaMalloc(&l.w_h1, n * 2)); m->split_allocs.push_back(l.w_h1);
    CUDA_CHECK(cudaMalloc(&l.w_h2, n * 2)); m->split_allocs.push_back(l.w_h2);
    m->weight_bytes += 2 * n * 2;
    split_half_kernel<<<sm_count() * 8, 256>>>((int64_t)n, l.w, std::ldexp(1.0f, sexp), l.w_h1, l.w_h2, m->err.as<int>() + 1);
    CUDA_CHECK(cudaGetLastError());
    l.maps_ready = false;
}

// The GEMM operands of l in m's gemm_mode, derived from its loaded weights (gemm_mode 6: the bf16 matrix as loaded).
// d_max: one device word of scratch for 3xFP16, whose weight split reports into m->err.
void derive_lin(sealbart* m, Lin& l, unsigned int* d_max) {
    if (m->cfg.gemm_mode == kGemmTf32) split_lin_tf32(m, l);
    else if (is_3xfp16(m->cfg.gemm_mode)) split_lin_half(m, l, d_max);
}

// 3xTF32 operand copies of every weight matrix (gemm_mode 2; also the range-safe fallback of the 3xFP16 modes)
void ensure_tf32_splits(sealbart* m) {
    if (m->tf32_ready) return;
    CUDA_CHECK(cudaSetDevice(m->device));
    for_each_lin(m, [&](Lin& l) { split_lin_tf32(m, l); });
    CUDA_CHECK(cudaDeviceSynchronize());
    m->tf32_ready = true;
}

// HF's T5Attention._relative_position_bucket for one relative position (key - query), in its float32 arithmetic:
// log(rel.float() / max_exact) in fp32, divided by math.log(max_distance / max_exact) (a Python float, rounded to fp32
// where it meets the fp32 tensor), times (num_buckets - max_exact), truncated.  Computed here once per model: a device
// logf may round differently from torch at the bucket boundaries.
int32_t t5_bucket(int32_t rel, bool bidirectional, int num_buckets, int max_distance) {
    int32_t ret = 0;
    int nb = num_buckets;
    if (bidirectional) {
        nb /= 2;
        if (rel > 0) ret += nb;
        rel = rel < 0 ? -rel : rel;
    } else
        rel = rel < 0 ? -rel : 0;
    const int max_exact = nb / 2;
    if (rel < max_exact) return ret + rel;
    const float den = (float)std::log((double)max_distance / (double)max_exact);
    const float v = std::log((float)rel / (float)max_exact) / den * (float)(nb - max_exact);
    const int64_t large = std::min<int64_t>((int64_t)max_exact + (int64_t)v, nb - 1);
    return ret + (int32_t)large;
}

// [2 kT5MaxSource - 1] encoder buckets (entry i: distance i - (kT5MaxSource - 1), bidirectional) and [kMaxLen] decoder
// buckets (entry i: distance i - (kMaxLen - 1) <= 0, unidirectional), uploaded once
void t5_bucket_tables(sealbart* m) {
    const int nb = m->t5.relative_attention_num_buckets, md = m->t5.relative_attention_max_distance;
    std::vector<int32_t> enc(2 * kT5MaxSource - 1), dec(kMaxLen);
    for (int i = 0; i < (int)enc.size(); ++i) enc[i] = t5_bucket(i - (kT5MaxSource - 1), true, nb, md);
    for (int i = 0; i < (int)dec.size(); ++i) dec[i] = t5_bucket(i - (kMaxLen - 1), false, nb, md);
    m->t5_bkt_enc = reinterpret_cast<int32_t*>(dalloc(m, enc.size()));
    m->t5_bkt_dec = reinterpret_cast<int32_t*>(dalloc(m, dec.size()));
    CUDA_CHECK(cudaMemcpy(m->t5_bkt_enc, enc.data(), enc.size() * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(m->t5_bkt_dec, dec.data(), dec.size() * 4, cudaMemcpyHostToDevice));
}

// Returns the number of CUDA devices; none is an error.
int require_device() {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) { cudaGetLastError(); throw ApiError(SEALFM_ENODEVICE, "no CUDA device available"); }
    return count;
}

void check_gemm_mode(int mode) {
    if (mode != kGemmTf32 && !is_3xfp16(mode) && mode != kGemmBf16)
        throw ApiError(SEALFM_EINVAL, "gemm_mode must be 3 (3xFP16, one CTA per tile, default), 5 (3xFP16 on 2-CTA clusters), 2 (3xTF32) "
                                      "or 6 (3xBF16, bf16 weights)");
}

// fp32 -> bf16 bits, round to nearest even (the weights of a bf16 checkpoint pass through exactly); NaN stays NaN
uint16_t bf16_rne(float x) {
    uint32_t u; std::memcpy(&u, &x, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((u >> 16) | 0x40u);
    return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}
// n host values times scale (a power of two: exact) into device weights: rounded into bf16 (gemm_mode 6's matrices and
// embedding table) or copied as fp32
void upload(void* dst, bool bf16, const float* host, uint64_t n, float scale = 1.f) {
    if (bf16) {
        std::vector<uint16_t> b(n);
        for (uint64_t i = 0; i < n; ++i) b[i] = bf16_rne(host[i] * scale);
        CUDA_CHECK(cudaMemcpy(dst, b.data(), n * 2, cudaMemcpyHostToDevice));
    } else if (scale != 1.f) {
        std::vector<float> x(host, host + n);
        for (float& v : x) v *= scale;
        CUDA_CHECK(cudaMemcpy(dst, x.data(), n * 4, cudaMemcpyHostToDevice));
    } else
        CUDA_CHECK(cudaMemcpy(dst, host, n * 4, cudaMemcpyHostToDevice));
}

// sealt5_create's shape checks (before any allocation)
void check_t5_config(const sealt5_config_t* c) {
    if (c->d_kv != kHeadDim || c->num_heads * kHeadDim != c->d_model)
        throw ApiError(SEALFM_EINVAL, "T5: d_kv must be 64 and num_heads * 64 == d_model");
    // the two t5_rms_row_kernel instantiations: 128 threads x 2 float4 up to 1 024; x 8 float4 at the XL / XXL widths
    // 2 048, 3 072 and 4 096 (the widths in between have no checkpoint with 64-wide heads and are not tested)
    const bool narrow = c->d_model > 0 && c->d_model % 128 == 0 && c->d_model <= 1024;
    const bool wide = c->d_model > 0 && c->d_model % 1024 == 0 && c->d_model <= 4096;
    if (!narrow && !wide)
        throw ApiError(SEALFM_EINVAL, "T5: d_model must be a multiple of 128 up to 1 024, or a multiple of 1 024 up to 4 096");
    if (c->d_ff <= 0 || c->d_ff % 64) throw ApiError(SEALFM_EINVAL, "T5: d_ff must be a positive multiple of 64");
    if (c->vocab_size <= 0 || c->num_layers < 1 || c->num_decoder_layers < 1) throw ApiError(SEALFM_EINVAL, "T5: bad vocab_size / layer counts");
    if (c->ffn_kind != 0 && c->ffn_kind != 1) throw ApiError(SEALFM_EINVAL, "T5: ffn_kind must be 0 (relu) or 1 (gated-gelu)");
    if (c->relative_attention_num_buckets < 4 || c->relative_attention_num_buckets > 1024 ||
        c->relative_attention_max_distance <= c->relative_attention_num_buckets / 2)
        throw ApiError(SEALFM_EINVAL, "T5: relative_attention_num_buckets must be in [4, 1024] and relative_attention_max_distance > num_buckets / 2");
    if (!(c->layer_norm_epsilon >= 0.f) || !std::isfinite(c->layer_norm_epsilon)) throw ApiError(SEALFM_EINVAL, "T5: bad layer_norm_epsilon");
    check_gemm_mode(c->gemm_mode);
}

}  // namespace

extern "C" {

int sealt5_relative_buckets(int32_t num_buckets, int32_t max_distance, int32_t bidirectional, int32_t n, int32_t* out) {
    return guarded([&] {
        if (!out || n < 1 || num_buckets < 4 || num_buckets > 1024 || max_distance <= num_buckets / 2)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (bidirectional) for (int i = 0; i < 2 * n - 1; ++i) out[i] = t5_bucket(i - (n - 1), true, num_buckets, max_distance);
        else for (int i = 0; i < n; ++i) out[i] = t5_bucket(-i, false, num_buckets, max_distance);
    });
}

int sealt5_create(const sealt5_config_t* cfg, int device, sealbart_t** out) {
    return guarded([&] {
        if (!cfg || !out) throw ApiError(SEALFM_EINVAL, "null argument");
        check_t5_config(cfg);
        if (device < 0 || device >= require_device()) throw ApiError(SEALFM_EINVAL, "bad device id");
        CUDA_CHECK(cudaSetDevice(device));
        std::unique_ptr<sealbart> m(new sealbart());
        m->arch = 1; m->t5 = *cfg; m->device = device;
        m->cfg = sealbart_config_t{cfg->vocab_size, cfg->d_model, cfg->num_layers, cfg->num_decoder_layers, cfg->num_heads, cfg->d_ff,
                                   kT5MaxSource, 0, cfg->gemm_mode};
        struct Guard { sealbart* m; ~Guard() { if (m) sealbart_free(m); } } guard{m.get()};
        build_slots_t5(m.get());
        t5_bucket_tables(m.get());
        guard.m = nullptr;
        *out = m.release();
    });
}

}  // extern "C"

namespace {

// sealbart_create and sealbart_create_ex: var == nullptr is bart-large's post-LayerNorm layer
void create_bart(const sealbart_config_t* cfg, const sealbart_variant_t* var, int device, sealbart_t** out) {
    if (!cfg || !out) throw ApiError(SEALFM_EINVAL, "null argument");
    if (cfg->d_model % 128 || cfg->d_model > 1024 || cfg->heads * kHeadDim != cfg->d_model)
        throw ApiError(SEALFM_EINVAL, "d_model must be a multiple of 128, <= 1024, with 64-wide heads");
    if (cfg->ffn_dim % 64 || cfg->vocab_size <= 0) throw ApiError(SEALFM_EINVAL, "bad ffn_dim / vocab_size");
    if (var && cfg->max_positions < 1) throw ApiError(SEALFM_EINVAL, "max_positions must be >= 1");
    check_gemm_mode(cfg->gemm_mode);
    if (device < 0 || device >= require_device()) throw ApiError(SEALFM_EINVAL, "bad device id");
    CUDA_CHECK(cudaSetDevice(device));
    std::unique_ptr<sealbart> m(new sealbart());
    m->cfg = *cfg; m->device = device;
    if (var) { m->arch = 2; m->variant = *var; }
    struct Guard { sealbart* m; ~Guard() { if (m) sealbart_free(m); } } guard{m.get()};
    build_slots(m.get());
    guard.m = nullptr;
    *out = m.release();
}

}  // namespace

extern "C" {

int sealbart_create(const sealbart_config_t* cfg, int device, sealbart_t** out) {
    return guarded([&] { create_bart(cfg, nullptr, device, out); });
}

int sealbart_create_ex(const sealbart_config_t* cfg, const sealbart_variant_t* variant, int device, sealbart_t** out) {
    return guarded([&] {
        if (!cfg || !variant || !out) throw ApiError(SEALFM_EINVAL, "null argument");
        const sealbart_variant_t& v = *variant;
        if (v.activation != SEALBART_ACT_GELU && v.activation != SEALBART_ACT_RELU)
            throw ApiError(SEALFM_EINVAL, "activation must be SEALBART_ACT_GELU or SEALBART_ACT_RELU");
        if (!v.pre_layer_norm) {                               // the post-LayerNorm layer exists in bart-large's form only
            if (v.position_offset != 2 || v.layernorm_embedding != 1 || v.activation != SEALBART_ACT_GELU)
                throw ApiError(SEALFM_EINVAL, "post-LayerNorm variant: only bart-large's (position_offset 2, layernorm_embedding, gelu)");
            create_bart(cfg, nullptr, device, out);
            return;
        }
        if (v.pre_layer_norm != 1) throw ApiError(SEALFM_EINVAL, "pre_layer_norm must be 0 or 1");
        if (v.position_offset != 0 && v.position_offset != 2) throw ApiError(SEALFM_EINVAL, "position_offset must be 0 or 2");
        if (v.layernorm_embedding != 0 && v.layernorm_embedding != 1) throw ApiError(SEALFM_EINVAL, "layernorm_embedding must be 0 or 1");
        create_bart(cfg, &v, device, out);
    });
}

void sealbart_free(sealbart_t* m) {
    if (!m) return;
    cudaSetDevice(m->device);
    if (m->lm_head_given) cudaFree(m->lm_head_bf ? (void*)m->lm_head_bf : (void*)m->lm_head);
    if (m->slice_fork) cudaEventDestroy(m->slice_fork);
    if (m->slice_join) cudaEventDestroy(m->slice_join);
    if (m->slice_stream) cudaStreamDestroy(m->slice_stream);
    for (auto e : m->events) cudaEventDestroy(e);
    for (auto& g : m->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (m->stream) cudaStreamDestroy(m->stream);
    delete m;                         // frees the weights and the workspace (Buf)
}

int sealbart_set_tensor(sealbart_t* m, const char* key, const float* host, uint64_t numel) {
    return guarded([&] {
        if (!m || !key || !host) throw ApiError(SEALFM_EINVAL, "null argument");
        CUDA_CHECK(cudaSetDevice(m->device));
        std::string k(key);
        if (k == "lm_head.weight") {
            const uint64_t want = (uint64_t)m->cfg.vocab_size * m->cfg.d_model;
            if (numel != want) throw ApiError(SEALFM_EINVAL, "lm_head.weight: wrong size");
            if (bf16_weights(m)) {
                if (!m->lm_head_given) { CUDA_CHECK(cudaMalloc(&m->lm_head_bf, want * 2)); m->lm_head_given = true; m->weight_bytes += want * 2; }
                upload(m->lm_head_bf, true, host, want);
                return;
            }
            if (!m->lm_head_given) { CUDA_CHECK(cudaMalloc(&m->lm_head, want * 4)); m->lm_head_given = true; m->weight_bytes += want * 4; }
            upload(m->lm_head, false, host, want);
            return;
        }
        if (m->arch != 1 && (k == "model.encoder.embed_tokens.weight" || k == "model.decoder.embed_tokens.weight")) k = "model.shared.weight";
        if (m->arch == 1 && (k == "encoder.embed_tokens.weight" || k == "decoder.embed_tokens.weight")) k = "shared.weight";
        auto it = m->slots.find(k);
        if (it == m->slots.end()) throw ApiError(SEALFM_EINVAL, "unknown state_dict key: " + k);
        if (it->second.numel != numel) throw ApiError(SEALFM_EINVAL, "wrong element count for " + k);
        static const std::string kCrossQ = ".layer.1.EncDecAttention.q.weight";
        const bool cross_q = m->arch == 1 && k.size() > kCrossQ.size() && k.compare(k.size() - kCrossQ.size(), kCrossQ.size(), kCrossQ) == 0;
        // T5 does not scale attention scores; the cross-attention kernels multiply by 0.125, so q is stored times 8
        // (a power of two: (8q . k) * 0.125 == q . k exactly)
        upload(it->second.dst, it->second.bf16, host, numel, cross_q ? 8.f : 1.f);
        m->loaded.insert(k);
        m->finalized = false;
    });
}

int sealbart_finalize(sealbart_t* m) {
    return guarded([&] {
        if (!m) throw ApiError(SEALFM_EINVAL, "null model");
        for (auto& kv : m->slots)
            if (!m->loaded.count(kv.first)) throw ApiError(SEALFM_EINVAL, "state_dict tensor missing: " + kv.first);
        if (!m->lm_head_given) { m->lm_head = m->shared; m->lm_head_bf = nullptr; }   // tied (seal/utils.py:48-49; T5: tie_word_embeddings)
        m->head.w = m->lm_head; m->head.b = m->final_bias; m->head.out = m->cfg.vocab_size; m->head.in = m->cfg.d_model;
        m->head.w_bf = m->lm_head_given ? m->lm_head_bf : m->shared_bf;
        CUDA_CHECK(cudaSetDevice(m->device));
        for (void* p : m->split_allocs) cudaFree(p);
        m->split_allocs.clear();
        m->tf32_ready = false;
        for_each_lin(m, [](Lin& l) { l.maps_ready = false; l.maps2_ready = false; });
        unsigned int* d_max = nullptr;
        if (is_3xfp16(m->cfg.gemm_mode)) { CUDA_CHECK(cudaMalloc(&d_max, 4)); m->err.ensure(16); CUDA_CHECK(cudaMemset(m->err.p, 0, 16)); }
        for_each_lin(m, [&](Lin& l) { derive_lin(m, l, d_max); });
        CUDA_CHECK(cudaDeviceSynchronize());
        cudaFree(d_max);
        m->tf32_ready = m->cfg.gemm_mode == kGemmTf32;
        m->finalized = true;
    });
}

uint64_t sealbart_device_bytes(const sealbart_t* m) { return m ? m->weight_bytes : 0; }

int64_t sealdec_hyps_per_query(const sealdec_params_t* p) {
    if (!p) return 0;
    return (int64_t)(p->max_length - 1) * 2 * p->num_beams + p->num_beams;
}


}  // extern "C"

namespace {

struct GenArgs {
    const sealfm_t* fm; const uint32_t* occ_d; const sealdec_params_t* p; sealdec_groups_t grp;
    const int64_t* ids_d; const int64_t* mask_d; int64_t Q, S;
    float* o_score; int32_t* o_len; int32_t* o_tok; uint8_t* o_valid; uint64_t* o_lo; uint64_t* o_hi; int32_t* err_d;
};

// Enqueues one whole generate (encoder, every decode step, records) on cx.s.  No host synchronisation unless
// src_hint == -1.  `timing` = bracket the phases with CUDA events (not possible while the stream is being captured).
bool fused_head_on(const sealbart* m) {
    static const bool env_on = [] { const char* e = std::getenv("SEALB200_FUSED_HEAD"); return !e || std::atoi(e) != 0; }();
    return m->fused_head >= 0 ? m->fused_head != 0 : env_on;
}

bool query_slices_on(const sealbart* m) {
    static const bool env_on = [] { const char* e = std::getenv("SEALB200_QUERY_SLICES"); return !e || std::atoi(e) != 0; }();
    return m->query_slices >= 0 ? m->query_slices != 0 : env_on;
}

void set_select_smem() {
    CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<512, 8192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SelSharedT<8192>)));
    CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<256, 4096>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SelSharedT<4096>)));
    CUDA_CHECK(cudaFuncSetAttribute(topk_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopkMaxVocab * 4));
    CUDA_CHECK(cudaFuncSetAttribute(topk_threshold_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopkMaxVocab * 4));
}

// topk_threshold_cluster_kernel on `rows` rows of 1 <= V <= kTopkClusterMaxVocab values: one cluster of
// topk_cluster_ctas(V) CTAs per row (set_select_smem() first)
void launch_topk_threshold_cluster(cudaStream_t s, int64_t rows, int V, int64_t ld, const float* logits, int top_k, float* row_thr) {
    const int n = topk_cluster_ctas(V);
    if (rows * n > INT32_MAX) throw ApiError(SEALFM_EINVAL, "too many logits rows for one top-k threshold launch");
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)n; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)(rows * n)); cfg.blockDim = dim3(kTopkThreads);
    cfg.dynamicSmemBytes = (size_t)topk_cluster_chunk(V) * 4; cfg.stream = s;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, topk_threshold_cluster_kernel, V, ld, logits, top_k, row_thr));
}

// (max, log sum exp over x >= tau, tau) of `rows` logits rows of V values at stride ld into row_thr[rows][3]
// (set_select_smem() first): one CTA per row up to kTopkMaxVocab, one cluster per row above.  The generate's top-k steps
// and sealdec_debug_topk_threshold.
void launch_topk_threshold(cudaStream_t s, int64_t rows, int V, int64_t ld, const float* logits, int top_k, float* row_thr) {
    if (V > kTopkMaxVocab) { launch_topk_threshold_cluster(s, rows, V, ld, logits, top_k, row_thr); return; }
    launch_k(topk_threshold_kernel, (unsigned)rows, kTopkThreads, (size_t)V * 4, s, V, ld, logits, top_k, row_thr);
}

// One decode step's selection on Q queries: topk_threshold_kernel on a top-k step (topk_warp_step), topk_rows_kernel, then
// select_merge_kernel (set_select_smem() first).  Returns `lists`, the candidate lists per query.  The first step (cur_len 1): beams 1.. carry -1e9 and are pruned
// exactly inside one CTA per query; afterwards one CTA per row.  Diverse beam groups at the first step: lists of row 0
// (every group leader) and row 1 (every other beam) only, see select_merge_kernel.
int launch_select_step(cudaStream_t s, const FmView& view, const StepCfg& c, const StepState& st, const RowScratch& rs, int64_t Q) {
    const int B = c.num_beams, gs = B / c.num_groups;
    int lists;
    if (topk_warp_step(c))
        launch_topk_threshold(s, c.logits_shared ? Q : Q * B, c.V, c.ld, st.logits, c.top_k, rs.row_thr);
    if (c.cur_len == 1 && c.num_groups > 1) {
        lists = gs > 1 ? 2 : 1;
        launch_k(topk_rows_kernel<512, 8192>, (unsigned)(Q * lists), 512, sizeof(SelSharedT<8192>), s, c, st, rs, lists, 1);
    } else if (c.cur_len == 1) {
        lists = 1;
        launch_k(topk_rows_kernel<512, 8192>, (unsigned)Q, 512, sizeof(SelSharedT<8192>), s, c, st, rs, 1, B);
    } else {
        lists = B;
        launch_k(topk_rows_kernel<256, 4096>, (unsigned)(Q * B), 256, sizeof(SelSharedT<4096>), s, c, st, rs, B, 1);
    }
    launch_k(select_merge_kernel, (unsigned)Q, kMergeThreads, 0, s, view, c, st, rs, lists);
    return lists;
}

// The StepCfg fields every step of a generate shares: the parameters, the groups and the vocabulary size V.  The
// per-step fields are set by set_step; hyp_base and head_tiles by the caller.
StepCfg step_cfg(const sealdec_params_t* p, const sealdec_groups_t& grp, int V) {
    StepCfg c{};
    c.num_beams = p->num_beams; c.K = 2 * p->num_beams; c.V = V; c.ld = (V + 3) / 4 * 4;
    c.min_length = p->min_length; c.max_length = p->max_length;
    c.eos_token_id = p->eos_token_id; c.pad_token_id = p->pad_token_id; c.model_eos_token_id = p->model_eos_token_id;
    c.forced_eos_token_id = p->forced_eos_token_id; c.forced_bos_token_id = p->forced_bos_token_id;
    c.stop_at_count = p->stop_at_count; c.always_allow_eos = p->always_allow_eos; c.disable_fm_index = p->disable_fm_index;
    c.remove_invalid_values = p->remove_invalid_values; c.shift = p->shift; c.T = p->max_length; c.mask_words = (V + 31) / 32;
    c.hyps_per_query = sealdec_hyps_per_query(p);
    c.num_groups = grp.num_beam_groups; c.diversity_penalty = grp.diversity_penalty;
    c.top_k = p->top_k < V ? p->top_k : 0;                 // top_k >= V keeps every logit: the top_k = 0 path
    return c;
}

// The fields of step cur_len: whether every row reads the occurring mask (the first step after a forced BOS, or the
// first), whether the next step's masks are expanded, and how the logits were produced (logits_shared: one row per
// query, the compact first step; logits_ignored: the forced-EOS step, on which the model did not run).
void set_step(StepCfg& c, int cur_len, bool logits_shared, bool logits_ignored) {
    const int eff_len = cur_len - (c.forced_bos_token_id >= 0 ? 1 : 0);
    c.cur_len = cur_len;
    c.first_step_shared_mask = (!c.disable_fm_index && eff_len == 1) ? 1 : 0;
    c.expand_next = (cur_len + 1 < c.T) ? 1 : 0;
    c.logits_shared = logits_shared ? 1 : 0;
    c.logits_ignored = logits_ignored ? 1 : 0;
}

void generate_enqueue(Ctx& cx, const Dims& D, const GenArgs& a, const FmView& view, uint64_t lo0, uint64_t hi0,
                      int64_t src_hint, bool timing) {
    sealbart* m = cx.m;
    const sealdec_params_t* p = a.p;
    const int B = D.B, K = 2 * B, T = D.T;
    const int64_t Q = D.Q, R = D.R;
    for (auto e : m->events) cudaEventDestroy(e);
    m->events.clear();
    auto mark = [&]() -> cudaEvent_t {
        if (!timing) return nullptr;
        cudaEvent_t e = new_event(m);
        CUDA_CHECK(cudaEventRecord(e, cx.s));
        return e;
    };
    CUDA_CHECK(cudaMemsetAsync(a.err_d, 0, 16, cx.s));
    m->fused_head_steps = 0;
    m->topk_cluster_steps = 0;
    mark();
    encoder_forward(cx, D, a.ids_d, a.mask_d, src_hint, a.err_d + 2);
    mark();

    float* sc[2] = {m->st_scores.as<float>(), m->st_scores.as<float>() + R};
    int32_t* tk[2] = {m->st_tokens.as<int32_t>(), m->st_tokens.as<int32_t>() + R * T};
    uint64_t* lo[2] = {m->st_lo.as<uint64_t>(), m->st_lo.as<uint64_t>() + R};
    uint64_t* hi[2] = {m->st_hi.as<uint64_t>(), m->st_hi.as<uint64_t>() + R};
    uint64_t* pw[2] = {m->st_pw.as<uint64_t>(), m->st_pw.as<uint64_t>() + R};
    int32_t* an[2] = {m->st_anc.as<int32_t>(), m->st_anc.as<int32_t>() + R * T};
    uint32_t* mk[2] = {m->st_mask.as<uint32_t>(), m->st_mask.as<uint32_t>() + (size_t)R * D.W};
    const int G = a.grp.num_beam_groups, gs = B / G;
    init_state_kernel<<<(unsigned)((R + 255) / 256), 256, 0, cx.s>>>(R, gs, T, p->decoder_start_token_id, p->pad_token_id,
                                                                    lo0, hi0, sc[0], tk[0], lo[0], hi[0], pw[0], an[0]);
    CUDA_CHECK(cudaGetLastError()); m->launches++;

    const StepCfg c = step_cfg(p, a.grp, D.V);
    set_select_smem();
    // Query slices.  The rows of a decode step are independent, so after the first step (compact: one row per query,
    // run on the whole batch) queries [0, Q0) and [Q0, Q), Q0 = ceil(Q / 2), run the rest of the decode -- decoder
    // layers, lm_head, selection, mask expansion -- on two streams: the caller's and m->slice_stream.  One
    // slice's attention and add+LN kernels then run beside the other slice's GEMM CTAs (wgmma_gemm_x3_kernel leaves
    // registers and shared memory on the SM for them), and each slice's last GEMM wave is filled by the other's work.
    // A kernel computes every row the same way on a slice as on the whole batch once a slice has more than kAddLnRowMax
    // rows (add+LN takes the warp-per-row kernel either way) and no GEMM of a slice is skinny enough for split-K (more
    // than sm_count / 2 tiles at the narrowest N; bart-large from 2 049 rows on): the lm_head's banded tile order only
    // reorders independent tiles -- the records are bit-identical with slicing on or off.  Off while profile_gemm
    // brackets every GEMM with events: overlapping GEMMs would make their summed durations meaningless.
    const int64_t Q0 = (Q + 1) / 2, R1 = (Q - Q0) * B;       // R1: rows of the smaller slice
    const int64_t min_tiles = (R1 + GM - 1) / GM * ((std::min(D.d, D.V) + GN - 1) / GN);
    const bool sliced = query_slices_on(m) && !m->profile_gemm && R1 > kAddLnRowMax && 2 * min_tiles > sm_count();
    auto slice_dims = [&](int64_t q0, int64_t nq) {
        Dims S = D;
        S.Q = nq; S.R = nq * B; S.q0 = q0; S.r0 = q0 * B; S.Qb = D.Q; S.Rb = D.R;
        return S;
    };
    const int H = (int)c.hyps_per_query, head_tiles = (D.V + GN - 1) / GN;
    static const bool compact_first = [] { const char* e = std::getenv("SEALB200_COMPACT_FIRST"); return !e || std::atoi(e) != 0; }();
    static const bool skip_dead = [] { const char* e = std::getenv("SEALB200_SKIP_DEAD_STEP"); return !e || std::atoi(e) != 0; }();
    auto is_dead = [&](int cur_len) {
        // Dead step: when ForcedEOSTokenLogitsProcessor fires (cur_len == max_length - 1, HF semantics restated
        // in apply_processors) it overwrites EVERY processed score with a constant, so neither the recorded
        // hypotheses nor the (already final) beams depend on the model output of this step -- the reference
        // computes it and discards it.  Nothing later reads this position's k / v either.
        const bool forced_all = p->forced_eos_token_id >= 0 && cur_len == p->max_length - 1 && cur_len + 1 == T &&
                                !(p->forced_bos_token_id >= 0 && cur_len == 1);
        return skip_dead && forced_all;
    };
    // The model forward of step `step` on the rows of PD (the whole batch or a slice); `timed` parts record the phase
    // events (sealdec_last_phase_us).  Returns whether the lm_head took the statistics epilogue.
    auto model_part = [&](Ctx& pc, const Dims& PD, int step, bool timed) {
        const int cur = step & 1, cur_len = step + 1;
        const bool compact = compact_first && cur_len == 1;
        const bool dead = is_dead(cur_len);
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
        cudaEvent_t b = (timing && timed) ? new_event(m) : nullptr;
        // Statistics epilogue of the lm_head (HeadEpi): the select kernels then read this step's logits only at the
        // row's read set.  topk_rows_kernel reads lp[v] for v in row_bits() and select_merge_kernel (G > 1) for the
        // candidates it re-scores.  With the FM index on, past the first (shared-mask) step and with one group,
        // row_bits() is the row's mask_in bits, or eos (rule 1), or pad (rule 2), plus eos with always_allow_eos --
        // within mask bits + {eos, pad}; apply_processors only overwrites values.  select_merge_kernel's -inf fill-ins
        // (fewer than K = 2B finite candidates, want < K) read the unconstrained score of the lowest flat indices of the
        // query that are not finite candidates: fewer than K + want < 2K <= 128 flat indices from the query's first
        // row, i.e. columns 0..127 of that row (V >= 128) -- the first n tile, which HeadEpi stores in full for every
        // row.  Every other case stays dense:
        // the compact first step, disable_fm_index, forced BOS (eff_len 1 reads the occurring mask), G > 1, the top-k
        // warp (its threshold needs every logit of the row), the other GEMM modes.
        const int eff_len = cur_len - (p->forced_bos_token_id >= 0 ? 1 : 0);
        HeadEpi he{};
        if (fused_head_on(m) && !dead && !compact && !p->disable_fm_index && eff_len > 1 && G == 1 && c.top_k == 0 &&
            head_stats_mode(m->cfg.gemm_mode)) {
            he = HeadEpi{m->st_hstat.as<float2>() + PD.r0 * head_tiles, mk[cur] + PD.r0 * D.W, (int)D.W, p->eos_token_id, p->pad_token_id};
            if (m->poison_logits) CUDA_CHECK(cudaMemsetAsync(m->logits.as<float>() + PD.r0 * D.ld, 0xFF, (size_t)PD.R * D.ld * 4, pc.s));
        }
        pc.head_fused = false;
        if (!dead) decoder_step(pc, PD, tk[cur] + PD.r0 * T, cur_len, an[cur] + PD.r0 * T, true, b, compact, he);
        else if (b) CUDA_CHECK(cudaEventRecord(b, pc.s));
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
        if (timed) m->fused_head_steps += pc.head_fused ? 1 : 0;
        return pc.head_fused;
    };
    // A StepState holding only where the hypothesis records of queries q0.. go (each step's and the final beams')
    auto records = [&](int64_t q0) {
        StepState st{};
        st.hyp_score = a.o_score + q0 * H; st.hyp_len = a.o_len + q0 * H; st.hyp_tokens = a.o_tok + q0 * H * T;
        st.hyp_valid = a.o_valid + q0 * H; st.hyp_lo = a.o_lo ? a.o_lo + q0 * H : nullptr; st.hyp_hi = a.o_hi ? a.o_hi + q0 * H : nullptr;
        return st;
    };
    // The selection of step `step` on the rows of PD, from the logits model_part left (head_fused: statistics epilogue).
    auto select_part = [&](Ctx& pc, const Dims& PD, unsigned long long* wide, int step, bool head_fused, bool timed) {
        const int cur = step & 1, cur_len = step + 1;
        const bool compact = compact_first && cur_len == 1;
        const bool dead = is_dead(cur_len);
        const int64_t r0 = PD.r0, q0 = PD.q0;
        StepCfg cs = c;
        set_step(cs, cur_len, compact && !dead, dead);
        cs.head_tiles = head_fused ? head_tiles : 0;
        cs.hyp_base = step * K;
        StepState st = records(q0);
        st.beam_scores_in = sc[cur] + r0; st.beam_scores_out = sc[cur ^ 1] + r0;
        st.tokens_in = tk[cur] + r0 * T; st.tokens_out = tk[cur ^ 1] + r0 * T;
        st.lo_in = lo[cur] + r0; st.lo_out = lo[cur ^ 1] + r0; st.hi_in = hi[cur] + r0; st.hi_out = hi[cur ^ 1] + r0;
        st.pw_in = pw[cur] + r0; st.pw_out = pw[cur ^ 1] + r0;
        st.anc_in = an[cur] + r0 * T; st.anc_out = an[cur ^ 1] + r0 * T;
        st.mask_in = mk[cur] + r0 * D.W; st.mask_out = mk[cur ^ 1] + r0 * D.W;
        // the compact first step wrote one logits row per query (of the whole batch)
        st.occurring_mask = a.occ_d; st.logits = m->logits.as<float>() + (cs.logits_shared ? q0 : r0) * D.ld;
        st.head_stats = m->st_hstat.as<float2>() + r0 * head_tiles;
        st.error_flag = a.err_d;
        const RowScratch rs{m->st_rowmax.as<float>() + r0, m->st_rowls.as<float>() + r0, m->st_rule.as<uint8_t>() + r0,
                            m->st_cval.as<float>() + r0 * K, m->st_cidx.as<int32_t>() + r0 * K, m->st_ccnt.as<int32_t>() + r0,
                            m->st_thr.as<float>() + (cs.logits_shared ? q0 : r0) * 3};
        launch_select_step(pc.s, view, cs, st, rs, PD.Q);
        m->launches += topk_warp_step(cs) ? 3 : 2;
        if (timed && topk_warp_step(cs) && cs.V > kTopkMaxVocab) m->topk_cluster_steps++;
        if (cs.expand_next && !p->disable_fm_index) {          // successor sets of the new beams -> next step's masks (:107)
            launch_expand_masks(view, pc.s, (uint64_t)PD.R, lo[cur ^ 1] + r0, hi[cur ^ 1] + r0, mk[cur ^ 1] + r0 * D.W, (uint32_t)D.W,
                                (uint32_t)D.V, (uint32_t)p->shift, wide);
            m->launches += 2;
        }
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
    };
    auto finalize_part = [&](Ctx& pc, const Dims& PD) {
        const int cur = (T - 1) & 1;
        const int64_t r0 = PD.r0;
        StepCfg cs = c;
        set_step(cs, T, false, false);
        cs.hyp_base = (T - 1) * K;
        finalize_kernel<<<(unsigned)((PD.R + 255) / 256), 256, 0, pc.s>>>(PD.Q, cs, sc[cur] + r0, tk[cur] + r0 * T, lo[cur] + r0, hi[cur] + r0,
                                                                         records(PD.q0));
        CUDA_CHECK(cudaGetLastError()); m->launches++;
    };
    if (!sliced) {
        for (int step = 0; step + 1 < T; ++step) {
            const bool fused = model_part(cx, D, step, true);
            select_part(cx, D, m->st_wide.as<unsigned long long>(), step, fused, true);
        }
        finalize_part(cx, D);
    } else {
        // slice 0 on the caller's stream (it records the per-step phase events), slice 1 on slice_stream; the steps of
        // the two are enqueued alternately so that both streams always have work queued
        m->last_paths |= kPathQuerySlices;
        const Dims PD[2] = {slice_dims(0, Q0), slice_dims(Q0, Q - Q0)};
        unsigned long long* wide[2] = {m->st_wide.as<unsigned long long>(), m->st_wide1.as<unsigned long long>()};
        // The first step selects per slice, so that every ancestor index is slice-relative from the start, but both
        // slices do so before the fork: the compact step's logits rows (one per query of the whole batch) lie inside
        // slice 0's rows, which its next lm_head overwrites.
        const bool fused0 = model_part(cx, D, 0, true);
        for (int i = 0; i < 2; ++i) select_part(cx, PD[i], wide[i], 0, fused0, i == 0);
        CUDA_CHECK(cudaEventRecord(m->slice_fork, cx.s));
        CUDA_CHECK(cudaStreamWaitEvent(m->slice_stream, m->slice_fork, 0));
        Ctx pcx[2] = {Ctx{m, cx.s}, Ctx{m, m->slice_stream}};
        pcx[1].slice = 1;
        for (int step = 1; step + 1 < T; ++step)
            for (int i = 0; i < 2; ++i) {
                const bool fused = model_part(pcx[i], PD[i], step, i == 0);
                select_part(pcx[i], PD[i], wide[i], step, fused, i == 0);
            }
        for (int i = 0; i < 2; ++i) finalize_part(pcx[i], PD[i]);
        CUDA_CHECK(cudaEventRecord(m->slice_join, m->slice_stream));
        CUDA_CHECK(cudaStreamWaitEvent(cx.s, m->slice_join, 0));
    }
    mark();
    // events in creation order: ev0, ev_enc, then per step a, b, c, d, then end (sealdec_last_phase_us); with query
    // slices a..d of every step after the first come from slice 0
}

template <typename T> void key_put(std::vector<uint8_t>& k, const T& v) {
    const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
    k.insert(k.end(), b, b + sizeof(T));
}

// NULL = one group.  1 <= G <= num_beams, num_beams % G == 0 (BeamSearchScorerWithMemory, seal/beam_search.py:597-601);
// the penalty only exists with G > 1 and > 0 (seal/beam_search.py:447-454), it is 0 otherwise.
sealdec_groups_t checked_groups(const sealdec_groups_t* g, int num_beams) {
    sealdec_groups_t r{1, 0.f};
    if (!g) return r;
    if (g->num_beam_groups < 1 || g->num_beam_groups > num_beams || num_beams % g->num_beam_groups != 0)
        throw ApiError(SEALFM_EINVAL, "num_beam_groups must divide num_beams and be in [1, num_beams]");
    if (!std::isfinite(g->diversity_penalty)) throw ApiError(SEALFM_EINVAL, "diversity_penalty must be finite");
    r.num_beam_groups = g->num_beam_groups;
    if (r.num_beam_groups > 1 && g->diversity_penalty > 0.f) r.diversity_penalty = g->diversity_penalty;
    return r;
}

// top_k: 0 = off, > 0 TopKLogitsWarper(top_k) on every step's logits -- only on the single-group path (group_beam_search
// has no warper, seal/beam_search.py:523-532) and for rows that fit the shared memory of one cluster of
// topk_threshold_cluster_kernel.
void check_top_k(int32_t top_k, const sealdec_groups_t& grp, int V) {
    if (top_k < 0) throw ApiError(SEALFM_EINVAL, "top_k must be >= 0 (0 = off)");
    if (top_k > 0 && grp.num_beam_groups > 1) throw ApiError(SEALFM_EINVAL, "top_k > 0 needs num_beam_groups == 1");
    if (top_k > 0 && V > kTopkClusterMaxVocab)
        throw ApiError(SEALFM_EINVAL, "top_k > 0 needs vocab_size <= " + std::to_string(kTopkClusterMaxVocab));
}

void drop_graphs(sealbart* m) {
    for (auto& g : m->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    m->graphs.clear();
    m->seen_keys.clear();
}

// A source whose attention mask is all zero has nothing to attend to: the softmax denominator of the encoder and
// cross-attention kernels stays zero (HF instead spreads the weight over the masked keys and gives finite logits).
// SEAL never builds one; the host-buffer
// entry points reject it, the device-buffer ones document it as a precondition.  The same holds for token ids
// outside [0, V): the embedding kernels index the table with them unchecked (the reference raises IndexError).
void check_token_ids(const int64_t* ids, int64_t n, int V, const char* what) {
    for (int64_t i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= V)
            throw ApiError(SEALFM_EINVAL, std::string(what) + " token id " + std::to_string(ids[i]) + " outside [0, vocab_size)");
}

void check_sources(const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, int V) {
    for (int64_t q = 0; q < Q; ++q) {
        bool any = false;
        for (int64_t s2 = 0; s2 < S && !any; ++s2) any = mask[q * S + s2] != 0;
        if (!any) throw ApiError(SEALFM_EINVAL, "source " + std::to_string(q) + " has an all-zero attention mask");
    }
    check_token_ids(ids, Q * S, V, "source");
}

// The number of real tokens of host masks [Q][S] whose every row is right-padded ("ones then zeros"), else -1
int64_t right_padded_tokens(const int64_t* mask, int64_t Q, int64_t S) {
    int64_t n = 0;
    for (int64_t q = 0; q < Q; ++q) {
        int64_t len = 0;
        for (int64_t s2 = 0; s2 < S; ++s2) { const bool on = mask[q * S + s2] != 0; if (on && s2 != len) return -1; len += on; }
        n += len;
    }
    return n;
}

// out[r * out_stride] = log_softmax(logits[r] / temperature)[targets[r * tgt_stride]] (0 for a target outside
// [0, V)) and / or the whole row into full[r * full_ld ..]: sealdec_teacher_forced and sealdec_debug_target_logprob
void launch_target_logprob(cudaStream_t s, int64_t R, int V, int64_t ld, const float* logits, const int64_t* targets,
                           int64_t tgt_stride, float temperature, float* out, int64_t out_stride, float* full,
                           int64_t full_ld) {
    target_logprob_kernel<<<(unsigned)R, 256, 0, s>>>(R, V, ld, logits, targets, tgt_stride, temperature, out, out_stride,
                                                      full, full_ld);
    CUDA_CHECK(cudaGetLastError());
}

}  // namespace

extern "C" {

int sealdec_generate_dx_ex(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_d, const sealdec_params_t* p,
                           const int64_t* ids_d, const int64_t* mask_d, int64_t Q, int64_t S, sealfm_stream_t stream,
                           float* o_score, int32_t* o_len, int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo,
                           uint64_t* o_hi, int32_t* err_d, int64_t src_tokens_hint, const sealdec_groups_t* groups) {
    return guarded([&] {
        check_model(m);
        if (!p || !ids_d || !mask_d || !o_score || !o_len || !o_tok || !o_valid || !err_d) throw ApiError(SEALFM_EINVAL, "null argument");
        const int B = p->num_beams, K = 2 * B, T = p->max_length;
        if (B < 1 || B > kSelMaxBeams || K > kSelMaxK) throw ApiError(SEALFM_EINVAL, "num_beams must be in [1,32]");
        const sealdec_groups_t grp = checked_groups(groups, B);
        check_top_k(p->top_k, grp, m->cfg.vocab_size);
        if (T < 2 || T > kMaxLen) throw ApiError(SEALFM_EINVAL, "max_length must be in [2,128]");
        if (Q <= 0 || S <= 0) throw ApiError(SEALFM_EINVAL, "empty batch");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        if (src_tokens_hint < -2 || src_tokens_hint > Q * S) throw ApiError(SEALFM_EINVAL, "bad source-token hint");
        FmView view{};
        uint64_t lo0 = 0, hi0 = 0;
        if (!p->disable_fm_index) {
            if (!fm || sealfm_device(fm) != m->device) throw ApiError(SEALFM_ENODEVICE, "FM index not bound to the model's device");
            if (!occ_d) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
            view = sealfm_view(fm);
            lo0 = 0; hi0 = view.m + 1;                               // get_range([]) = (0, size()+1)  (index.py:106-110)
            if (p->n_force_decoding_from > 0) {
                std::vector<uint64_t> q(p->n_force_decoding_from), off{0, (uint64_t)p->n_force_decoding_from};
                for (int i = 0; i < p->n_force_decoding_from; ++i) q[i] = (uint64_t)p->force_decoding_from[i] + p->shift;
                int rc = sealfm_backward_search_multi(fm, 1, q.data(), off.data(), &lo0, &hi0);
                if (rc) throw ApiError(rc, sealfm_last_error());
            }
        }
        Ctx cx{m, (cudaStream_t)stream};
        m->launches = 0;
        m->last_paths = 0;
        m->ovf = err_d + 1;
        m->last_used_graph = 0;
        const Dims D = make_dims(m, Q, S, B, T);
        ensure_workspace(m, D);
        if (!p->disable_fm_index) m->st_wide.ensure(expand_scratch_bytes(view.L, (uint64_t)D.R));   // wide-row work list + BFS frontiers
        if (query_slices_on(m)) {                              // generate_enqueue may run the batch as two query slices
            if (!m->slice_stream) CUDA_CHECK(cudaStreamCreateWithFlags(&m->slice_stream, cudaStreamNonBlocking));
            if (!m->slice_fork) CUDA_CHECK(cudaEventCreateWithFlags(&m->slice_fork, cudaEventDisableTiming));
            if (!m->slice_join) CUDA_CHECK(cudaEventCreateWithFlags(&m->slice_join, cudaEventDisableTiming));
            if (!p->disable_fm_index) m->st_wide1.ensure(expand_scratch_bytes(view.L, (uint64_t)(Q / 2) * B));
        }
        const GenArgs a{fm, occ_d, p, grp, ids_d, mask_d, Q, S, o_score, o_len, o_tok, o_valid, o_lo, o_hi, err_d};

        // ---- CUDA graph of the whole call: a batch-20 generate is ~1 900 short kernels, i.e. launch-latency-bound.
        // Shapes, parameters and buffer addresses are the key; the first call of a key runs eagerly (it sizes every
        // lazily grown buffer), the second is captured, later ones are one cudaGraphLaunch.
        static const int env_graph = [] { const char* e = std::getenv("SEALB200_GRAPH"); return e ? std::atoi(e) : -1; }();
        const int policy = m->graph_policy >= 0 ? m->graph_policy : env_graph;
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        if (cx.s) CUDA_CHECK(cudaStreamIsCapturing(cx.s, &cap));
        const bool small = D.R <= 4096;
        bool want_graph = cx.s != nullptr && cap == cudaStreamCaptureStatusNone && !m->profile_gemm &&
                          (policy == 1 || (policy < 0 && small));
        // inside a graph the encoder never needs the host: small batches compute the padded rows (the key then does
        // not depend on the batch's contents), larger ones use the caller's token count
        int64_t eff_hint = src_tokens_hint;
        if (want_graph) { if (small) eff_hint = -2; else if (src_tokens_hint == -1) want_graph = false; }
        if (!want_graph) { generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, cap == cudaStreamCaptureStatusNone); m->phase_us[0] = -1; return; }

        std::vector<uint8_t> key;
        key_put(key, Q); key_put(key, S); key_put(key, eff_hint); key_put(key, lo0); key_put(key, hi0);
        key_put(key, m->cfg.gemm_mode); key_put(key, cx.s);
        sealdec_params_t pc = *p; pc.force_decoding_from = nullptr; key_put(key, pc);
        for (int i = 0; i < p->n_force_decoding_from; ++i) key_put(key, p->force_decoding_from[i]);
        key_put(key, grp.num_beam_groups); key_put(key, grp.diversity_penalty);
        key_put(key, fused_head_on(m)); key_put(key, m->poison_logits); key_put(key, query_slices_on(m));
        key_put(key, view.blocks); key_put(key, view.csym); key_put(key, view.node_tab); key_put(key, view.m);
        key_put(key, occ_d); key_put(key, ids_d); key_put(key, mask_d); key_put(key, o_score); key_put(key, o_len);
        key_put(key, o_tok); key_put(key, o_valid); key_put(key, o_lo); key_put(key, o_hi); key_put(key, err_d);
        if (!m->graphs.empty() && m->graphs.front().epoch != g_ws_epoch) drop_graphs(m);
        for (auto& g : m->graphs)
            if (g.key == key) {
                CUDA_CHECK(cudaGraphLaunch(g.exec, cx.s));
                g.stamp = ++m->graph_stamp; m->launches = g.launches; m->last_paths = g.paths; m->last_used_graph = 1;
                m->topk_cluster_steps = g.topk_cluster_steps;
                return;
            }
        bool seen = false;
        for (auto& k2 : m->seen_keys) if (k2 == key) { seen = true; break; }
        if (!seen) {                                           // first time: eager (sizes split-K / staging buffers)
            if (m->seen_keys.size() >= 16) m->seen_keys.erase(m->seen_keys.begin());
            m->seen_keys.push_back(key);
            generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, true);
            m->phase_us[0] = -1;
            return;
        }
        const uint64_t epoch0 = g_ws_epoch;
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        bool captured = false;
        if (cudaStreamBeginCapture(cx.s, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
            try {
                generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, false);
                captured = cudaStreamEndCapture(cx.s, &graph) == cudaSuccess && graph != nullptr;
            } catch (...) {
                cudaStreamEndCapture(cx.s, &graph);
                captured = false;
            }
            if (captured && g_ws_epoch == epoch0) captured = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
            else captured = false;
            if (graph) cudaGraphDestroy(graph);
        }
        if (!captured) {
            // a buffer moved while capturing, or this driver cannot capture / instantiate the call (the launches were
            // only recorded, nothing ran): run it the ordinary way, and stop trying on this model
            cudaGetLastError();
            if (g_ws_epoch == epoch0) m->graph_policy = 0;
            m->launches = 0; m->last_paths = 0;
            generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, true);
            return;
        }
        if (m->graphs.size() >= 8) {                           // evict the least recently used
            size_t victim = 0;
            for (size_t i = 1; i < m->graphs.size(); ++i) if (m->graphs[i].stamp < m->graphs[victim].stamp) victim = i;
            cudaGraphExecDestroy(m->graphs[victim].exec);
            m->graphs.erase(m->graphs.begin() + victim);
        }
        sealbart::GraphEntry ge; ge.key = std::move(key); ge.epoch = g_ws_epoch; ge.exec = exec; ge.launches = m->launches; ge.paths = m->last_paths; ge.stamp = ++m->graph_stamp;
        ge.topk_cluster_steps = m->topk_cluster_steps;
        m->graphs.push_back(std::move(ge));
        CUDA_CHECK(cudaGraphLaunch(exec, cx.s));
        m->last_used_graph = 1;
    });
}

int sealdec_generate_dx(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_d, const sealdec_params_t* p,
                        const int64_t* ids_d, const int64_t* mask_d, int64_t Q, int64_t S, sealfm_stream_t stream,
                        float* o_score, int32_t* o_len, int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo,
                        uint64_t* o_hi, int32_t* err_d, int64_t src_tokens_hint) {
    return sealdec_generate_dx_ex(m, fm, occ_d, p, ids_d, mask_d, Q, S, stream, o_score, o_len, o_tok, o_valid, o_lo, o_hi,
                                  err_d, src_tokens_hint, nullptr);
}

int sealdec_generate_d(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_d, const sealdec_params_t* p,
                       const int64_t* ids_d, const int64_t* mask_d, int64_t Q, int64_t S, sealfm_stream_t stream,
                       float* o_score, int32_t* o_len, int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo,
                       uint64_t* o_hi, int32_t* err_d) {
    return sealdec_generate_dx(m, fm, occ_d, p, ids_d, mask_d, Q, S, stream, o_score, o_len, o_tok, o_valid, o_lo, o_hi, err_d, -1);
}

int sealbart_set_option(sealbart_t* m, const char* name, int64_t value) {
    return guarded([&] {
        if (!m || !name) throw ApiError(SEALFM_EINVAL, "null argument");
        const std::string n(name);
        if (n == "cuda_graph") { if (value < -1 || value > 1) throw ApiError(SEALFM_EINVAL, "cuda_graph: -1 auto, 0 off, 1 on"); m->graph_policy = (int)value; }
        else if (n == "gemm_mode") {
            check_model(m);
            if (value == m->cfg.gemm_mode) return;
            if (value == kGemmBf16 || bf16_weights(m))
                throw ApiError(SEALFM_EINVAL, "gemm_mode 6 (bf16 weights) is chosen at creation: the handle has no fp32 weights to switch to or from");
            if (value == kGemmTf32 && is_3xfp16(m->cfg.gemm_mode)) { ensure_tf32_splits(m); m->cfg.gemm_mode = kGemmTf32; }
            else if (is_3xfp16(value) && m->head.w_h1) m->cfg.gemm_mode = (int)value;
            else throw ApiError(SEALFM_EINVAL, "gemm_mode can only switch between the 3xFP16 modes (3, 5) and 2 (3xTF32)");
            for_each_lin(m, [](Lin& l) { l.maps_ready = false; l.maps2_ready = false; });
            drop_graphs(m);
        }
        else if (n == "fused_head") {
            if (value < -1 || value > 1) throw ApiError(SEALFM_EINVAL, "fused_head: -1 environment, 0 off, 1 on");
            m->fused_head = (int)value;
        }
        else if (n == "poison_logits") m->poison_logits = value != 0;
        else if (n == "query_slices") {
            if (value < -1 || value > 1) throw ApiError(SEALFM_EINVAL, "query_slices: -1 environment, 0 off, 1 on");
            m->query_slices = (int)value;
        }
        else throw ApiError(SEALFM_EINVAL, "unknown option: " + n);
    });
}

int64_t sealbart_get_stat(const sealbart_t* m, const char* name) {
    if (!m || !name) return -1;
    const std::string n(name);
    if (n == "last_used_graph") return m->last_used_graph;
    if (n == "overflow_fallbacks") return m->overflow_fallbacks;
    if (n == "gemm_mode") return m->cfg.gemm_mode;
    if (n == "cached_graphs") return (int64_t)m->graphs.size();
    if (n == "fused_head_steps") return m->fused_head_steps;
    if (n == "topk_cluster_steps") return m->topk_cluster_steps;
    if (n == "last_paths") return m->last_paths;
    return -1;
}

int sealdec_last_phase_us(const sealbart_t* mc, double out5[5]) {
    return guarded([&] {
        sealbart* m = const_cast<sealbart*>(mc);
        if (!m || !out5) throw ApiError(SEALFM_EINVAL, "null argument");
        CUDA_CHECK(cudaSetDevice(m->device));
        const size_t n = m->events.size();
        if (n < 3) throw ApiError(SEALFM_EINVAL, "no generate call recorded");
        CUDA_CHECK(cudaEventSynchronize(m->events[n - 1]));
        auto ms = [&](size_t a, size_t b) { float t = 0; CUDA_CHECK(cudaEventElapsedTime(&t, m->events[a], m->events[b])); return (double)t * 1e3; };
        double enc = ms(0, 1), layers = 0, head = 0, sel = 0;
        for (size_t i = 2; i + 3 < n; i += 4) { layers += ms(i, i + 1); head += ms(i + 1, i + 2); sel += ms(i + 2, i + 3); }
        out5[0] = enc; out5[1] = layers; out5[2] = head; out5[3] = sel; out5[4] = ms(0, n - 1);
    });
}

int sealdec_debug_gemm_trace(int enable, int64_t out20[20]) {
    return guarded([&] {
        if (out20) {
            CUDA_CHECK(cudaDeviceSynchronize());
            long long h[20];
            CUDA_CHECK(cudaMemcpyFromSymbol(h, g_gemm_trace, sizeof(h)));
            for (int i = 0; i < 20; ++i) out20[i] = h[i];
        }
        const int on = enable ? 1 : 0;
        CUDA_CHECK(cudaMemcpyToSymbol(g_gemm_trace_on, &on, sizeof(int)));
    });
}

int sealdec_debug_gemm_units(int64_t* out, int32_t n) {
    return guarded([&] {
        if (!out || n < 0 || n > 4 * kTraceUnits) throw ApiError(SEALFM_EINVAL, "out is null or n is outside [0, 4 * 256]");
#ifndef SEAL_GEMM_UNIT_TRACE
        throw ApiError(SEALFM_EINVAL, "built without the per-unit GEMM timeline (make GEMM_UNIT_TRACE=1)");
#endif
        CUDA_CHECK(cudaDeviceSynchronize());
        std::vector<long long> h(4 * kTraceUnits);
        CUDA_CHECK(cudaMemcpyFromSymbol(h.data(), g_gemm_units, h.size() * sizeof(long long)));
        for (int i = 0; i < n; ++i) out[i] = h[i];
        std::fill(h.begin(), h.end(), 0ll);
        CUDA_CHECK(cudaMemcpyToSymbol(g_gemm_units, h.data(), h.size() * sizeof(long long)));
    });
}

int64_t sealdec_last_launch_count(const sealbart_t* m) { return m ? m->launches : 0; }

int sealdec_profile_gemm(sealbart_t* m, int enable, double* total_us, int64_t* launches, double* flops) {
    return guarded([&] {
        if (!m) throw ApiError(SEALFM_EINVAL, "null model");
        CUDA_CHECK(cudaSetDevice(m->device));
        if (total_us && launches && flops) {
            CUDA_CHECK(cudaDeviceSynchronize());
            double us = 0;
            for (auto& e : m->gemm_events) { float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e.first, e.second)); us += (double)ms * 1e3; }
            *total_us = us; *launches = (int64_t)m->gemm_events.size(); *flops = m->gemm_flops;
        }
        for (auto& e : m->gemm_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
        m->gemm_events.clear(); m->gemm_flops = 0;
        m->profile_gemm = enable != 0;
    });
}

int sealdec_generate(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_host, const sealdec_params_t* p,
                     const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, float* o_score, int32_t* o_len,
                     int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo, uint64_t* o_hi) {
    return sealdec_generate_ex(m, fm, occ_host, p, ids, mask, Q, S, o_score, o_len, o_tok, o_valid, o_lo, o_hi, nullptr);
}

int sealdec_generate_ex(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_host, const sealdec_params_t* p,
                        const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, float* o_score, int32_t* o_len,
                        int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo, uint64_t* o_hi, const sealdec_groups_t* groups) {
    return guarded([&] {
        check_model(m);
        if (!p || !ids || !mask || Q <= 0 || S <= 0) throw ApiError(SEALFM_EINVAL, "null argument / empty batch");
        checked_groups(groups, p->num_beams);
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        const int64_t H = sealdec_hyps_per_query(p), T = p->max_length;
        const int W = (m->cfg.vocab_size + 31) / 32;
        // the caller's buffers are host memory: the real-token count costs nothing to know here, so the encoder
        // never has to ask the device for it (right-padded masks only; anything else takes the padded path)
        int64_t hint = right_padded_tokens(mask, Q, S);
        if (hint <= 0) hint = -2;
        if (!m->stream) CUDA_CHECK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
        cudaStream_t s = m->stream;
        m->in_ids.ensure(Q * S * 8); m->in_mask.ensure(Q * S * 8); m->in_occ.ensure((size_t)W * 4);
        m->hy_score.ensure(Q * H * 4); m->hy_len.ensure(Q * H * 4); m->hy_tok.ensure(Q * H * T * 4);
        m->hy_valid.ensure(Q * H); m->hy_lo.ensure(Q * H * 8); m->hy_hi.ensure(Q * H * 8); m->err.ensure(16);
        CUDA_CHECK(cudaMemcpyAsync(m->in_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(m->in_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        if (occ_host) CUDA_CHECK(cudaMemcpyAsync(m->in_occ.p, occ_host, (size_t)W * 4, cudaMemcpyHostToDevice, s));
        int32_t errs[4] = {0, 0, 0, 0};
        auto run = [&] {                                       // one pass on the staged inputs
            return sealdec_generate_dx_ex(m, fm, occ_host ? m->in_occ.as<uint32_t>() : nullptr, p, m->in_ids.as<int64_t>(),
                                          m->in_mask.as<int64_t>(), Q, S, s, m->hy_score.as<float>(), m->hy_len.as<int32_t>(),
                                          m->hy_tok.as<int32_t>(), m->hy_valid.as<uint8_t>(), o_lo ? m->hy_lo.as<uint64_t>() : nullptr,
                                          o_hi ? m->hy_hi.as<uint64_t>() : nullptr, m->err.as<int32_t>(), hint, groups);
        };
        if (const int rc = run()) throw ApiError(rc, last_error());
        CUDA_CHECK(cudaMemcpyAsync(errs, m->err.p, 16, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (errs[1] && is_3xfp16(m->cfg.gemm_mode)) {
            // An activation left the fp16 range (|x| > 65504; the producers saturate and raise the flag): this pass is
            // redone with the 3xTF32 kernels, which have fp32's range -- the caller gets exact-range results either way.
            const int mode = m->cfg.gemm_mode;
            { const int r0 = sealbart_set_option(m, "gemm_mode", kGemmTf32); if (r0) throw ApiError(r0, last_error()); }
            m->overflow_fallbacks++;
            const int rc = run();
            const int rc2 = sealbart_set_option(m, "gemm_mode", mode);
            if (rc) throw ApiError(rc, last_error());
            if (rc2) throw ApiError(rc2, last_error());
            CUDA_CHECK(cudaMemcpyAsync(errs, m->err.p, 16, cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
        }
        CUDA_CHECK(cudaMemcpyAsync(o_score, m->hy_score.p, Q * H * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_len, m->hy_len.p, Q * H * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_tok, m->hy_tok.p, Q * H * T * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_valid, m->hy_valid.p, Q * H, cudaMemcpyDeviceToHost, s));
        if (o_lo) CUDA_CHECK(cudaMemcpyAsync(o_lo, m->hy_lo.p, Q * H * 8, cudaMemcpyDeviceToHost, s));
        if (o_hi) CUDA_CHECK(cudaMemcpyAsync(o_hi, m->hy_hi.p, Q * H * 8, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (errs[2]) throw ApiError(SEALFM_EINVAL, "internal: source-token count mismatch");
        if (errs[0]) throw ApiError(SEALFM_EINVAL, "beam: fewer than num_beams non-EOS candidates (seal/beam_search.py:687-690)");
    });
}

int sealdec_debug_step_logits(sealbart_t* m, const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, int32_t B,
                              const int64_t* dec_ids, int64_t t, float* out_logits) {
    return sealdec_debug_step_logits_ex(m, ids, mask, Q, S, B, dec_ids, t, nullptr, -1, out_logits);
}

int sealdec_debug_step_logits_ex(sealbart_t* m, const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, int32_t B,
                                 const int64_t* dec_ids, int64_t t, const int32_t* anc, int64_t src_tokens_hint,
                                 float* out_logits) {
    return guarded([&] {
        check_model(m);
        if (!ids || !mask || !dec_ids || !out_logits || t < 1 || t > kMaxLen || Q <= 0 || S <= 0 || B < 1)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        // a count is only valid for right-padded masks; checked here, where the mask is host memory
        if (src_tokens_hint != -1 && src_tokens_hint != -2 && right_padded_tokens(mask, Q, S) != src_tokens_hint)
            throw ApiError(SEALFM_EINVAL, "src_tokens_hint does not match a right-padded mask");
        const int T = (int)t;
        if (m->arch == 2 && T > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "decoder inputs longer than the position table");
        const Dims D = make_dims(m, Q, S, B, T);
        check_token_ids(dec_ids, D.R * T, m->cfg.vocab_size, "decoder");
        if (anc)
            for (int64_t i = 0; i < D.R * T; ++i)
                if (anc[i] < 0 || anc[i] >= D.R) throw ApiError(SEALFM_EINVAL, "ancestor row out of range");
        ensure_workspace(m, D);
        m->ovf = m->err.as<int>() + 1;
        Buf d_ids, d_mask;
        d_ids.ensure(Q * S * 8); d_mask.ensure(Q * S * 8); m->dbg_ids.ensure(D.R * t * 8);
        cudaStream_t s = nullptr;
        CUDA_CHECK(cudaMemcpyAsync(d_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(d_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(m->dbg_ids.p, dec_ids, D.R * t * 8, cudaMemcpyHostToDevice, s));
        Ctx cx{m, s};
        m->launches = 0;
        m->last_paths = 0;
        encoder_forward(cx, D, d_ids.as<int64_t>(), d_mask.as<int64_t>(), src_tokens_hint);
        int32_t* tk = m->st_tokens.as<int32_t>(); int32_t* an = m->st_anc.as<int32_t>();
        ids_to_tokens_kernel<<<(unsigned)((D.R + 255) / 256), 256, 0, s>>>(D.R, T, T, m->dbg_ids.as<int64_t>(), tk, an);
        CUDA_CHECK(cudaGetLastError());
        if (anc) CUDA_CHECK(cudaMemcpyAsync(an, anc, (size_t)D.R * T * 4, cudaMemcpyHostToDevice, s));   // replaces the identity
        for (int cur_len = 1; cur_len <= T; ++cur_len) decoder_step(cx, D, tk, cur_len, an, cur_len == T, nullptr);
        CUDA_CHECK(cudaMemcpy2DAsync(out_logits, (size_t)D.V * 4, m->logits.p, (size_t)D.ld * 4, (size_t)D.V * 4, D.R,
                                     cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int sealdec_teacher_forced(sealbart_t* m, const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S,
                           const int64_t* dec_ids, const int32_t* row_query, int64_t N, int64_t T, float temperature,
                           float* out_logprob, int64_t out_full_pos, float* out_full) {
    return guarded([&] {
        check_model(m);
        if (!ids || !mask || !dec_ids || !row_query || N <= 0 || T < 1 || T > kMaxLen || Q <= 0 || S <= 0)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        if (out_full && (out_full_pos < 0 || out_full_pos >= T)) throw ApiError(SEALFM_EINVAL, "out_full_pos must be in [0, T)");
        if (m->arch == 2 && T > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "decoder inputs longer than the position table");
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        check_token_ids(dec_ids, N * T, m->cfg.vocab_size, "decoder");
        for (int64_t r = 0; r < N; ++r) {
            if (row_query[r] < 0 || row_query[r] >= Q || (r && row_query[r] < row_query[r - 1]))
                throw ApiError(SEALFM_EINVAL, "row_query must be sorted and within [0, Q)");
        }
        const int64_t kChunk = 4096;                           // decoder rows per pass (logits: 4096 x V floats)
        Dims D = make_dims(m, Q, S, 1, (int)T);
        D.R = std::min<int64_t>(N, kChunk);
        ensure_workspace(m, D);
        m->ovf = m->err.as<int>() + 1;
        cudaStream_t s = nullptr;
        CUDA_CHECK(cudaMemsetAsync(m->ovf, 0, 4, s));          // before the encoder: its producers raise it too
        Buf d_ids, d_mask, d_dec, d_gq, d_gs, d_out, d_full;
        d_ids.ensure(Q * S * 8); d_mask.ensure(Q * S * 8);
        CUDA_CHECK(cudaMemcpyAsync(d_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(d_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        Ctx cx{m, s};
        m->launches = 0;
        m->last_paths = 0;
        encoder_forward(cx, D, d_ids.as<int64_t>(), d_mask.as<int64_t>());
        d_dec.ensure(D.R * T * 8); d_gq.ensure((D.R + 1) * 4); d_gs.ensure((D.R + 2) * 4);
        if (T > 1) d_out.ensure(D.R * (T - 1) * 4);
        if (out_full) d_full.ensure((size_t)D.R * D.V * 4);
        for (int64_t r0 = 0; r0 < N; r0 += kChunk) {
            const int64_t rows = std::min(kChunk, N - r0);
            std::vector<int32_t> gq, gs;
            for (int64_t r = 0; r < rows; ++r)
                if (r == 0 || row_query[r0 + r] != row_query[r0 + r - 1]) { gq.push_back(row_query[r0 + r]); gs.push_back((int32_t)r); }
            gs.push_back((int32_t)rows);
            CUDA_CHECK(cudaMemcpyAsync(d_dec.p, dec_ids + r0 * T, rows * T * 8, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(d_gq.p, gq.data(), gq.size() * 4, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(d_gs.p, gs.data(), gs.size() * 4, cudaMemcpyHostToDevice, s));
            Dims C = D;
            C.R = rows; C.G = (int64_t)gq.size(); C.grp_query = d_gq.as<int32_t>(); C.grp_start = d_gs.as<int32_t>();
            int32_t* tk = m->st_tokens.as<int32_t>(); int32_t* an = m->st_anc.as<int32_t>();
            ids_to_tokens_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(rows, (int)T, (int)T, d_dec.as<int64_t>(), tk, an);
            CUDA_CHECK(cudaGetLastError());
            for (int p = 0; p < T; ++p) {
                const bool need = (p + 1 < T) || (out_full && p == out_full_pos);
                if (!need) continue;                           // the last position only feeds the full-vector output
                decoder_step(cx, C, tk, p + 1, an, true, nullptr);
                launch_target_logprob(s, rows, C.V, C.ld, m->logits.as<float>(), d_dec.as<int64_t>() + (p + 1 < T ? p + 1 : 0), T,
                                      temperature, (p + 1 < T) ? d_out.as<float>() + p : nullptr, T - 1,
                                      (out_full && p == out_full_pos) ? d_full.as<float>() : nullptr, C.V);
                m->launches++;
            }
            if (T > 1 && out_logprob)
                CUDA_CHECK(cudaMemcpyAsync(out_logprob + r0 * (T - 1), d_out.p, rows * (T - 1) * 4, cudaMemcpyDeviceToHost, s));
            if (out_full)
                CUDA_CHECK(cudaMemcpyAsync(out_full + (size_t)r0 * D.V, d_full.p, (size_t)rows * D.V * 4, cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));              // gq/gs are stack temporaries; outputs consumed per chunk
        }
        int32_t ovf = 0;
        CUDA_CHECK(cudaMemcpy(&ovf, m->err.as<int>() + 1, 4, cudaMemcpyDeviceToHost));
        if (ovf) throw ApiError(SEALFM_EINVAL, "fp16 range exceeded in the 3xFP16 GEMM path (|x| > 65504); use gemm_mode 2 (3xTF32)");
    });
}

}  // extern "C"

namespace {

// The lm_head statistics epilogue of sealdec_debug_head: the row masks [M][ceil(N/32)] (host), eos / pad, and where
// the statistics [Mpad][ceil(N/128)] go (host; Mpad = M rounded up to 128 rows) and whether the epilogue ran.
struct DebugHead { const uint32_t* mask; int eos, pad; float* stats; int32_t* fused; };

// presplit: 3xFP16 and 3xBF16 split the activations once, outside the timed calls (as the decoder's producers do)
int debug_gemm(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias, float* C,
               int32_t gelu, int32_t iters, double* avg_us, int32_t band, int32_t store, bool presplit,
               const DebugHead* head = nullptr) {
    return guarded([&] {
        if (!A || !W || (store && !C) || M <= 0 || N <= 0 || K <= 0 || band < -1) throw ApiError(SEALFM_EINVAL, "bad argument");
        if (head && (!head_stats_mode(mode) || !store || gelu || iters > 0 || !head->mask || !head->stats || !head->fused))
            throw ApiError(SEALFM_EINVAL, "bad argument");
        require_device();
        check_gemm_mode(mode);
        sealbart fake; fake.cfg.gemm_mode = mode;              // owns the weights and the scratch, as a model does
        CUDA_CHECK(cudaGetDevice(&fake.device));
        fake.err.ensure(16); CUDA_CHECK(cudaMemset(fake.err.p, 0, 16)); fake.ovf = fake.err.as<int>() + 1;
        Lin l;                                                 // loaded (sealbart_set_tensor) and derived (sealbart_finalize) as the model's
        make_lin(&fake, l, N, K);
        upload(l.w_bf ? (void*)l.w_bf : (void*)l.w, l.w_bf != nullptr, W, (uint64_t)N * K);
        if (bias) upload(l.b, false, bias, N);
        else l.b = nullptr;
        Buf d_max; d_max.ensure(4);
        derive_lin(&fake, l, d_max.as<unsigned int>());
        fake.gemm_band = band;
        Buf dA, dC, ah1, ah2;
        const int ldc = (N + 3) / 4 * 4;
        dA.ensure((size_t)M * K * 4); dC.ensure((size_t)M * ldc * 4);
        CUDA_CHECK(cudaMemcpy(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice));
        Act a{dA.as<float>()};
        if (presplit && mode != kGemmTf32)
            with_format(mode, [&](auto t) { a = split_act<decltype(t)>(nullptr, a.x, M * K, ah1, ah2, fake.ovf); });
        const Act c{store ? dC.as<float>() : nullptr};
        Ctx cx{&fake, nullptr};
        Buf dmask, dstats;
        const int64_t m_pad = (M + GM - 1) / GM * GM;
        const int n_tiles = (N + GN - 1) / GN, mask_words = (N + 31) / 32;
        if (head) {
            // every output the epilogue may skip starts poisoned: C is NaN, the statistics all-ones bits (NaN)
            dC.release(); dC.ensure((size_t)m_pad * ldc * 4);
            CUDA_CHECK(cudaMemset(dC.p, 0xFF, (size_t)m_pad * ldc * 4));
            dstats.ensure((size_t)m_pad * n_tiles * 8);
            CUDA_CHECK(cudaMemset(dstats.p, 0xFF, (size_t)m_pad * n_tiles * 8));
            dmask.ensure((size_t)M * mask_words * 4);
            CUDA_CHECK(cudaMemcpy(dmask.p, head->mask, (size_t)M * mask_words * 4, cudaMemcpyHostToDevice));
            cx.head = HeadEpi{dstats.as<float2>(), dmask.as<uint32_t>(), mask_words, head->eos, head->pad};
        }
        gemm(cx, M, N, K, a, K, l, head ? Act{dC.as<float>()} : c, ldc, gelu ? kActGelu : kActNone);
        CUDA_CHECK(cudaDeviceSynchronize());
        if (head) {
            *head->fused = cx.head_fused ? 1 : 0;
            CUDA_CHECK(cudaMemcpy2D(C, (size_t)N * 4, dC.p, (size_t)ldc * 4, (size_t)N * 4, m_pad, cudaMemcpyDeviceToHost));
            CUDA_CHECK(cudaMemcpy(head->stats, dstats.p, (size_t)m_pad * n_tiles * 8, cudaMemcpyDeviceToHost));
            return;
        }
        if (iters > 0 && avg_us) {
            cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
            CUDA_CHECK(cudaEventRecord(e0, nullptr));
            for (int i = 0; i < iters; ++i) gemm(cx, M, N, K, a, K, l, c, ldc, gelu ? kActGelu : kActNone);
            CUDA_CHECK(cudaEventRecord(e1, nullptr));
            CUDA_CHECK(cudaEventSynchronize(e1));
            float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
            *avg_us = (double)ms * 1e3 / iters;
            cudaEventDestroy(e0); cudaEventDestroy(e1);
        }
        if (store) CUDA_CHECK(cudaMemcpy2D(C, (size_t)N * 4, dC.p, (size_t)ldc * 4, (size_t)N * 4, M, cudaMemcpyDeviceToHost));
    });
}

// deterministic pseudo-random logits in [-8, 8) and `per_row` allowed tokens per row
__global__ void debug_fill_rows_kernel(int64_t R, int V, int ld, int W, int per_row, float* __restrict__ logits, uint32_t* __restrict__ mask) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R * ld; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t h = (uint32_t)i * 2654435761u; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
        logits[i] = (float)(h >> 8) * (16.f / 16777216.f) - 8.f;
        if (i < R * per_row) {
            const int64_t r = i / per_row;
            const int v = (int)((uint64_t)(i % per_row + 1) * 7919u * (uint64_t)(r + 1) % (uint64_t)V);
            atomicOr(&mask[r * W + (v >> 5)], 1u << (v & 31));
        }
    }
}

}  // namespace

extern "C" {

int sealdec_debug_gemm(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias, float* C,
                       int32_t gelu, int32_t iters, double* avg_us) {
    return debug_gemm(mode, M, N, K, A, W, bias, C, gelu, iters, avg_us, -1, 1, false);
}

int sealdec_debug_gemm_ex(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias, float* C,
                          int32_t gelu, int32_t iters, double* avg_us, int32_t band, int32_t store) {
    return debug_gemm(mode, M, N, K, A, W, bias, C, gelu, iters, avg_us, band, store, true);
}

int sealdec_debug_head(int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias,
                       const uint32_t* mask, int32_t eos, int32_t pad, float* C, float* stats, int32_t* fused) {
    const DebugHead h{mask, eos, pad, stats, fused};
    return debug_gemm(3, M, N, K, A, W, bias, C, 0, 0, nullptr, -1, 1, true, &h);
}

int sealdec_debug_head_ex(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias,
                          const uint32_t* mask, int32_t eos, int32_t pad, float* C, float* stats, int32_t* fused) {
    const DebugHead h{mask, eos, pad, stats, fused};
    return debug_gemm(mode, M, N, K, A, W, bias, C, 0, 0, nullptr, -1, 1, true, &h);
}

int sealdec_debug_select_step(const sealfm_t* fm, const sealdec_params_t* p, const sealdec_groups_t* groups, int64_t Q,
                              int32_t V, int32_t cur_len, int32_t logits_shared, int32_t logits_ignored,
                              const float* logits, const float* head_stats, const uint32_t* masks,
                              const uint32_t* occurring_mask, const float* beam_scores, const int32_t* tokens,
                              const int32_t* ancestry, const uint64_t* lo, const uint64_t* hi, const uint64_t* pw,
                              float* row_max, float* row_logsum, uint8_t* row_rule, float* cand_val, int32_t* cand_idx,
                              int32_t* cand_cnt, int32_t* lists, float* beam_scores_out, int32_t* tokens_out,
                              int32_t* ancestry_out, uint64_t* lo_out, uint64_t* hi_out, uint64_t* pw_out,
                              float* rec_score, int32_t* rec_len, int32_t* rec_tokens, uint8_t* rec_valid,
                              uint64_t* rec_lo, uint64_t* rec_hi, int32_t* error_flag) {
    return guarded([&] {
        if (!p || !beam_scores || !tokens || !ancestry || !lo || !hi || !pw || !row_max || !row_logsum || !row_rule ||
            !cand_val || !cand_idx || !cand_cnt || !lists || !beam_scores_out || !tokens_out || !ancestry_out || !lo_out ||
            !hi_out || !pw_out || !rec_score || !rec_len || !rec_tokens || !rec_valid || !rec_lo || !rec_hi || !error_flag)
            throw ApiError(SEALFM_EINVAL, "null argument");
        // only configurations a generate produces (generate_enqueue)
        const int B = p->num_beams, K = 2 * B, T = p->max_length;
        if (B < 1 || B > kSelMaxBeams || K > kSelMaxK) throw ApiError(SEALFM_EINVAL, "num_beams must be in [1,32]");
        const sealdec_groups_t grp = checked_groups(groups, B);
        if (T < 2 || T > kMaxLen) throw ApiError(SEALFM_EINVAL, "max_length must be in [2,128]");
        if (cur_len < 1 || cur_len > T - 1) throw ApiError(SEALFM_EINVAL, "cur_len must be in [1, max_length - 1]");
        if (Q <= 0 || V <= 0 || (int64_t)B * V > INT32_MAX) throw ApiError(SEALFM_EINVAL, "bad Q / V");
        if (p->eos_token_id < 0 || p->eos_token_id >= V || p->pad_token_id < 0 || p->pad_token_id >= V ||
            p->model_eos_token_id >= V || p->forced_eos_token_id >= V || p->forced_bos_token_id >= V)
            throw ApiError(SEALFM_EINVAL, "token ids must be below V");
        const bool fb_step = p->forced_bos_token_id >= 0 && cur_len == 1;
        const int eff_len = cur_len - (p->forced_bos_token_id >= 0 ? 1 : 0);
        const bool fm_on = !p->disable_fm_index;
        const bool shared_mask = fm_on && eff_len == 1;
        if (logits_ignored && !(p->forced_eos_token_id >= 0 && cur_len == T - 1 && !fb_step))
            throw ApiError(SEALFM_EINVAL, "logits_ignored: only on the forced-EOS step");
        if (logits_shared && (cur_len != 1 || logits_ignored)) throw ApiError(SEALFM_EINVAL, "logits_shared: only at cur_len 1");
        if (!logits_ignored && !logits) throw ApiError(SEALFM_EINVAL, "logits missing");
        if (head_stats && !(fm_on && eff_len > 1 && grp.num_beam_groups == 1 && V >= GN && !logits_ignored && !logits_shared))
            throw ApiError(SEALFM_EINVAL, "head statistics: only after the first step, with the FM index on, one group and V >= 128");
        check_top_k(p->top_k, grp, V);
        if (head_stats && p->top_k > 0) throw ApiError(SEALFM_EINVAL, "head statistics: not with top_k > 0 (dense logits)");
        if (fm_on && !fb_step && !shared_mask && !masks) throw ApiError(SEALFM_EINVAL, "masks missing");
        if (shared_mask && !occurring_mask) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
        FmView view{};
        if (fm_on) {
            if (!fm || sealfm_device(fm) < 0) throw ApiError(SEALFM_ENODEVICE, "FM index not on a device");
            CUDA_CHECK(cudaSetDevice(sealfm_device(fm)));
            view = sealfm_view(fm);
        } else
            require_device();
        const int64_t R = Q * B;
        for (int64_t r = 0; r < R; ++r) {
            if (lo[r] > hi[r] || (fm_on && hi[r] > view.m + 1)) throw ApiError(SEALFM_EINVAL, "SA range out of the index");
            for (int i = 0; i < T; ++i)
                if (ancestry[r * T + i] < 0 || ancestry[r * T + i] >= R) throw ApiError(SEALFM_EINVAL, "ancestor row out of range");
        }
        const int ld = (V + 3) / 4 * 4, W = (V + 31) / 32, tiles = (V + GN - 1) / GN;
        const int64_t lrows = logits_shared ? Q : R;

        Buf d_lg, d_hs, d_mk, d_occ, d_sc, d_tk, d_an, d_lo, d_hi, d_pw, d_rmax, d_rls, d_rule, d_cval, d_cidx, d_ccnt, d_sco, d_tko,
            d_ano, d_loo, d_hio, d_pwo, d_hsc, d_hlen, d_htk, d_hval, d_hlo, d_hhi, d_err, d_thr;
        auto up = [&](Buf& d, const void* h, size_t bytes) {
            d.ensure(bytes);
            if (h) CUDA_CHECK(cudaMemcpy(d.p, h, bytes, cudaMemcpyHostToDevice));
            else CUDA_CHECK(cudaMemset(d.p, 0, bytes));
        };
        // outputs and scratch start as NaN / all-ones bits: a value read before it is written, or never written, shows
        auto poisoned = [&](Buf& d, size_t bytes) { d.ensure(bytes); CUDA_CHECK(cudaMemset(d.p, 0xFF, bytes)); };
        poisoned(d_lg, (size_t)lrows * ld * 4);                 // the padding columns ld - V stay NaN
        if (!logits_ignored)
            CUDA_CHECK(cudaMemcpy2D(d_lg.p, (size_t)ld * 4, logits, (size_t)V * 4, (size_t)V * 4, lrows, cudaMemcpyHostToDevice));
        if (head_stats) up(d_hs, head_stats, (size_t)R * tiles * 8);
        up(d_mk, masks, (size_t)R * W * 4);
        up(d_occ, occurring_mask, (size_t)W * 4);
        up(d_sc, beam_scores, R * 4); up(d_tk, tokens, (size_t)R * T * 4); up(d_an, ancestry, (size_t)R * T * 4);
        up(d_lo, lo, R * 8); up(d_hi, hi, R * 8); up(d_pw, pw, R * 8);
        poisoned(d_rmax, R * 4); poisoned(d_rls, R * 4); poisoned(d_rule, R); poisoned(d_thr, (size_t)R * 3 * 4);
        poisoned(d_cval, (size_t)R * K * 4); poisoned(d_cidx, (size_t)R * K * 4); poisoned(d_ccnt, R * 4);
        poisoned(d_sco, R * 4); poisoned(d_tko, (size_t)R * T * 4); poisoned(d_ano, (size_t)R * T * 4);
        poisoned(d_loo, R * 8); poisoned(d_hio, R * 8); poisoned(d_pwo, R * 8);
        poisoned(d_hsc, (size_t)Q * K * 4); poisoned(d_hlen, (size_t)Q * K * 4); poisoned(d_htk, (size_t)Q * K * T * 4);
        poisoned(d_hval, (size_t)Q * K); poisoned(d_hlo, (size_t)Q * K * 8); poisoned(d_hhi, (size_t)Q * K * 8);
        d_err.ensure(16); CUDA_CHECK(cudaMemset(d_err.p, 0, 16));

        StepCfg c = step_cfg(p, grp, V);
        set_step(c, cur_len, logits_shared, logits_ignored);
        c.hyps_per_query = K; c.hyp_base = 0;                  // the step's 2B records of each query
        c.head_tiles = head_stats ? tiles : 0;
        StepState st{};
        st.beam_scores_in = d_sc.as<float>(); st.beam_scores_out = d_sco.as<float>();
        st.tokens_in = d_tk.as<int32_t>(); st.tokens_out = d_tko.as<int32_t>();
        st.lo_in = d_lo.as<uint64_t>(); st.lo_out = d_loo.as<uint64_t>(); st.hi_in = d_hi.as<uint64_t>(); st.hi_out = d_hio.as<uint64_t>();
        st.pw_in = d_pw.as<uint64_t>(); st.pw_out = d_pwo.as<uint64_t>();
        st.anc_in = d_an.as<int32_t>(); st.anc_out = d_ano.as<int32_t>();
        st.mask_in = d_mk.as<uint32_t>(); st.occurring_mask = d_occ.as<uint32_t>();
        st.logits = d_lg.as<float>(); st.head_stats = head_stats ? d_hs.as<float2>() : nullptr;
        st.hyp_score = d_hsc.as<float>(); st.hyp_len = d_hlen.as<int32_t>(); st.hyp_tokens = d_htk.as<int32_t>();
        st.hyp_valid = d_hval.as<uint8_t>(); st.hyp_lo = d_hlo.as<uint64_t>(); st.hyp_hi = d_hhi.as<uint64_t>();
        st.error_flag = d_err.as<int32_t>();
        RowScratch rs{d_rmax.as<float>(), d_rls.as<float>(), d_rule.as<uint8_t>(), d_cval.as<float>(), d_cidx.as<int32_t>(),
                      d_ccnt.as<int32_t>(), d_thr.as<float>()};
        set_select_smem();
        *lists = launch_select_step(nullptr, view, c, st, rs, Q);
        CUDA_CHECK(cudaDeviceSynchronize());
        auto down = [&](void* h, const Buf& d, size_t bytes) { CUDA_CHECK(cudaMemcpy(h, d.p, bytes, cudaMemcpyDeviceToHost)); };
        down(row_max, d_rmax, R * 4); down(row_logsum, d_rls, R * 4); down(row_rule, d_rule, R);
        down(cand_val, d_cval, (size_t)R * K * 4); down(cand_idx, d_cidx, (size_t)R * K * 4); down(cand_cnt, d_ccnt, R * 4);
        down(beam_scores_out, d_sco, R * 4); down(tokens_out, d_tko, (size_t)R * T * 4); down(ancestry_out, d_ano, (size_t)R * T * 4);
        down(lo_out, d_loo, R * 8); down(hi_out, d_hio, R * 8); down(pw_out, d_pwo, R * 8);
        down(rec_score, d_hsc, (size_t)Q * K * 4); down(rec_len, d_hlen, (size_t)Q * K * 4); down(rec_tokens, d_htk, (size_t)Q * K * T * 4);
        down(rec_valid, d_hval, (size_t)Q * K); down(rec_lo, d_hlo, (size_t)Q * K * 8); down(rec_hi, d_hhi, (size_t)Q * K * 8);
        down(error_flag, d_err, 4);
    });
}

int sealdec_debug_topk_rows(int64_t R, int32_t V, int32_t num_beams, int32_t per_row, int32_t iters, double* avg_us) {
    return guarded([&] {
        if (R <= 0 || V <= 0 || num_beams < 1 || num_beams > kSelMaxBeams || R % num_beams || per_row < 0 || iters <= 0 || !avg_us)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        require_device();
        const int ld = (V + 3) / 4 * 4, W = (V + 31) / 32, B = num_beams, K = 2 * B, T = 3;
        Buf lg, mk, sc, tk, pw, rmax, rls, rule, cval, cidx, ccnt;
        lg.ensure((size_t)R * ld * 4); mk.ensure((size_t)R * W * 4); sc.ensure((size_t)R * 4); tk.ensure((size_t)R * T * 4);
        pw.ensure((size_t)R * 8); rmax.ensure((size_t)R * 4); rls.ensure((size_t)R * 4); rule.ensure((size_t)R);
        cval.ensure((size_t)R * K * 4); cidx.ensure((size_t)R * K * 4); ccnt.ensure((size_t)R * 4);
        CUDA_CHECK(cudaMemset(mk.p, 0, (size_t)R * W * 4)); CUDA_CHECK(cudaMemset(sc.p, 0, (size_t)R * 4));
        CUDA_CHECK(cudaMemset(tk.p, 0, (size_t)R * T * 4)); CUDA_CHECK(cudaMemset(pw.p, 0, (size_t)R * 8));
        debug_fill_rows_kernel<<<sm_count() * 8, 256>>>(R, V, ld, W, per_row, lg.as<float>(), mk.as<uint32_t>());
        CUDA_CHECK(cudaGetLastError());
        // a later step (cur_len 2) of plain constrained beam search: every row is its own candidate list
        StepCfg c{};
        c.num_beams = B; c.K = K; c.V = V; c.ld = ld; c.cur_len = 2; c.min_length = 0; c.max_length = T;
        c.eos_token_id = 2; c.pad_token_id = 1; c.model_eos_token_id = 2; c.forced_eos_token_id = -1; c.forced_bos_token_id = -1;
        c.T = T; c.mask_words = W; c.expand_next = 1; c.num_groups = 1;
        StepState st{};
        st.beam_scores_in = sc.as<float>(); st.tokens_in = tk.as<int32_t>(); st.pw_in = pw.as<uint64_t>();
        st.mask_in = mk.as<uint32_t>(); st.logits = lg.as<float>();
        RowScratch rs{rmax.as<float>(), rls.as<float>(), rule.as<uint8_t>(), cval.as<float>(), cidx.as<int32_t>(), ccnt.as<int32_t>(),
                      nullptr};
        using RowsLater = SelSharedT<4096>;
        CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<256, 4096>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RowsLater)));
        launch_k(topk_rows_kernel<256, 4096>, (unsigned)R, 256, sizeof(RowsLater), nullptr, c, st, rs, B, 1);
        CUDA_CHECK(cudaDeviceSynchronize());
        cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0, nullptr));
        for (int i = 0; i < iters; ++i) launch_k(topk_rows_kernel<256, 4096>, (unsigned)R, 256, sizeof(RowsLater), nullptr, c, st, rs, B, 1);
        CUDA_CHECK(cudaEventRecord(e1, nullptr));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *avg_us = (double)ms * 1e3 / iters;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    });
}

}  // extern "C"

namespace {

// sealdec_debug_topk_threshold (cluster = false: V <= kTopkMaxVocab, the generate's dispatch) and
// sealdec_debug_topk_threshold_cluster (cluster = true: topk_threshold_cluster_kernel for V <= kTopkClusterMaxVocab)
int debug_topk_threshold(bool cluster, int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k, float* out_thr,
                         float* out_max, float* out_logsum) {
    return guarded([&] {
        if (R <= 0 || V <= 0 || ld < V || !logits || top_k < 1 || !out_thr || !out_max || !out_logsum || (uint64_t)R > INT32_MAX)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        const int max_v = cluster ? kTopkClusterMaxVocab : kTopkMaxVocab;
        if (V > max_v) throw ApiError(SEALFM_EINVAL, "V must be <= " + std::to_string(max_v));
        require_device();
        Buf d_lg, d_thr;
        d_lg.ensure((size_t)R * ld * 4); d_thr.ensure((size_t)R * 3 * 4);
        CUDA_CHECK(cudaMemcpy(d_lg.p, logits, (size_t)R * ld * 4, cudaMemcpyHostToDevice));
        CUDA_CHECK(cudaMemset(d_thr.p, 0xFF, (size_t)R * 3 * 4));
        set_select_smem();
        if (cluster) launch_topk_threshold_cluster(nullptr, R, V, ld, d_lg.as<float>(), top_k, d_thr.as<float>());
        else launch_topk_threshold(nullptr, R, V, ld, d_lg.as<float>(), top_k, d_thr.as<float>());
        CUDA_CHECK(cudaDeviceSynchronize());
        std::vector<float> h((size_t)R * 3);
        CUDA_CHECK(cudaMemcpy(h.data(), d_thr.p, h.size() * 4, cudaMemcpyDeviceToHost));
        for (int64_t r = 0; r < R; ++r) { out_max[r] = h[r * 3]; out_logsum[r] = h[r * 3 + 1]; out_thr[r] = h[r * 3 + 2]; }
    });
}

}  // namespace

extern "C" {

int sealdec_debug_topk_threshold(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k, float* out_thr,
                                 float* out_max, float* out_logsum) {
    return debug_topk_threshold(false, R, V, ld, logits, top_k, out_thr, out_max, out_logsum);
}

int sealdec_debug_topk_threshold_cluster(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k,
                                         float* out_thr, float* out_max, float* out_logsum) {
    return debug_topk_threshold(true, R, V, ld, logits, top_k, out_thr, out_max, out_logsum);
}

int sealdec_debug_target_logprob(int64_t R, int32_t V, int64_t ld, const float* logits, const int64_t* targets,
                                 int64_t tgt_stride, float temperature, float* out, int64_t out_stride, float* full,
                                 int64_t full_ld) {
    return guarded([&] {
        // only what sealdec_teacher_forced passes: ld >= V, a positive finite temperature, at least one output
        if (R <= 0 || V <= 0 || ld < V || !logits || (!out && !full)) throw ApiError(SEALFM_EINVAL, "bad argument");
        if (!(temperature > 0.f) || !std::isfinite(temperature)) throw ApiError(SEALFM_EINVAL, "temperature must be positive and finite");
        if (out && (!targets || tgt_stride < 1 || out_stride < 1)) throw ApiError(SEALFM_EINVAL, "bad target / output stride");
        if (full && full_ld < V) throw ApiError(SEALFM_EINVAL, "full_ld must be >= V");
        if ((uint64_t)R > INT32_MAX) throw ApiError(SEALFM_EINVAL, "too many rows");
        require_device();
        Buf d_lg, d_tg, d_out, d_full;
        const size_t n_out = out ? (size_t)(R - 1) * out_stride + 1 : 0;
        const size_t n_tg = out ? (size_t)(R - 1) * tgt_stride + 1 : 0;
        const size_t n_full = full ? (size_t)(R - 1) * full_ld + V : 0;
        d_lg.ensure((size_t)R * ld * 4);
        CUDA_CHECK(cudaMemcpy(d_lg.p, logits, (size_t)R * ld * 4, cudaMemcpyHostToDevice));
        // the outputs start as NaN: an element the kernel does not write comes back that way
        if (out) {
            d_tg.ensure(n_tg * 8); d_out.ensure(n_out * 4);
            CUDA_CHECK(cudaMemcpy(d_tg.p, targets, n_tg * 8, cudaMemcpyHostToDevice));
            CUDA_CHECK(cudaMemset(d_out.p, 0xFF, n_out * 4));
        }
        if (full) { d_full.ensure(n_full * 4); CUDA_CHECK(cudaMemset(d_full.p, 0xFF, n_full * 4)); }
        launch_target_logprob(nullptr, R, V, ld, d_lg.as<float>(), out ? d_tg.as<int64_t>() : nullptr, tgt_stride, temperature,
                              out ? d_out.as<float>() : nullptr, out_stride, full ? d_full.as<float>() : nullptr, full_ld);
        CUDA_CHECK(cudaDeviceSynchronize());
        if (out) CUDA_CHECK(cudaMemcpy(out, d_out.p, n_out * 4, cudaMemcpyDeviceToHost));
        if (full) CUDA_CHECK(cudaMemcpy(full, d_full.p, n_full * 4, cudaMemcpyDeviceToHost));
    });
}

int sealdec_debug_attention(const sealdec_attn_case_t* c, float* out, void* split1, void* split2, void* split3,
                            int32_t* overflow, float* kc_out, float* vc_out, uint32_t* path) {
    return guarded([&] {
        auto bad = [](const char* what) { return ApiError(SEALFM_EINVAL, what); };
        if (!c || !out || !path) throw bad("null argument");
        if (c->kind < 0 || c->kind > 2 || (c->arch != 0 && c->arch != 1)) throw bad("kind must be 0, 1 or 2 and arch 0 or 1");
        const bool t5 = c->arch == 1, enc = c->kind == 0, self = c->kind == 1, cross = c->kind == 2;
        const int d = c->d, heads = c->heads;
        if (heads < 1 || (int64_t)heads * kHeadDim != d) throw bad("heads must be 64 wide (d = 64 * heads)");
        if (d > (t5 ? 4096 : 1024)) throw bad("d must be <= 1024 (BART) / 4096 (T5)");
        if (c->Q < 1 || c->Q > (1 << 20)) throw bad("Q must be in [1, 2^20]");
        if (c->out_split < 0 || c->out_split > 3) throw bad("out_split must be 0..3");
        if (c->out_split == 0 && t5 && !cross) throw bad("the T5 kernels write only the split: out_split must not be 0");
        if (c->out_split && (!split1 || !split2 || (c->out_split == 3 && !split3) || (c->out_split == 2 && !overflow)))
            throw bad("split output missing");
        if (c->G && !cross) throw bad("ragged groups: cross-attention only");
        if (c->compact && (enc || c->G)) throw bad("compact: decoder steps without ragged groups only");
        const int64_t Q = c->Q;
        const bool t5_bias = t5 && !cross;
        if (t5_bias && (!c->rel_bias || c->num_buckets < 4 || c->num_buckets > 1024 || c->max_distance <= c->num_buckets / 2))
            throw bad("T5: rel_bias needed, num_buckets in [4, 1024], max_distance > num_buckets / 2");
        // the encoder side (kinds 0 and 2): N source rows, packed or masked
        int64_t N = 0;
        if (!self) {
            if (c->S < 1 || c->S > kT5MaxSource) throw bad("S must be in [1, 1024]");
            if (c->src_off) {
                if (c->src_off[0] != 0) throw bad("src_off[0] must be 0");
                for (int64_t qi = 0; qi < Q; ++qi) {
                    const int64_t len = (int64_t)c->src_off[qi + 1] - c->src_off[qi];
                    if (len < 1 || len > c->S) throw bad("packed source lengths must be in [1, S]");
                }
                N = c->src_off[Q];
            } else {
                if (!c->src_mask) throw bad("src_mask or src_off needed");
                for (int64_t qi = 0; qi < Q; ++qi) {
                    bool any = false;
                    for (int64_t s = 0; s < c->S; ++s) any |= c->src_mask[qi * c->S + s] != 0;
                    if (!any) throw bad("a query without a valid key");
                }
                N = Q * c->S;
            }
        }
        int64_t rows = 0, Rc = 0;
        if (enc) {
            if (!c->qkv) throw bad("qkv missing");
            rows = N;
        } else if (self) {
            if (c->B < 1 || c->B > 32) throw bad("B must be in [1, 32]");
            if (c->pos < 0 || c->T < c->pos + 1 || c->T > kMaxLen) throw bad("need 0 <= pos < T <= 128");
            if (c->compact && c->pos != 0) throw bad("compact: the first step (pos 0) only");
            if (!c->kc || !c->vc || !c->anc || !kc_out || !vc_out) throw bad("cache, ancestry or cache output missing");
            Rc = Q * c->B;
            rows = c->compact ? Q : Rc;
            for (int64_t i = 0; i < Rc * c->T; ++i)
                if (c->anc[i] < 0 || c->anc[i] >= Rc) throw bad("ancestor row out of range");
        } else {
            if (!c->ckv) throw bad("ckv missing");
            if (c->G) {
                if (c->G < 0 || !c->grp_query || !c->grp_start || c->grp_start[0] != 0) throw bad("ragged groups: G, grp_query, grp_start[0] = 0");
                for (int64_t g = 0; g < c->G; ++g) {
                    if (c->grp_start[g + 1] < c->grp_start[g]) throw bad("grp_start must be non-decreasing");
                    if (c->grp_query[g] < 0 || c->grp_query[g] >= Q) throw bad("grp_query out of range");
                }
                rows = c->grp_start[c->G];
            } else {
                if (c->B < 1) throw bad("B must be >= 1");
                rows = c->compact ? Q : Q * c->B;
            }
        }
        if (rows < 1) throw bad("no rows");
        const int cols = cross ? d : 3 * d;                    // the row width of qkv (kinds 0, 1) / q (kind 2)
        const bool use_saq = self && !t5 && use_self_attn_query(c->pos, c->B, c->compact != 0, false);
        if (c->split_ks > 1) {
            if (!(use_saq || (cross && use_cross_attn_small(c->S)))) throw bad("split-K slices: only for the kernels that sum them");
            if (!c->split_part || !c->split_bias) throw bad("split-K slices or bias missing");
        } else if (!enc && !(self ? c->qkv : c->q)) throw bad(self ? "qkv missing" : "q missing");
        require_device();

        Buf d_in, d_ckv, d_kc, d_vc, d_anc, d_mask, d_off, d_gq, d_gs, d_part, d_pb, d_rel, d_bkt, d_out, d_s1, d_s2, d_s3, d_ovf;
        auto up = [&](Buf& b, const void* h, size_t bytes) { b.ensure(bytes); CUDA_CHECK(cudaMemcpy(b.p, h, bytes, cudaMemcpyHostToDevice)); };
        auto nan = [&](Buf& b, size_t bytes) { b.ensure(bytes); CUDA_CHECK(cudaMemset(b.p, 0xFF, bytes)); };
        const size_t in_bytes = (size_t)rows * cols * 4;
        // qkv (kinds 0, 1) or q; with split-K slices the plain input is not read: NaN
        if (c->split_ks > 1) {
            nan(d_in, in_bytes);
            up(d_part, c->split_part, in_bytes * c->split_ks); up(d_pb, c->split_bias, (size_t)cols * 4);
        } else up(d_in, enc ? c->qkv : self ? c->qkv : c->q, in_bytes);
        if (cross) up(d_ckv, c->ckv, (size_t)N * 2 * d * 4);
        if (!self) {
            if (c->src_off) up(d_off, c->src_off, (size_t)(Q + 1) * 4);
            else up(d_mask, c->src_mask, (size_t)Q * c->S * 4);
        }
        const size_t cache_bytes = self ? (size_t)c->T * Rc * d * 4 : 0;
        if (self) {
            up(d_kc, c->kc, cache_bytes); up(d_vc, c->vc, cache_bytes); up(d_anc, c->anc, (size_t)Rc * c->T * 4);
            const size_t at_pos = (size_t)c->pos * Rc * d * 4, pos_bytes = (size_t)Rc * d * 4;      // the rows the step writes
            CUDA_CHECK(cudaMemset(d_kc.as<char>() + at_pos, 0xFF, pos_bytes)); CUDA_CHECK(cudaMemset(d_vc.as<char>() + at_pos, 0xFF, pos_bytes));
        }
        if (cross && c->G) { up(d_gq, c->grp_query, (size_t)c->G * 4); up(d_gs, c->grp_start, (size_t)(c->G + 1) * 4); }
        RelBias rb{};
        if (t5_bias) {
            // the model's bucket tables (t5_bucket_tables): distance key - query at entry dist + off
            const int off = enc ? kT5MaxSource - 1 : kMaxLen - 1;
            std::vector<int32_t> bkt(enc ? 2 * kT5MaxSource - 1 : kMaxLen);
            for (int i = 0; i < (int)bkt.size(); ++i) bkt[i] = t5_bucket(i - off, enc, c->num_buckets, c->max_distance);
            up(d_bkt, bkt.data(), bkt.size() * 4); up(d_rel, c->rel_bias, (size_t)c->num_buckets * heads * 4);
            rb = RelBias{d_rel.as<float>(), d_bkt.as<int32_t>(), off, heads};
        }
        const size_t out_n = (size_t)rows * d, piece = c->out_split == 1 ? 4 : 2;
        nan(d_out, out_n * 4);
        if (c->out_split) { nan(d_s1, out_n * piece); nan(d_s2, out_n * piece); }
        if (c->out_split == 3) nan(d_s3, out_n * piece);
        d_ovf.ensure(4); CUDA_CHECK(cudaMemset(d_ovf.p, 0, 4));
        SplitSrc src{};
        if (c->split_ks > 1) src = SplitSrc{d_part.as<float>(), c->split_ks, (int64_t)rows * cols, d_pb.as<float>(), c->split_unscale};

        const float* in = d_in.as<float>();
        const int32_t* mask = c->src_off ? nullptr : d_mask.as<int32_t>();
        const int32_t* soff = c->src_off ? d_off.as<int32_t>() : nullptr;
        auto run = [&](auto so) -> uint32_t {
            if (enc) return launch_enc_self_attn(nullptr, Q, d, heads, (int)c->S, in, mask, t5 ? &rb : nullptr, d_out.as<float>(), so, soff);
            if (self) {
                const SelfAttnArgs a{Q, rows, Rc, c->B, d, heads, c->pos, c->T, c->compact ? c->B : 1, in, d_kc.as<float>(), d_vc.as<float>(),
                                     d_anc.as<int32_t>(), d_out.as<float>()};
                return t5 ? launch_t5_dec_self_attn(nullptr, a, rb, so) : launch_bart_self_attn(nullptr, a, use_saq, so, src);
            }
            const CrossAttnArgs a{c->G ? c->G : Q, d, heads, c->compact ? 1 : c->B, (int)c->S, in, d_ckv.as<float>(), mask,
                                  c->G ? d_gq.as<int32_t>() : nullptr, c->G ? d_gs.as<int32_t>() : nullptr, d_out.as<float>(), soff};
            return launch_cross_attn(nullptr, a, so, src);
        };
        uint32_t bit;
        if (c->out_split == 3) bit = run(SplitBf16{d_s1.as<__nv_bfloat16>(), d_s2.as<__nv_bfloat16>(), d_s3.as<__nv_bfloat16>()});
        else bit = run(SplitOut{d_s1.p, d_s2.p, c->out_split, c->out_split == 2 ? d_ovf.as<int>() : nullptr});
        CUDA_CHECK(cudaDeviceSynchronize());
        auto down = [&](void* h, const Buf& b, size_t bytes) { CUDA_CHECK(cudaMemcpy(h, b.p, bytes, cudaMemcpyDeviceToHost)); };
        down(out, d_out, out_n * 4);
        if (c->out_split) { down(split1, d_s1, out_n * piece); down(split2, d_s2, out_n * piece); }
        if (c->out_split == 3) down(split3, d_s3, out_n * piece);
        if (overflow) down(overflow, d_ovf, 4);
        if (self) { down(kc_out, d_kc, cache_bytes); down(vc_out, d_vc, cache_bytes); }
        *path = bit;
    });
}

int sealdec_apply_index_mask_d(const sealfm_t* fm, sealfm_stream_t stream, const sealdec_processor_cfg_t* cfg,
                               const int64_t* input_ids_d, int64_t R, int64_t t, const uint32_t* occ_d,
                               const float* in_d, float* out_d, int64_t V, int64_t ld) {
    return guarded([&] {
        if (!fm || !cfg || !input_ids_d || !in_d || !out_d) throw ApiError(SEALFM_EINVAL, "null argument");
        const int dev = sealfm_device(fm);
        if (dev < 0) throw ApiError(SEALFM_ENODEVICE, "index not bound to a CUDA device (call sealfm_to_device)");
        CUDA_CHECK(cudaSetDevice(dev));
        if (R <= 0 || t < 1) throw ApiError(SEALFM_EINVAL, "empty input");
        cudaStream_t s = (cudaStream_t)stream;
        const FmView view = sealfm_view(fm);
        const int W = (int)((V + 31) / 32);
        dim3 grid((unsigned)R, (unsigned)std::min<int64_t>((V + 255) / 256, 64));
        const bool fb = cfg->forced_bos_token_id >= 0;
        if (fb && t == 1) {                                                     // :66-69
            apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, nullptr, W, 1, nullptr, cfg->eos_token_id,
                                                   cfg->pad_token_id, 0, cfg->forced_bos_token_id);
            CUDA_CHECK(cudaGetLastError());
            return;
        }
        const int skip = fb ? 1 : 0;                                            // :71
        if (t - skip == 1) {                                                    // :73-77
            if (!occ_d) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
            apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, occ_d, W, 1, nullptr, cfg->eos_token_id,
                                                   cfg->pad_token_id, cfg->always_allow_eos, -1);
            CUDA_CHECK(cudaGetLastError());
            return;
        }
        // scratch: lo, hi (u64), rule (u8), masks — stream-ordered allocation, no host sync
        uint64_t* lo = nullptr; uint64_t* hi = nullptr; uint8_t* rule = nullptr; uint32_t* masks = nullptr; uint64_t* fsyms = nullptr;
        // stream-ordered frees on EVERY exit path (an ApiError / CUDA_CHECK below must not leak the scratch)
        struct Scratch { void** p[5]; cudaStream_t s; ~Scratch() { for (void** q : p) if (*q) cudaFreeAsync(*q, s); } }
            guard{{(void**)&lo, (void**)&hi, (void**)&rule, (void**)&masks, (void**)&fsyms}, s};
        CUDA_CHECK(cudaMallocAsync(&lo, R * 8, s)); CUDA_CHECK(cudaMallocAsync(&hi, R * 8, s));
        CUDA_CHECK(cudaMallocAsync(&rule, R, s)); CUDA_CHECK(cudaMallocAsync(&masks, (size_t)R * W * 4, s));
        const int nf = cfg->n_force_decoding_from;
        if (nf > 0) {
            std::vector<uint64_t> f(nf);
            for (int i = 0; i < nf; ++i) f[i] = (uint64_t)cfg->force_decoding_from[i] + cfg->shift;
            CUDA_CHECK(cudaMallocAsync(&fsyms, nf * 8, s));
            CUDA_CHECK(cudaMemcpyAsync(fsyms, f.data(), nf * 8, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaStreamSynchronize(s));   // f is a stack temporary
        }
        rows_fold_kernel<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(view, R, (int)t, input_ids_d, skip, cfg->eos_token_id,
                                                                    cfg->pad_token_id, cfg->stop_at_count, fsyms, nf, cfg->shift,
                                                                    lo, hi, rule);
        CUDA_CHECK(cudaGetLastError());
        int rc = sealfm_expand_mask_d(fm, s, R, lo, hi, masks, W, (uint32_t)V, (uint32_t)cfg->shift);
        if (rc) throw ApiError(rc, sealfm_last_error());
        apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, masks, W, 0, rule, cfg->eos_token_id,
                                               cfg->pad_token_id, cfg->always_allow_eos, -1);
        CUDA_CHECK(cudaGetLastError());
    });
}

}  // extern "C"
