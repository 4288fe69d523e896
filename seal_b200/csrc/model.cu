// The model handle of the decode library (include/sealdec.h): weight storage and the state-dict slot tables of the BART,
// pre-LayerNorm BART-family and T5 weights, creation, loading and finalize, options and stats, and the workspace.
#include "decode_model.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <string_view>
#include <vector>

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

// fp32 -> bf16 bits, round to nearest even (the weights of a bf16 checkpoint pass through exactly); NaN stays NaN
uint16_t bf16_rne(float x) {
    uint32_t u; std::memcpy(&u, &x, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return (uint16_t)((u >> 16) | 0x40u);
    return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
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

// var == nullptr is bart-large's post-LayerNorm layer
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

namespace sealb200 {

uint64_t g_ws_epoch = 0;

void make_lin(sealbart* m, Lin& l, int out, int in) {
    l.out = out; l.in = in;
    if (bf16_weights(m)) l.w_bf = dalloc_bf16(m, (uint64_t)out * in);
    else l.w = dalloc(m, (uint64_t)out * in);
    l.b = dalloc(m, out);
}

// n host values times scale (a power of two: exact) into device weights: rounded into bf16 (gemm_mode 6's matrices and
// embedding table) or copied as fp32
void upload(void* dst, bool bf16, const float* host, uint64_t n, float scale) {
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

void check_model(const sealbart* m) {
    if (!m) throw ApiError(SEALFM_EINVAL, "null model");
    if (!m->finalized) throw ApiError(SEALFM_EINVAL, "sealbart_finalize not called");
    CUDA_CHECK(cudaSetDevice(m->device));
}

// Returns the number of CUDA devices; none is an error.
int require_device() {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) { cudaGetLastError(); throw ApiError(SEALFM_ENODEVICE, "no CUDA device available"); }
    return count;
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
    m->ex_split.ensure(Tk * D.d * 8); m->eattn_split.ensure(Tk * D.d * 8); m->effn_split.ensure(Tk * D.f * 8);
    m->dx_split.ensure(D.R * D.d * 8); m->dattn_split.ensure(D.R * D.d * 8); m->dffn_split.ensure(D.R * D.f * 8);
    m->err.ensure(16);
}

}  // namespace sealb200

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

int sealbart_create(const sealbart_config_t* cfg, const sealbart_variant_t* variant, int device, sealbart_t** out) {
    return guarded([&] {
        if (!variant) { create_bart(cfg, nullptr, device, out); return; }
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
    const std::string_view n(name);                       // compared inline: no std::string operator== joins the exports
    if (n == "last_used_graph") return m->last_used_graph;
    if (n == "overflow_fallbacks") return m->overflow_fallbacks;
    if (n == "gemm_mode") return m->cfg.gemm_mode;
    if (n == "cached_graphs") return (int64_t)m->graphs.size();
    if (n == "fused_head_steps") return m->fused_head_steps;
    if (n == "topk_cluster_steps") return m->topk_cluster_steps;
    if (n == "last_paths") return m->last_paths;
    if (n == "launches") return m->launches;
    return -1;
}

}  // extern "C"
