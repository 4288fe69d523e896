// The model forward of the decode library: the encoder pass and one decoder step of the BART, pre-LayerNorm BART-family
// (Pegasus, mBART) and T5 layers, and the choice of the attention kernel of each block.
#include "decode_model.hpp"
#include "bart_kernels.cuh"
#include "preln_kernels.cuh"
#include "t5_kernels.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>
#include <vector>

namespace {

// The split-K output the last GEMM left unsummed for its consumer (none if it finished itself), handed over once
SplitSrc take_pending(Ctx& cx) {
    const SplitSrc ps = cx.pending;
    cx.pending = SplitSrc{};
    return ps;
}

// The split a producer of activation a writes in format T (bart_kernels.cuh): SplitOut kind 1 / 2 for 3xTF32 / 3xFP16
// (kind 0 if a has no split), SplitBf16 for 3xBF16
template <typename T> auto producer_split(const Act& a, int* overflow) {
    if constexpr (std::is_same<T, __nv_bfloat16>::value) return SplitBf16{a.piece<T>(0), a.piece<T>(1), a.piece<T>(2)};
    else if (!a.p[0]) return SplitOut{};
    else if constexpr (std::is_same<T, float>::value) return SplitOut{a.p[0], a.p[1], 1};
    else return SplitOut{a.p[0], a.p[1], 2, overflow};
}

// f(so) with the split a producer of activation a writes in m's gemm_mode.  The producer kernels are instantiated per
// split type, so f launches kernel<decltype(so)>.
template <typename F> void with_split(const sealbart* m, const Act& a, F&& f) {
    with_format(m->cfg.gemm_mode, [&](auto t) { f(producer_split<decltype(t)>(a, m->ovf)); });
}
// the embedding table a producer with split type SO gathers from
template <class SO> const EmbT<SO>* embed_table(const sealbart* m) {
    if constexpr (std::is_same<SO, SplitBf16>::value) return m->shared_bf;
    else return m->shared;
}

// Split buffer b (and plain, if not null) as an Act in gemm_mode's format from element off on (split_view).  plain is
// null for activations whose producers write the split only.
Act act_view(int gemm_mode, float* plain, const Buf& b, int64_t off = 0) {
    Act a;
    with_format(gemm_mode, [&](auto t) { a = split_view<decltype(t)>(plain, b, off); });
    return a;
}

// ---- producer dispatch -------------------------------------------------------------------------------------------
// The kernels that normalise or gate a row and write the next GEMM's split operand.  The layer loops and
// sealdec_debug_rownorm both go through these launchers; each enqueues one kernel and returns its kPath* bit (0 for
// the BART embedding, which has none).  b_src: the split-K GEMM output b still is, if it was left unsummed.

// BART's embedding + layernorm_embedding: row r = LN(embed[tok[r * tok_stride]] * scale + pos_table[pos(r) + 2]), pos(r) =
// pos[r] or pos_const, the row clamped to the table's pos_rows - 1
template <class SO>
uint32_t launch_embed_ln(cudaStream_t s, int64_t rows, int d, const int32_t* tok, int64_t tok_stride, const int32_t* pos, int pos_const,
                         const EmbT<SO>* embed, float scale, const float* pos_table, int pos_rows, const float* g, const float* beta,
                         float* out, const SO& so) {
    launch_k(embed_ln_kernel<SO>, (unsigned)((rows + 3) / 4), 128, 0, s, rows, d, tok, tok_stride, pos, pos_const, embed, scale, pos_table,
             pos_rows, g, beta, out, so);
    return 0;
}

// BART's post-LN add: out = LN(a + b), a CTA per row up to kAddLnRowMax rows (which also sums a split-K b), else a
// warp per row (the GEMM never defers there)
template <class SO>
uint32_t launch_add_ln(cudaStream_t s, int64_t rows, int d, const float* a, const float* b, const SplitSrc& b_src, const float* g,
                       const float* beta, float* out, const SO& so) {
    if (rows <= kAddLnRowMax) {
        launch_k(add_ln_row_kernel<SO>, (unsigned)rows, 128, 0, s, rows, d, a, b, g, beta, out, so, b_src);
        return kPathAddLnRow;
    }
    launch_k(add_ln_kernel<SO>, (unsigned)((rows + 3) / 4), 128, 0, s, rows, d, a, b, g, beta, out, so);
    return kPathAddLnWarp;
}

// T5's embedding (tok != nullptr) or add, then RMSNorm (t5_kernels.cuh); the wide kernel above d = 1024
template <class SO>
uint32_t launch_t5_rms(cudaStream_t s, int64_t rows, int d, const int32_t* tok, int64_t tok_stride, const EmbT<SO>* embed, float* x,
                       const float* b, const SplitSrc& b_src, const float* w, float eps, float out_scale, const SO& so) {
    const bool wide = d > 4 * 128 * kT5RmsVec;
    launch_k(wide ? t5_rms_row_kernel<kT5RmsVecWide, SO> : t5_rms_row_kernel<kT5RmsVec, SO>, (unsigned)rows, 128, 0, s, rows, d, tok,
             tok_stride, embed, x, b, b_src, w, eps, out_scale, so);
    return wide ? kPathT5RmsWide : kPathT5Rms;
}

// the pre-LayerNorm family's embedding (em.tok != nullptr) or add, then LayerNorm (preln_kernels.cuh)
template <class SO>
uint32_t launch_preln_norm(cudaStream_t s, int64_t rows, int d, const PreLnEmbedT<EmbT<SO>>& em, float* x, const float* b,
                           const SplitSrc& b_src, const float* g, const float* beta, const SO& so) {
    launch_k(preln_row_kernel<SO>, (unsigned)rows, 128, 0, s, rows, d, em, x, b, b_src, g, beta, so);
    return kPathPreLn | (em.tok && em.ln_g ? kPathPreLnEmbedLn : 0u);
}

// T5's gated-gelu: h [rows][2f] -> gelu_new(h[:, :f]) * h[:, f:], a grid-stride loop of at most 8 CTAs per SM
template <class SO> uint32_t launch_t5_gate(cudaStream_t s, int64_t rows, int f, const float* h, const SO& so) {
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((rows * (f / 4) + 255) / 256, (int64_t)sm_count() * 8));
    launch_k(t5_gate_kernel<SO>, (unsigned)blocks, 256, 0, s, rows, f, h, so);
    return kPathT5Gate;
}

void add_ln(Ctx& cx, int64_t rows, int d, const float* a, const float* b, const LNp& ln, const Act& out) {
    const SplitSrc ps = take_pending(cx);
    with_split(cx.m, out, [&](auto so) { cx.m->last_paths |= launch_add_ln(cx.s, rows, d, a, b, ps, ln.g, ln.b, out.x, so); });
    cx.m->launches++;
}

// the BART embedding of rows tok[r * tok_stride] at positions pos[r] or pos_const, through the table pos_table
void embed_ln(Ctx& cx, int64_t rows, int d, const int32_t* tok, int64_t tok_stride, const int32_t* pos, int pos_const,
              const float* pos_table, const LNp& ln, const Act& x) {
    sealbart* m = cx.m;
    const float scale = m->cfg.scale_embedding ? sqrtf((float)d) : 1.0f;
    with_split(m, x, [&](auto so) {
        launch_embed_ln(cx.s, rows, d, tok, tok_stride, pos, pos_const, embed_table<decltype(so)>(m), scale, pos_table,
                        m->cfg.max_positions + 2, ln.g, ln.b, x.x, so);
    });
    m->launches++;
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

// ---- T5 forward --------------------------------------------------------------------------------------
// Pre-norm layers: x (fp32, the residual stream) += sublayer(RMSNorm(x)).  The plain half of the Act x holds the
// residual, its split half the normed operand of the next GEMM: every t5_rms launch adds the previous sublayer's output
// (or gathers the embedding), stores the residual and writes RMSNorm(x) with the next sublayer's weight -- after the
// last layer the stack's final_layer_norm (and, in the decoder, the d_model^-0.5 output scale).
void t5_rms(Ctx& cx, int64_t rows, int d, const int32_t* tok, int64_t tok_stride, const Act& x, const float* b, const float* w,
            float out_scale) {
    const SplitSrc ps = take_pending(cx);
    with_split(cx.m, x, [&](auto so) {
        cx.m->last_paths |= launch_t5_rms(cx.s, rows, d, tok, tok_stride, embed_table<decltype(so)>(cx.m), x.x, b, ps, w,
                                          cx.m->t5.layer_norm_epsilon, out_scale, so);
    });
    cx.m->launches++;
}

// wi (ReLU epilogue) or [wi_0; wi_1] + gate, then wo into tmp (split-K slices left to the next t5_rms)
void t5_ffn(Ctx& cx, int64_t rows, int d, int f, const Act& x, Lin& fc1, Lin& fc2, const Act& ffn, float* ffn2, const Act& tmp) {
    sealbart* m = cx.m;
    if (m->t5.ffn_kind == 1) {
        gemm(cx, rows, 2 * f, d, x, d, fc1, Act{ffn2}, 2 * f, kActNone);
        with_split(m, ffn, [&](auto so) { m->last_paths |= launch_t5_gate(cx.s, rows, f, ffn2, so); });
        m->launches++;
    } else
        gemm(cx, rows, f, d, x, d, fc1, ffn, f, kActRelu);
    gemm(cx, rows, d, f, ffn, f, fc2, tmp, d, kActNone, INT64_MAX);
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
    const size_t saq_smem = self_attn_query_smem(pos + 1, B);
    return !compact && !ragged && pos >= 1 && B >= 2 && B <= 32 && pos + 1 <= 128 && saq_smem <= 112 * 1024;
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
    gemm(cx, S.R, d, d, S.x, d, L.cq, S.cq, d, kActNone, use_cross_attn_small(D.S) ? INT64_MAX : 0);
    const SplitSrc cq_src = take_pending(cx);
    const CrossAttnArgs a{D.grp_start ? D.G : D.Q, d, heads, S.compact ? 1 : D.B, (int)D.S, S.cq.x,
                          m->ckv.as<float>() + (size_t)l * S.Tk * 2 * d + S.ckv_q0, S.m32, D.grp_query, D.grp_start, S.attn.x, S.soff_x};
    with_split(m, S.attn, [&](auto so) { m->last_paths |= launch_cross_attn(cx.s, a, so, cq_src); });
    m->launches++;
    gemm(cx, S.R, d, d, S.attn, d, L.co, S.tmp, d, kActNone, defer_rows);
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
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone, INT64_MAX);
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
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone, INT64_MAX);
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
    embed_ln(cx, Te, d, tok, 1, pos, 0, m->enc_pos, m->enc_ln_emb, A.x);
    for (auto& L : m->enc) {
        gemm(cx, Te, 3 * d, d, A.x, d, L.qkv, A.qkv, 3 * d, kActNone);
        with_split(m, A.attn, [&](auto so) { launch_enc_self_attn(cx.s, D.Q, d, heads, (int)D.S, A.qkv.x, m32, nullptr, A.attn.x, so, soff); });
        m->launches++;
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone, kAddLnRowMax);
        add_ln(cx, Te, d, A.x.x, A.tmp.x, L.ln_attn, A.x);
        gemm(cx, Te, D.f, d, A.x, d, L.fc1, A.ffn, D.f, kActGelu);
        gemm(cx, Te, d, D.f, A.ffn, D.f, L.fc2, A.tmp, d, kActNone, kAddLnRowMax);
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
    gemm(cx, S.R, 3 * d, d, S.x, d, L.qkv, S.qkv, 3 * d, kActNone, use_saq ? INT64_MAX : 0);
    const SplitSrc qkv_src = take_pending(cx);
    const SelfAttnArgs a{D.Q, S.R, S.Rc, D.B, d, heads, pos, D.T, S.row_mul, S.qkv.x, kc, vc, S.anc, S.attn.x};
    with_split(m, S.attn, [&](auto so) { m->last_paths |= launch_bart_self_attn(cx.s, a, use_saq, so, qkv_src); });
    m->launches++;
}

void bart_decoder_layers(Ctx& cx, const Dims& D, const DecStep& S) {
    sealbart* m = cx.m;
    const int d = D.d, pos = S.pos;
    embed_ln(cx, S.R, d, S.tokens + pos, (int64_t)(D.T * S.row_mul), nullptr, pos, m->dec_pos, m->dec_ln_emb, S.x);
    for (int l = 0; l < m->cfg.decoder_layers; ++l) {
        DecLayerW& L = m->dec[l];
        bart_self_attention(cx, D, S, l);
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone, kAddLnRowMax);
        add_ln(cx, S.R, d, S.x.x, S.tmp.x, L.ln_self, S.x);
        cross_attention(cx, D, S, l, kAddLnRowMax);
        add_ln(cx, S.R, d, S.x.x, S.tmp.x, L.ln_cross, S.x);
        gemm(cx, S.R, D.f, d, S.x, d, L.fc1, S.ffn, D.f, kActGelu);
        gemm(cx, S.R, d, D.f, S.ffn, D.f, L.fc2, S.tmp, d, kActNone, kAddLnRowMax);
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
    const SplitSrc ps = take_pending(cx);
    with_split(cx.m, x, [&](auto so) {
        using SO = decltype(so);
        PreLnEmbedT<EmbT<SO>> e;                           // em with the table in the mode's element type
        e.tok = em.tok; e.tok_stride = em.tok_stride; e.pos = em.pos; e.pos_const = em.pos_const; e.pos_offset = em.pos_offset;
        e.pos_rows = em.pos_rows; e.embed = em.tok ? embed_table<SO>(cx.m) : nullptr; e.scale = em.scale; e.pos_table = em.pos_table;
        e.ln_g = em.ln_g; e.ln_b = em.ln_b;
        cx.m->last_paths |= launch_preln_norm(cx.s, rows, d, e, x.x, b, ps, ln.g, ln.b, so);
    });
    cx.m->launches++;
}

// fc1 with the variant's activation epilogue, then fc2 into tmp (split-K slices left to the next preln_norm)
void preln_ffn(Ctx& cx, int64_t rows, const Dims& D, const Act& x, Lin& fc1, Lin& fc2, const Act& ffn, const Act& tmp) {
    const int act = cx.m->variant.activation == SEALBART_ACT_RELU ? kActRelu : kActGelu;
    gemm(cx, rows, D.f, D.d, x, D.d, fc1, ffn, D.f, act);
    gemm(cx, rows, D.d, D.f, ffn, D.f, fc2, tmp, D.d, kActNone, INT64_MAX);
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
        gemm(cx, Te, d, d, A.attn, d, L.o, A.tmp, d, kActNone, INT64_MAX);
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
        gemm(cx, S.R, d, d, S.attn, d, L.o, S.tmp, d, kActNone, INT64_MAX);
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, L.ln_cross);
        cross_attention(cx, D, S, l, INT64_MAX);
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, L.ln_final);
        preln_ffn(cx, S.R, D, S.x, L.fc1, L.fc2, S.ffn, S.tmp);
        preln_norm(cx, S.R, d, PreLnEmbed{}, S.x, S.tmp.x, l + 1 < n ? m->dec[l + 1].ln_self : m->dec_ln_out);
    }
}

}  // namespace

namespace sealb200 {

// src_tokens_hint: >= 0 the caller's count of real source tokens (right-padded masks): no host synchronisation, the
// kernel that derives the offsets checks it and raises err_d[2] on a mismatch; -1 unknown: one 16-byte read-back;
// -2 do not pack (padded rows are computed; also no synchronisation).
void encoder_forward(Ctx& cx, const Dims& D, const int64_t* ids_d, const int64_t* mask_d, int64_t src_tokens_hint,
                     int32_t* hint_err) {
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
    A.x = act_view(gm, m->ex.as<float>(), m->ex_split);
    A.qkv = Act{m->eqkv.as<float>()};
    A.attn = act_view(gm, nullptr, m->eattn_split);
    A.tmp = Act{m->etmp.as<float>()};
    A.ffn = act_view(gm, nullptr, m->effn_split);
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
                  cudaEvent_t ev_layers_done, bool compact, const HeadEpi& head) {
    sealbart* m = cx.m;
    if (compact && (cur_len != 1 || D.grp_start || D.Qb)) throw ApiError(SEALFM_EINVAL, "internal: compact step only at position 0 of a generate");
    const int d = D.d, gm = m->cfg.gemm_mode;
    DecStep S;
    S.x = act_view(gm, m->dx.as<float>(), m->dx_split, D.r0 * d);
    S.qkv = Act{m->dqkv.as<float>() + D.r0 * 3 * d};
    S.attn = act_view(gm, nullptr, m->dattn_split, D.r0 * d);
    S.tmp = Act{m->dtmp.as<float>() + D.r0 * d};
    S.cq = Act{m->dcq.as<float>() + D.r0 * d};
    S.ffn = act_view(gm, nullptr, m->dffn_split, D.r0 * D.f);
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

}  // namespace sealb200

// ---- test hooks ------------------------------------------------------------------------------------------------

extern "C" {

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

        Buf d_in, d_ckv, d_kc, d_vc, d_anc, d_mask, d_off, d_gq, d_gs, d_part, d_pb, d_rel, d_bkt, d_out, d_split, d_ovf;
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
        const size_t out_n = (size_t)rows * d;
        nan(d_out, out_n * 4);
        if (c->out_split) nan(d_split, out_n * 8);
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
        // out_split 1 / 2 / 3: the split of gemm_mode 2 / 3 / 6, laid out as the model's split buffers (split_view)
        uint32_t bit = 0;
        Act split;
        size_t elem = 0;
        if (c->out_split)
            with_format(c->out_split == 1 ? kGemmTf32 : c->out_split == 2 ? kGemmFp16 : kGemmBf16, [&](auto t) {
                using T = decltype(t);
                split = split_view<T>(nullptr, d_split); elem = sizeof(T);
                bit = run(producer_split<T>(split, d_ovf.as<int>()));
            });
        else bit = run(SplitOut{});
        CUDA_CHECK(cudaDeviceSynchronize());
        auto down = [&](void* h, const void* d, size_t bytes) { CUDA_CHECK(cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost)); };
        down(out, d_out.p, out_n * 4);
        void* const split_out[3] = {split1, split2, split3};
        for (int i = 0; i < 3; ++i)
            if (split.p[i]) down(split_out[i], split.p[i], out_n * elem);
        if (overflow) down(overflow, d_ovf.p, 4);
        if (self) { down(kc_out, d_kc.p, cache_bytes); down(vc_out, d_vc.p, cache_bytes); }
        *path = bit;
    });
}

}  // extern "C"

extern "C" {

int sealdec_debug_rownorm(const sealdec_norm_case_t* c, float* out, void* split1, void* split2, void* split3, int32_t* overflow,
                          uint32_t* path) {
    return guarded([&] {
        auto bad = [](const char* what) { return ApiError(SEALFM_EINVAL, what); };
        constexpr int kMaxPos = 1024;                                     // the largest position accepted
        if (!c || !path) throw bad("null argument");
        if (c->kind < 0 || c->kind > 4) throw bad("kind must be 0..4");
        const int kind = c->kind, d = c->d;
        const int64_t rows = c->rows;
        const bool t5 = kind == 2 || kind == 4;
        if (kind == 4 ? (d < 64 || d > 65536 || d % 64) : t5 ? !((d > 0 && d <= 1024 && d % 128 == 0) || (d > 0 && d <= 4096 && d % 1024 == 0))
                                                          : (d < 128 || d > 1024 || d % 128))
            throw bad("d outside the family's widths (BART / pre-LN: multiples of 128 up to 1024; T5: also 2048, 3072, 4096; "
                      "gate: multiples of 64 up to 65536)");
        if (rows < 1 || rows > (1 << 20)) throw bad("rows must be in [1, 2^20]");
        if (c->out_split < 0 || c->out_split > 3) throw bad("out_split must be 0..3");
        if (c->out_split == 0 && kind >= 2) throw bad("kinds 2..4 write the split only: out_split must not be 0");
        if (c->out_split && (!split1 || !split2 || (c->out_split == 3 && !split3) || (c->out_split == 2 && !overflow)))
            throw bad("split output missing");
        if (kind != 4 && !out) throw bad("out missing");
        // the input form: the embedding (kind 0; kinds 2, 3 with tok), the add (kind 1; kinds 2, 3 with a), the gate's h
        const bool emb = kind == 0 || ((kind == 2 || kind == 3) && c->tok);
        const bool add = kind == 1 || ((kind == 2 || kind == 3) && !c->tok);
        if ((kind == 2 || kind == 3) && c->tok && c->a) throw bad("tok and a: one input form only");
        const bool sums = add && (kind != 1 || rows <= kAddLnRowMax);      // the kernels that sum split-K slices
        if (c->split_ks != 0 && c->split_ks != 1) {
            if (c->split_ks < 2 || c->split_ks > 8) throw bad("split_ks must be 2..8");
            if (!sums) throw bad("split-K slices: only for the kernels that sum them");
            if (!c->split_part || !c->split_bias) throw bad("split-K slices or bias missing");
        }
        const bool sliced = c->split_ks > 1;
        if (add && (!c->a || (!sliced && !c->b))) throw bad("a or b missing");
        if (kind == 4 && !c->h) throw bad("h missing");
        if (kind != 4 && !c->gamma) throw bad("gamma missing");
        if ((kind == 0 || kind == 1 || kind == 3) && !c->beta) throw bad("beta missing");
        if (kind == 2 && !(std::isfinite(c->eps) && c->eps >= 0.f && std::isfinite(c->out_scale))) throw bad("eps and out_scale must be finite");
        const bool has_pos = kind == 0 || (kind == 3 && emb);
        const int pos_offset = kind == 0 ? 2 : c->pos_offset;
        if (emb) {
            if (!c->embed || c->V < 1 || c->tok_stride < 1) throw bad("embedding: embed, V >= 1 and tok_stride >= 1 needed");
            for (int64_t r = 0; r < rows; ++r)
                if (c->tok[r * c->tok_stride] < 0 || c->tok[r * c->tok_stride] >= c->V) throw bad("token id outside [0, V)");
        }
        if (has_pos) {
            if (kind == 3 && pos_offset != 0 && pos_offset != 2) throw bad("pos_offset must be 0 or 2");
            if (!c->pos_table || c->pos_rows < pos_offset + 1 || c->pos_rows > kMaxPos + 2) throw bad("pos_table of pos_offset + 1 .. 1026 rows needed");
            for (int64_t r = 0; r < (c->pos ? rows : 1); ++r) {
                const int p = c->pos ? c->pos[r] : c->pos_const;
                if (p < 0 || p > kMaxPos) throw bad("position outside [0, 1024]");
            }
            if (kind == 3 && !c->ln_emb_g != !c->ln_emb_b) throw bad("ln_emb_g and ln_emb_b together");
        }
        require_device();

        Buf d_tok, d_pos, d_emb, d_ptab, d_lg, d_lb, d_a, d_b, d_part, d_pb, d_g, d_beta, d_h, d_out, d_split, d_ovf;
        auto up = [&](Buf& b, const void* h, size_t bytes) { b.ensure(bytes); CUDA_CHECK(cudaMemcpy(b.p, h, bytes, cudaMemcpyHostToDevice)); };
        auto nan = [&](Buf& b, size_t bytes) { b.ensure(bytes); CUDA_CHECK(cudaMemset(b.p, 0xFF, bytes)); };
        const size_t n = (size_t)rows * d;
        if (emb) {
            std::vector<int32_t> tok((size_t)rows);                        // row r's token at r (tok_stride 1 on the device)
            for (int64_t r = 0; r < rows; ++r) tok[r] = c->tok[r * c->tok_stride];
            up(d_tok, tok.data(), tok.size() * 4);
            const size_t ne = (size_t)c->V * d;
            d_emb.ensure(ne * (c->out_split == 3 ? 2 : 4));
            upload(d_emb.p, c->out_split == 3, c->embed, ne);               // bf16 as sealbart_set_tensor rounds it (gemm_mode 6)
        }
        if (has_pos) {
            if (c->pos) up(d_pos, c->pos, (size_t)rows * 4);
            // the table, then NaN guard rows up to row 1026 = the last one an accepted position can name
            const size_t tab = (size_t)c->pos_rows * d * 4, all = (size_t)std::max(c->pos_rows, kMaxPos + 3) * d * 4;
            nan(d_ptab, all);
            CUDA_CHECK(cudaMemcpy(d_ptab.p, c->pos_table, tab, cudaMemcpyHostToDevice));
        }
        if (kind == 3 && emb && c->ln_emb_g) { up(d_lg, c->ln_emb_g, (size_t)d * 4); up(d_lb, c->ln_emb_b, (size_t)d * 4); }
        if (kind != 4) up(d_g, c->gamma, (size_t)d * 4);
        if (kind != 4 && kind != 2) up(d_beta, c->beta, (size_t)d * 4);
        if (kind == 4) up(d_h, c->h, n * 2 * 4);
        // the residual: out for kind 1 (add_ln runs in place, out == a), x_out for kinds 2 and 3; NaN where not an input
        nan(d_out, n * 4);
        if (add) CUDA_CHECK(cudaMemcpy(d_out.p, c->a, n * 4, cudaMemcpyHostToDevice));
        SplitSrc src{};
        if (add) {
            if (sliced) {
                nan(d_b, n * 4);                                          // not read
                up(d_part, c->split_part, n * 4 * c->split_ks); up(d_pb, c->split_bias, (size_t)d * 4);
                src = SplitSrc{d_part.as<float>(), c->split_ks, (int64_t)n, d_pb.as<float>(), c->split_unscale};
            } else up(d_b, c->b, n * 4);
        }
        if (c->out_split) nan(d_split, n * 8);
        d_ovf.ensure(4); CUDA_CHECK(cudaMemset(d_ovf.p, 0, 4));

        float* x = d_out.as<float>();
        const int32_t* tok = d_tok.as<int32_t>();
        const int32_t* pos = c->pos ? d_pos.as<int32_t>() : nullptr;
        auto run = [&](auto so) -> uint32_t {
            using SO = decltype(so);
            const EmbT<SO>* table = d_emb.as<EmbT<SO>>();
            switch (kind) {
            case 0:
                return launch_embed_ln(nullptr, rows, d, tok, 1, pos, c->pos_const, table, c->scale, d_ptab.as<float>(), c->pos_rows,
                                       d_g.as<float>(), d_beta.as<float>(), x, so);
            case 1: return launch_add_ln(nullptr, rows, d, x, d_b.as<float>(), src, d_g.as<float>(), d_beta.as<float>(), x, so);
            case 2:
                return launch_t5_rms(nullptr, rows, d, emb ? tok : nullptr, 1, table, x, d_b.as<float>(), src, d_g.as<float>(), c->eps,
                                     c->out_scale, so);
            case 3: {
                PreLnEmbedT<EmbT<SO>> e;
                if (emb) {
                    e.tok = tok; e.tok_stride = 1; e.pos = pos; e.pos_const = c->pos_const; e.pos_offset = pos_offset;
                    e.pos_rows = c->pos_rows; e.embed = table; e.scale = c->scale; e.pos_table = d_ptab.as<float>();
                    e.ln_g = d_lg.as<float>(); e.ln_b = d_lb.as<float>();
                }
                return launch_preln_norm(nullptr, rows, d, e, x, d_b.as<float>(), src, d_g.as<float>(), d_beta.as<float>(), so);
            }
            default: return launch_t5_gate(nullptr, rows, d, d_h.as<float>(), so);
            }
        };
        // out_split 1 / 2 / 3: the split of gemm_mode 2 / 3 / 6, laid out as the model's split buffers (split_view)
        uint32_t bit = 0;
        Act split;
        size_t elem = 0;
        if (c->out_split)
            with_format(c->out_split == 1 ? kGemmTf32 : c->out_split == 2 ? kGemmFp16 : kGemmBf16, [&](auto t) {
                using T = decltype(t);
                split = split_view<T>(nullptr, d_split); elem = sizeof(T);
                bit = run(producer_split<T>(split, d_ovf.as<int>()));
            });
        else bit = run(SplitOut{});
        CUDA_CHECK(cudaDeviceSynchronize());
        auto down = [&](void* h, const void* dp, size_t bytes) { CUDA_CHECK(cudaMemcpy(h, dp, bytes, cudaMemcpyDeviceToHost)); };
        if (kind != 4) down(out, d_out.p, n * 4);
        void* const split_out[3] = {split1, split2, split3};
        for (int i = 0; i < 3; ++i)
            if (split.p[i]) down(split_out[i], split.p[i], n * elem);
        if (overflow) down(overflow, d_ovf.p, 4);
        *path = bit;
    });
}

}  // extern "C"
