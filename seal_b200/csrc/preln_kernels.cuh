// Pre-LayerNorm BART-family building blocks (transformers' eager fp32 Pegasus and mBART): the residual stream stays
// in fp32 and every sub-layer reads LayerNorm(x).  Everything else -- biased projections, the 0.125-scaled attention
// kernels, learned or fixed position tables, exact-erf GELU or ReLU GEMM epilogues, final_logits_bias -- is BART's
// (bart_kernels.cuh, wgmma_gemm.cuh).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "bart_kernels.cuh"

namespace sealb200 {

// The embedding form of preln_row_kernel (tok != nullptr):
//   v = embed[tok[r * tok_stride]] * scale + pos_table[min(p + pos_offset, pos_rows - 1)]
// with p = pos[r] (the encoder's per-row positions) or pos_const (a decoder step), in HF's order: the scaled embedding
// is rounded before the position row is added.  A position past the table reads its last row: the table is never read
// out of bounds (the caller decides whether such a position may occur, see sealdec.h).  ln_g / ln_b: mBART's
// layernorm_embedding, applied to v before it becomes the residual; null for Pegasus.
// E: the table's element type (bf16 in gemm_mode 6).
template <class E>
struct PreLnEmbedT {
    const int32_t* tok = nullptr; int64_t tok_stride = 0;
    const int32_t* pos = nullptr; int pos_const = 0, pos_offset = 0, pos_rows = 1;
    const E* embed = nullptr; float scale = 1.f; const float* pos_table = nullptr;
    const float* ln_g = nullptr; const float* ln_b = nullptr;
};
using PreLnEmbed = PreLnEmbedT<float>;

// Mean and 1 / sqrt(var + 1e-5) of the row a CTA of 128 threads holds as v[0..1] (float4 c4 = tid + 128 i, n4 of
// them), in add_ln_row_kernel's order: the mean, then the biased variance of the centred values, then eps.  red:
// [2][4] shared floats; two calls in a row need no barrier between them (each slot is rewritten only after a
// __syncthreads that follows every read of it).
__device__ __forceinline__ void preln_stats(const float4 (&v)[2], int n4, int d, float (*red)[4], float& mean, float& rstd) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i)
        if (tid + i * 128 < n4) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    s = warp_sum(s);
    if (lane == 0) red[0][warp] = s;
    __syncthreads();
    mean = ((red[0][0] + red[0][1]) + (red[0][2] + red[0][3])) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (tid + i * 128 < n4) {
            const float e0 = v[i].x - mean, e1 = v[i].y - mean, e2 = v[i].z - mean, e3 = v[i].w - mean;
            q += (e0 * e0 + e1 * e1) + (e2 * e2 + e3 * e3);
        }
    }
    q = warp_sum(q);
    if (lane == 0) red[1][warp] = q;
    __syncthreads();
    rstd = rsqrtf(((red[1][0] + red[1][1]) + (red[1][2] + red[1][3])) / (float)d + 1e-5f);
}

// One CTA of 128 threads per row, d = 4 * n4 <= 1024:
//   v = the embedding (em.tok != nullptr, see PreLnEmbed; with em.ln_g, v = LN(v; em.ln_g, em.ln_b))
//   v = x[r] + b[r]        (otherwise: residual + sub-layer output; b may still be an unsummed split-K GEMM output,
//                           bsrc, summed here like add_ln_row_kernel does)
// then x[r] = v (the fp32 residual stream) and the operand of the next GEMM, written in split form only:
//   out = LN(v; gamma, beta)
// gamma / beta: the next sub-layer's norm, or after the last layer the stack's final layer_norm (the encoder's feeds
// the cross-attention K / V projections, the decoder's the lm_head).
template <class SO>
__global__ void __launch_bounds__(128) preln_row_kernel(int64_t rows, int d, PreLnEmbedT<EmbT<SO>> em, float* __restrict__ x,
                                                        const float* __restrict__ b, SplitSrc bsrc,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        SO so) {
    __shared__ float red[2][4];
    const int64_t r = blockIdx.x;
    const int tid = threadIdx.x;
    const int n4 = d / 4;
    const EmbT<SO>* e = nullptr; const float* pe = nullptr;
    if (em.tok) {
        e = em.embed + (int64_t)em.tok[r * em.tok_stride] * d;
        const int p = min((em.pos ? em.pos[r] : em.pos_const) + em.pos_offset, em.pos_rows - 1);
        pe = em.pos_table + (int64_t)p * d;
    }
    float4 v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c4 = tid + i * 128;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c4 < n4) {
            if (e) {
                const float4 a = load_emb4(e + 4 * c4);
                const float4 q = *reinterpret_cast<const float4*>(pe + 4 * c4);
                v[i] = make_float4(__fmul_rn(a.x, em.scale) + q.x, __fmul_rn(a.y, em.scale) + q.y,
                                   __fmul_rn(a.z, em.scale) + q.z, __fmul_rn(a.w, em.scale) + q.w);
            } else {
                const float4 a = *reinterpret_cast<const float4*>(x + r * d + 4 * c4);
                const float4 y = load_split4(b, bsrc, r * d + 4 * c4, 4 * c4);
                v[i] = make_float4(a.x + y.x, a.y + y.y, a.z + y.z, a.w + y.w);
            }
        }
    }
    float mean, rstd;
    if (e && em.ln_g) {
        preln_stats(v, n4, d, red, mean, rstd);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int c4 = tid + i * 128;
            if (c4 < n4) {
                const float4 g = *reinterpret_cast<const float4*>(em.ln_g + 4 * c4);
                const float4 bt = *reinterpret_cast<const float4*>(em.ln_b + 4 * c4);
                v[i].x = (v[i].x - mean) * rstd * g.x + bt.x; v[i].y = (v[i].y - mean) * rstd * g.y + bt.y;
                v[i].z = (v[i].z - mean) * rstd * g.z + bt.z; v[i].w = (v[i].w - mean) * rstd * g.w + bt.w;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c4 = tid + i * 128;
        if (c4 < n4) *reinterpret_cast<float4*>(x + r * d + 4 * c4) = v[i];
    }
    preln_stats(v, n4, d, red, mean, rstd);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c4 = tid + i * 128;
        if (c4 < n4) {
            const float4 g = *reinterpret_cast<const float4*>(gamma + 4 * c4);
            const float4 bt = *reinterpret_cast<const float4*>(beta + 4 * c4);
            float4 o;
            o.x = (v[i].x - mean) * rstd * g.x + bt.x; o.y = (v[i].y - mean) * rstd * g.y + bt.y;
            o.z = (v[i].z - mean) * rstd * g.z + bt.z; o.w = (v[i].w - mean) * rstd * g.w + bt.w;
            store_split4(so, r * d + 4 * c4, o);
        }
    }
}

}  // namespace sealb200
