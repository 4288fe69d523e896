// T5 building blocks as hand-written CUDA kernels (fp32 arithmetic, matching transformers' eager fp32
// T5ForConditionalGeneration): pre-norm layers with T5LayerNorm (RMS, weight only, variance in fp32), a residual
// stream kept in fp32, relative position biases read from host-computed bucket tables, unscaled attention scores,
// and the gated-GELU (gelu_new) feed-forward.  Cross-attention reuses the BART kernels (bart_kernels.cuh) with the
// query projection pre-multiplied by 8 at load time; the ReLU feed-forward is a GEMM epilogue (wgmma_gemm.cuh).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "bart_kernels.cuh"

namespace sealb200 {

// One CTA of 128 threads per row, d = 4 * n4 <= 512 * NV (each thread holds NV float4 of the row):
//   v = embed[tok[r * tok_stride]]            (tok != nullptr: the embedding; T5 does not scale it)
//   v = x[r] + b[r]                           (otherwise: residual + sub-layer output; b may still be an unsummed
//                                              split-K GEMM output, bsrc, summed here like add_ln_row_kernel does)
// then x[r] = v (the fp32 residual stream) and the operand of the next GEMM, written in split form only:
//   out = (w * (v * rsqrt(mean(v^2) + eps))) * out_scale
// in HF T5LayerNorm's order; out_scale is the decoder's d_model^-0.5 after its final_layer_norm, else 1.
// Instantiated for NV = kT5RmsVec (d <= 1024) and kT5RmsVecWide (d <= 4096, the XL / XXL widths).
constexpr int kT5RmsVec = 2, kT5RmsVecWide = 8;
template <int NV, class SO>
__global__ void __launch_bounds__(128) t5_rms_row_kernel(int64_t rows, int d, const int32_t* __restrict__ tok, int64_t tok_stride,
                                                         const EmbT<SO>* __restrict__ embed, float* __restrict__ x,
                                                         const float* __restrict__ b, SplitSrc bsrc,
                                                         const float* __restrict__ w, float eps, float out_scale, SO so) {
    __shared__ float red[4];
    const int64_t r = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n4 = d / 4;
    const EmbT<SO>* src = tok ? embed + (int64_t)tok[r * tok_stride] * d : nullptr;
    // The wide form moves the row into the x / b / split-K slice pointers (base): indexed by r * d + 4 * c4 in each of
    // its 8 slice loops, ptxas keeps the offset's high word in local memory.  The narrow form keeps base = 0.
    const int64_t base = NV == kT5RmsVec ? 0 : r * d, off = r * d - base;
    SplitSrc bs = bsrc;
    if (bs.ks > 1) bs.part += base;
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c4 = tid + i * 128;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c4 < n4) {
            if (src) v[i] = load_emb4(src + 4 * c4);
            else {
                const float4 a = *reinterpret_cast<const float4*>(x + base + off + 4 * c4);
                const float4 y = load_split4(b + base, bs, off + 4 * c4, 4 * c4);
                v[i] = make_float4(a.x + y.x, a.y + y.y, a.z + y.z, a.w + y.w);
            }
            *reinterpret_cast<float4*>(x + base + off + 4 * c4) = v[i];
            s += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
        }
    }
    s = warp_sum(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    const float rs = rsqrtf(((red[0] + red[1]) + (red[2] + red[3])) / (float)d + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c4 = tid + i * 128;
        if (c4 < n4) {
            const float4 g = *reinterpret_cast<const float4*>(w + 4 * c4);
            float4 o;
            o.x = (g.x * (v[i].x * rs)) * out_scale; o.y = (g.y * (v[i].y * rs)) * out_scale;
            o.z = (g.z * (v[i].z * rs)) * out_scale; o.w = (g.w * (v[i].w * rs)) * out_scale;
            store_split4(so, r * d + 4 * c4, o);
        }
    }
}

// gated-gelu feed-forward: h [rows][2f] = [wi_0 x | wi_1 x] (one GEMM) -> gelu_new(h[:, :f]) * h[:, f:], written as the
// split operand of wo.  gelu_new is HF's NewGELUActivation, the tanh form.
__device__ __forceinline__ float gelu_new_f(float x) {
    return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * (x * x * x))));
}
template <class SO>
__global__ void __launch_bounds__(256) t5_gate_kernel(int64_t rows, int f, const float* __restrict__ h, SO so) {
    const int64_t n4 = rows * (f / 4);
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n4; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / (f / 4);
        const int c = (int)(e % (f / 4)) * 4;
        const float4 a = *reinterpret_cast<const float4*>(h + r * 2 * f + c);
        const float4 g = *reinterpret_cast<const float4*>(h + r * 2 * f + f + c);
        const float4 o = make_float4(gelu_new_f(a.x) * g.x, gelu_new_f(a.y) * g.y, gelu_new_f(a.z) * g.z, gelu_new_f(a.w) * g.w);
        store_split4(so, r * f + c, o);
    }
}

// Relative position bias of head h at distance `dist` (key - query) through a bucket table: bucket[dist + off] indexes the
// layer-0 relative_attention_bias [num_buckets][heads] that every layer shares.
struct RelBias {
    const float* table; const int32_t* bucket; int off; int heads;
    __device__ __forceinline__ float operator()(int dist, int h) const { return __ldg(table + (int64_t)__ldg(bucket + dist + off) * heads + h); }
};

// Encoder self-attention with the relative position bias, bidirectional: one CTA per (query, head); the query's n rows
// attend to its n keys (packed: the real tokens, at the indices of the padded row; unpacked: the S padded positions,
// masked keys excluded).  Scores are q.k + bias(key - query), unscaled.  Structure of grouped_attention
// (bart_kernels.cuh): 32-key chunks of K (transposed) and V staged in shared memory once per sweep of NW*MAXP rows,
// online softmax across chunks.
template <int NW, int MAXP, class SO>
__global__ void __launch_bounds__(NW * 32) t5_enc_self_attn_kernel(int64_t Q, int d, int S, const float* __restrict__ qkv,
                                                                   const int32_t* __restrict__ src_mask, RelBias rb,
                                                                   SO so, const int32_t* __restrict__ src_off) {
    __shared__ float Kt[kHeadDim][33];
    __shared__ __align__(16) float Vs[32][kHeadDim];
    __shared__ __align__(16) float q_s[NW * MAXP][kHeadDim];
    __shared__ int32_t valid_s[32];
    const int64_t qi = blockIdx.x;
    const int h = blockIdx.y, head_off = h * kHeadDim;
    const int64_t r0 = src_off ? src_off[qi] : qi * S;
    const int n = src_off ? src_off[qi + 1] - src_off[qi] : S;
    const int32_t* mask = src_off ? nullptr : src_mask + qi * S;
    const float* base = qkv + r0 * 3 * d;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int rbase = 0; rbase < n; rbase += NW * MAXP) {
        float m[MAXP], l[MAXP], ax[MAXP], ay[MAXP];
        bool has[MAXP];
#pragma unroll
        for (int p = 0; p < MAXP; ++p) {
            const int r = rbase + p * NW + warp;
            has[p] = r < n;
            m[p] = -INFINITY; l[p] = 0.f; ax[p] = 0.f; ay[p] = 0.f;
            if (has[p]) {
                const float2 q2 = *reinterpret_cast<const float2*>(base + (int64_t)r * 3 * d + head_off + 2 * lane);
                q_s[warp * MAXP + p][2 * lane] = q2.x; q_s[warp * MAXP + p][2 * lane + 1] = q2.y;
            }
        }
        for (int s0 = 0; s0 < n; s0 += 32) {
            __syncthreads();
            for (int e = threadIdx.x; e < 32 * (kHeadDim / 4); e += blockDim.x) {
                const int s = e / (kHeadDim / 4), i4 = e % (kHeadDim / 4);
                float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
                if (s0 + s < n) {
                    kk = *reinterpret_cast<const float4*>(base + (int64_t)(s0 + s) * 3 * d + d + head_off + 4 * i4);
                    vv = *reinterpret_cast<const float4*>(base + (int64_t)(s0 + s) * 3 * d + 2 * d + head_off + 4 * i4);
                }
                Kt[4 * i4 + 0][s] = kk.x; Kt[4 * i4 + 1][s] = kk.y; Kt[4 * i4 + 2][s] = kk.z; Kt[4 * i4 + 3][s] = kk.w;
                *reinterpret_cast<float4*>(&Vs[s][4 * i4]) = vv;
            }
            if (threadIdx.x < 32) valid_s[threadIdx.x] = (s0 + threadIdx.x < n) && (!mask || mask[s0 + threadIdx.x] != 0);
            __syncthreads();
            const bool ok = valid_s[lane] != 0;
            const int cnt = n - s0 < 32 ? n - s0 : 32;
#pragma unroll
            for (int p = 0; p < MAXP; ++p) {
                if (!has[p]) continue;                         // warp-uniform
                const int r = rbase + p * NW + warp;
                const float* qq = q_s[warp * MAXP + p];
                float sc = -INFINITY;
                if (ok) {
                    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
                    for (int i = 0; i < kHeadDim; i += 4) {
                        c0 = fmaf(qq[i], Kt[i][lane], c0); c1 = fmaf(qq[i + 1], Kt[i + 1][lane], c1);
                        c2 = fmaf(qq[i + 2], Kt[i + 2][lane], c2); c3 = fmaf(qq[i + 3], Kt[i + 3][lane], c3);
                    }
                    sc = ((c0 + c1) + (c2 + c3)) + rb(s0 + lane - r, h);
                }
                const float mn = fmaxf(m[p], warp_max(sc));
                if (mn == -INFINITY) continue;
                const float pr = ok ? expf(sc - mn) : 0.f;
                const float corr = (m[p] == -INFINITY) ? 0.f : expf(m[p] - mn);
                l[p] = l[p] * corr + warp_sum(pr);
                float bx0 = ax[p] * corr, by0 = ay[p] * corr, bx1 = 0.f, by1 = 0.f;
#pragma unroll 8
                for (int j = 0; j < 32; j += 2) {
                    const float p0 = __shfl_sync(0xffffffffu, pr, j), p1 = __shfl_sync(0xffffffffu, pr, j + 1);
                    if (j < cnt) {
                        const float2 v0 = *reinterpret_cast<const float2*>(&Vs[j][2 * lane]);
                        const float2 v1 = *reinterpret_cast<const float2*>(&Vs[j + 1][2 * lane]);
                        bx0 = fmaf(p0, v0.x, bx0); by0 = fmaf(p0, v0.y, by0);
                        bx1 = fmaf(p1, v1.x, bx1); by1 = fmaf(p1, v1.y, by1);
                    }
                }
                ax[p] = bx0 + bx1; ay[p] = by0 + by1;
                m[p] = mn;
            }
        }
#pragma unroll
        for (int p = 0; p < MAXP; ++p) {
            const int r = rbase + p * NW + warp;
            if (has[p]) store_split2(so, (r0 + r) * d + head_off + 2 * lane, make_float2(ax[p] / l[p], ay[p] / l[p]));
        }
        __syncthreads();
    }
}

// Decoder self-attention with the relative position bias, unidirectional, for the new token of every row at position
// cur_pos: key s < cur_pos is read from the cache row anc[r][s] (beam ancestry, as dec_self_attn_kernel), key cur_pos
// from this step's qkv; the score is q.k + bias(s - cur_pos), unscaled.  One warp per (row, head), lane = key inside a
// 32-key chunk, chunks merged with an online softmax.  The current k / v are persisted to the cache entries of rows
// r*row_mul .. r*row_mul + bcast - 1 (the compact first step: one row stands for all beams of a query).
template <class SO>
__global__ void __launch_bounds__(512) t5_dec_self_attn_kernel(int64_t R, int d, int heads, int cur_pos, int T,
                                                               const float* __restrict__ qkv, float* kc, float* vc,
                                                               const int32_t* __restrict__ anc, RelBias rb, SO so,
                                                               int row_mul, int bcast) {
    __shared__ __align__(16) float q_s[16][kHeadDim];
    const int64_t r = blockIdx.x, pr = r * row_mul;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t* arow = anc + pr * T;
    const int n_keys = cur_pos + 1;
    for (int h = warp; h < heads; h += blockDim.x >> 5) {
        const int col = h * kHeadDim;
        const float* qp = qkv + r * 3 * d + col;
        const float* kcur = qp + d; const float* vcur = qp + 2 * d;
        float* qs = q_s[warp];
        {
            const float2 q2 = *reinterpret_cast<const float2*>(qp + 2 * lane);
            qs[2 * lane] = q2.x; qs[2 * lane + 1] = q2.y;
        }
        __syncwarp();
        float m = -INFINITY, l = 0.f, ax = 0.f, ay = 0.f;
        for (int s0 = 0; s0 < n_keys; s0 += 32) {
            const int s = s0 + lane;
            const bool ok = s < n_keys;
            float sc = -INFINITY;
            if (ok) {
                const float* kp = s == cur_pos ? kcur : kc + ((int64_t)s * R + arow[s]) * d + col;
                float acc = 0.f;
#pragma unroll
                for (int i = 0; i < kHeadDim / 4; ++i) {
                    const float4 kk = *reinterpret_cast<const float4*>(kp + 4 * i);
                    const float4 qq = *reinterpret_cast<const float4*>(qs + 4 * i);
                    acc = fmaf(qq.x, kk.x, acc); acc = fmaf(qq.y, kk.y, acc); acc = fmaf(qq.z, kk.z, acc); acc = fmaf(qq.w, kk.w, acc);
                }
                sc = acc + rb(s - cur_pos, h);
            }
            const float mn = fmaxf(m, warp_max(sc));
            const float p = ok ? expf(sc - mn) : 0.f;
            const float corr = (m == -INFINITY) ? 0.f : expf(m - mn);
            l = l * corr + warp_sum(p);
            ax *= corr; ay *= corr;
            const int cnt = n_keys - s0 < 32 ? n_keys - s0 : 32;
            for (int j = 0; j < cnt; ++j) {
                const float pj = __shfl_sync(0xffffffffu, p, j);
                const int sj = s0 + j;
                const float* vp = sj == cur_pos ? vcur : vc + ((int64_t)sj * R + arow[sj]) * d + col;
                const float2 vv = *reinterpret_cast<const float2*>(vp + 2 * lane);
                ax = fmaf(pj, vv.x, ax); ay = fmaf(pj, vv.y, ay);
            }
            m = mn;
        }
        store_split2(so, r * d + col + 2 * lane, make_float2(ax / l, ay / l));
        const float2 k2 = *reinterpret_cast<const float2*>(kcur + 2 * lane);
        const float2 v2 = *reinterpret_cast<const float2*>(vcur + 2 * lane);
        for (int b2 = 0; b2 < bcast; ++b2) {
            const int64_t off = ((int64_t)cur_pos * R + pr + b2) * d + col + 2 * lane;
            *reinterpret_cast<float2*>(kc + off) = k2;
            *reinterpret_cast<float2*>(vc + off) = v2;
        }
        __syncwarp();                                          // q_s is rewritten for the next head
    }
}

}  // namespace sealb200
