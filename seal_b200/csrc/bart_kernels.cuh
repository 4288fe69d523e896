// BART-large building blocks as hand-written CUDA kernels (fp32 arithmetic, matching the
// reference's eager fp32 forward: transformers BartForConditionalGeneration, call sites
// seal/beam_search.py:231-238,481-483).  Post-LN encoder/decoder layers, learned positions with
// offset 2, layernorm_embedding, exact-erf GELU, tied lm_head + final_logits_bias.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "decode_types.cuh"
#include "launch.cuh"
#include "operand_split.cuh"

namespace sealb200 {

// ---- small helpers -----------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Where a producer writes the operand split its consumer GEMM wants: kind 0 = none, 1 = TF32 (two
// fp32 arrays), 2 = FP16 (two half arrays; saturates at +-65504 and raises *overflow).
struct SplitOut { void* a = nullptr; void* b = nullptr; int kind = 0; int* overflow = nullptr; };

// A GEMM output that may still be in split-K form (SplitSrc, decode_types.cuh), read as the finished value.
__device__ __forceinline__ float4 load_split4(const float* __restrict__ plain, const SplitSrc& ss, int64_t off, int col) {
    if (ss.ks <= 1) return *reinterpret_cast<const float4*>(plain + off);
    float4 y = *reinterpret_cast<const float4*>(ss.part + off);
    for (int sl = 1; sl < ss.ks; ++sl) {
        const float4 p = *reinterpret_cast<const float4*>(ss.part + sl * ss.stride + off);
        y.x += p.x; y.y += p.y; y.z += p.z; y.w += p.w;
    }
    const float4 bb = *reinterpret_cast<const float4*>(ss.bias + col);
    return make_float4(y.x * ss.unscale + bb.x, y.y * ss.unscale + bb.y, y.z * ss.unscale + bb.z, y.w * ss.unscale + bb.w);
}
__device__ __forceinline__ float2 load_split2(const float* __restrict__ plain, const SplitSrc& ss, int64_t off, int col) {
    if (ss.ks <= 1) return *reinterpret_cast<const float2*>(plain + off);
    float2 y = *reinterpret_cast<const float2*>(ss.part + off);
    for (int sl = 1; sl < ss.ks; ++sl) {
        const float2 p = *reinterpret_cast<const float2*>(ss.part + sl * ss.stride + off);
        y.x += p.x; y.y += p.y;
    }
    const float2 bb = *reinterpret_cast<const float2*>(ss.bias + col);
    return make_float2(y.x * ss.unscale + bb.x, y.y * ss.unscale + bb.y);
}

// The producers' split stores (operand_split.cuh): SplitOut kind 1 / 2 stores the 3xTF32 / 3xFP16 pieces, and raises
// *overflow once per store whose values the fp16 split saturated.
template <int V> __device__ __forceinline__ void store_split(const SplitOut& so, int64_t idx, const float (&v)[V]) {
    int ov = 0;
    if (so.kind == 1) {
        float* const s[2] = {static_cast<float*>(so.a), static_cast<float*>(so.b)};
        store_split<float, V>(s, idx, v, ov);
    } else if (so.kind == 2) {
        __half* const s[2] = {static_cast<__half*>(so.a), static_cast<__half*>(so.b)};
        __half q[V][2];
        split_values(v, q, ov);
        if (ov) atomicExch(so.overflow, 1);
        store_pieces(s, idx, q);
    }
}

// The producer split of a gemm_mode 6 model, the three bf16 pieces (operand_split.cuh).  A producer takes this type in
// place of SplitOut (its kernels are instantiated per split type); b1 == nullptr: no split wanted.
struct SplitBf16 { __nv_bfloat16* b1 = nullptr; __nv_bfloat16* b2 = nullptr; __nv_bfloat16* b3 = nullptr; };
template <int V> __device__ __forceinline__ void store_split(const SplitBf16& so, int64_t idx, const float (&v)[V]) {
    if (!so.b1) return;
    __nv_bfloat16* const s[3] = {so.b1, so.b2, so.b3};
    int ov = 0;
    store_split<__nv_bfloat16, V>(s, idx, v, ov);
}
template <class SO> __device__ __forceinline__ void store_split4(const SO& so, int64_t idx, const float4& o) {
    store_split<4>(so, idx, {o.x, o.y, o.z, o.w});
}
template <class SO> __device__ __forceinline__ void store_split2(const SO& so, int64_t idx, const float2& o) {
    store_split<2>(so, idx, {o.x, o.y});
}

// Element type of the token-embedding table a producer with split type SO gathers from: bf16 in gemm_mode 6
template <class SO> struct EmbOf { using type = float; };
template <> struct EmbOf<SplitBf16> { using type = __nv_bfloat16; };
template <class SO> using EmbT = typename EmbOf<SO>::type;
__device__ __forceinline__ float4 load_emb4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load_emb4(const __nv_bfloat16* p) {
    const uint2 u = *reinterpret_cast<const uint2*>(p);
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xFFFF0000u));
}

// LayerNorm of one row held as `per` float4 per lane (d = 128*per), torch semantics:
// biased variance, eps inside the sqrt, fp32.
template <int MAXV, class SO>
__device__ __forceinline__ void warp_layernorm(float4 (&v)[MAXV], int nv, int d, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, float eps, float* __restrict__ out,
                                               const SO& so, int64_t row_off, int lane) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) if (i < nv) s += v[i].x + v[i].y + v[i].z + v[i].w;
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) if (i < nv) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
        q += a * a + b * b + c * c + e * e;
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) if (i < nv) {
        const int col = (i * 32 + lane) * 4;
        const float4 g = *reinterpret_cast<const float4*>(gamma + col);
        const float4 b = *reinterpret_cast<const float4*>(beta + col);
        float4 o;
        o.x = (v[i].x - mean) * rstd * g.x + b.x;
        o.y = (v[i].y - mean) * rstd * g.y + b.y;
        o.z = (v[i].z - mean) * rstd * g.z + b.z;
        o.w = (v[i].w - mean) * rstd * g.w + b.w;
        if (out) *reinterpret_cast<float4*>(out + row_off + col) = o;
        store_split4(so, row_off + col, o);
    }
}

constexpr int kLnMaxVec = 8;     // d_model <= 1024

// out[r] = LN(embed[tok[r]] * scale + pos_table[min(pos(r) + 2, pos_rows - 1)])      (BartEncoder/BartDecoder embedding)
// tok: int32, row r reads tok[r * tok_stride].  pos(r) = pos_const if pos_per_row == nullptr else pos_per_row[r].
// A position past the table of pos_rows rows reads its last row, as preln_row_kernel does (see sealdec.h).
template <class SO>
__global__ void __launch_bounds__(128) embed_ln_kernel(int64_t rows, int d, const int32_t* __restrict__ tok,
                                                       int64_t tok_stride,
                                                       const int32_t* __restrict__ pos_per_row, int pos_const,
                                                       const EmbT<SO>* __restrict__ embed, float scale,
                                                       const float* __restrict__ pos_table, int pos_rows,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       float* __restrict__ out, SO so) {
    const int lane = threadIdx.x & 31;
    const int64_t r = blockIdx.x * 4LL + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int nv = d / 128;
    const EmbT<SO>* e = embed + (int64_t)tok[r * tok_stride] * d;
    const int p = min((pos_per_row ? pos_per_row[r] : pos_const) + 2, pos_rows - 1);
    const float* pe = pos_table + (int64_t)p * d;
    float4 v[kLnMaxVec];
#pragma unroll
    for (int i = 0; i < kLnMaxVec; ++i) if (i < nv) {
        const int col = (i * 32 + lane) * 4;
        const float4 a = load_emb4(e + col);
        const float4 b = *reinterpret_cast<const float4*>(pe + col);
        v[i] = make_float4(a.x * scale + b.x, a.y * scale + b.y, a.z * scale + b.z, a.w * scale + b.w);
    }
    warp_layernorm<kLnMaxVec>(v, nv, d, gamma, beta, 1e-5f, out, so, r * d, lane);
}

// out[r] = LN(a[r] + b[r])     (residual + sub-layer output, post-LN)
// (Folding the split-K finish pass of the preceding GEMM into this kernel was tried: at 300 rows it has 75 CTAs and
// became slower than the two separate kernels -- reverted.)
template <class SO>
__global__ void __launch_bounds__(128) add_ln_kernel(int64_t rows, int d, const float* __restrict__ a,
                                                     const float* __restrict__ b, const float* __restrict__ gamma,
                                                     const float* __restrict__ beta, float* __restrict__ out,
                                                     SO so) {
    const int lane = threadIdx.x & 31;
    const int64_t r = blockIdx.x * 4LL + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int nv = d / 128;
    float4 v[kLnMaxVec];
#pragma unroll
    for (int i = 0; i < kLnMaxVec; ++i) if (i < nv) {
        const int col = (i * 32 + lane) * 4;
        const float4 x = *reinterpret_cast<const float4*>(a + r * d + col);
        const float4 y = *reinterpret_cast<const float4*>(b + r * d + col);
        v[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
    }
    warp_layernorm<kLnMaxVec>(v, nv, d, gamma, beta, 1e-5f, out, so, r * d, lane);
}

// add+LN for SMALL row counts (batch 20: 300 rows): one CTA of 128 threads per row instead of one warp per row, so a row's
// 4 KB are read by 128 threads at once and the kernel is not a chain of 8 dependent 16-byte loads per lane on 75 CTAs
// (312 launches per generate at batch 20).
// bsrc: b may still be the raw split-K output of the preceding GEMM (SplitSrc) -- the finish launch of o / co / fc2 is folded in
// (the same fold into the warp-per-row kernel was slower: 75 CTAs at 300 rows; here a row has its own 128 threads).
template <class SO>
__global__ void __launch_bounds__(128) add_ln_row_kernel(int64_t rows, int d, const float* __restrict__ a,
                                                         const float* __restrict__ b, const float* __restrict__ gamma,
                                                         const float* __restrict__ beta, float* __restrict__ out,
                                                         SO so, SplitSrc bsrc) {
    __shared__ float red[2][4];
    const int64_t r = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n4 = d / 4;                                      // float4 per row (<= 256)
    float4 v[2];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c4 = tid + i * 128;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c4 < n4) {
            const float4 x = *reinterpret_cast<const float4*>(a + r * d + 4 * c4);
            const float4 y = load_split4(b, bsrc, r * d + 4 * c4, 4 * c4);
            v[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
    s = warp_sum(s);
    if (lane == 0) red[0][warp] = s;
    __syncthreads();
    const float mean = ((red[0][0] + red[0][1]) + (red[0][2] + red[0][3])) / (float)d;
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
    const float rstd = rsqrtf(((red[1][0] + red[1][1]) + (red[1][2] + red[1][3])) / (float)d + 1e-5f);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c4 = tid + i * 128;
        if (c4 < n4) {
            const float4 g = *reinterpret_cast<const float4*>(gamma + 4 * c4);
            const float4 bt = *reinterpret_cast<const float4*>(beta + 4 * c4);
            float4 o;
            o.x = (v[i].x - mean) * rstd * g.x + bt.x; o.y = (v[i].y - mean) * rstd * g.y + bt.y;
            o.z = (v[i].z - mean) * rstd * g.z + bt.z; o.w = (v[i].w - mean) * rstd * g.w + bt.w;
            if (out) *reinterpret_cast<float4*>(out + r * d + 4 * c4) = o;
            store_split4(so, r * d + 4 * c4, o);
        }
    }
}

// ---- attention ---------------------------------------------------------------------------------
// One warp per (row, head).  Scores: lane s owns key s (its own 256-byte K row against the query
// staged in shared memory) -> two warp reductions per 32 keys instead of one per key; values: lane l
// owns dims {2l, 2l+1} and accumulates p_s * V[s] with the probabilities broadcast by shuffle.
// fp32 throughout; scores scaled by head_dim^-0.5 = 0.125; chunks of 32 keys merged online.
template <typename KV>
__device__ __forceinline__ float2 warp_attend(const float* __restrict__ q_head, int n_keys, const KV& kv,
                                              float* __restrict__ q_s) {
    const int lane = threadIdx.x & 31;
    {
        const float2 q2 = *reinterpret_cast<const float2*>(q_head + 2 * lane);
        q_s[2 * lane] = q2.x; q_s[2 * lane + 1] = q2.y;
    }
    __syncwarp();
    float m = -INFINITY, l = 0.f, ax = 0.f, ay = 0.f;
    for (int s0 = 0; s0 < n_keys; s0 += 32) {
        const int s = s0 + lane;
        const bool ok = s < n_keys && kv.valid(s);
        float sc = -INFINITY;
        if (ok) {
            const float4* kp = reinterpret_cast<const float4*>(kv.k(s));
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < kHeadDim / 4; ++i) {
                const float4 kk = kp[i];
                const float4 qq = *reinterpret_cast<const float4*>(q_s + 4 * i);
                acc = fmaf(qq.x, kk.x, acc); acc = fmaf(qq.y, kk.y, acc); acc = fmaf(qq.z, kk.z, acc); acc = fmaf(qq.w, kk.w, acc);
            }
            sc = acc * 0.125f;
        }
        const float mn = fmaxf(m, warp_max(sc));
        if (mn == -INFINITY) continue;                         // every key so far is masked (warp-uniform)
        const float p = ok ? expf(sc - mn) : 0.f;
        const float corr = (m == -INFINITY) ? 0.f : expf(m - mn);
        l = l * corr + warp_sum(p);
        ax *= corr; ay *= corr;
        const int cnt = n_keys - s0 < 32 ? n_keys - s0 : 32;
        for (int j = 0; j < cnt; ++j) {
            const float pj = __shfl_sync(0xffffffffu, p, j);
            if (pj != 0.f) {                                   // warp-uniform
                const float2 vv = *reinterpret_cast<const float2*>(kv.v(s0 + j) + 2 * lane);
                ax = fmaf(pj, vv.x, ax); ay = fmaf(pj, vv.y, ay);
            }
        }
        m = mn;
    }
    __syncwarp();
    return make_float2(ax / l, ay / l);
}

template <class SO>
__device__ __forceinline__ void store_attn(float2 o, int64_t idx, float* __restrict__ out, const SO& so) {
    if (out) *reinterpret_cast<float2*>(out + idx) = o;
    store_split2(so, idx, o);
}

// Decoder self-attention for one new token per row with beam-ancestry indirection instead of a
// cache reorder (the reference index_selects 24 cache tensors per step, seal/beam_search.py:331-332).
// qkv: [R][3d] (q | k | v) of the current position; kc/vc: [T][R][d] per layer; anc: [R][T] source row
// of every earlier position.  One warp per (row, head), split into 4 groups of 8 lanes: a group owns
// one key at a time and each of its lanes 8 of the 64 head dims, so four K (then V) rows stream
// concurrently with two 16-byte loads per lane — the key count here is tiny (<= max_length), so
// lane-per-key would leave most lanes idle.  The current position's k/v are taken from qkv (and
// written to the cache for the later steps).
template <int ROUNDS>
__device__ __forceinline__ void self_attend_head(const float* __restrict__ qp, const float* __restrict__ kc,
                                                 const float* __restrict__ vc, const int32_t* __restrict__ arow,
                                                 int64_t R, int d, int col, int cur_pos, int n_keys, int g,
                                                 float4& o0, float4& o1) {
    const float4 q0 = __ldg(reinterpret_cast<const float4*>(qp)), q1 = __ldg(reinterpret_cast<const float4*>(qp + 4));
    const float* kcur = qp + d; const float* vcur = qp + 2 * d;
    // issue every K and V load of this (row, head) before any arithmetic: the rows come from HBM
    // (the KV cache is 14 GB at R = 15 000) and nothing below depends on more than registers
    float4 kf[ROUNDS][2], vf[ROUNDS][2];
#pragma unroll
    for (int rd = 0; rd < ROUNDS; ++rd) {
        const int s = rd * 4 + g;
        if (s < n_keys) {
            const int64_t off = (s == cur_pos) ? 0 : ((int64_t)s * R + arow[s]) * d + col;
            const float* kp = (s == cur_pos) ? kcur : kc + off;
            const float* vp = (s == cur_pos) ? vcur : vc + off;
            kf[rd][0] = __ldg(reinterpret_cast<const float4*>(kp)); kf[rd][1] = __ldg(reinterpret_cast<const float4*>(kp + 4));
            vf[rd][0] = __ldg(reinterpret_cast<const float4*>(vp)); vf[rd][1] = __ldg(reinterpret_cast<const float4*>(vp + 4));
        }
    }
    float sc[ROUNDS];
    float mloc = -INFINITY;
#pragma unroll
    for (int rd = 0; rd < ROUNDS; ++rd) {
        const int s = rd * 4 + g;
        sc[rd] = -INFINITY;
        if (rd * 4 < n_keys) {                                 // warp-uniform
            float part = 0.f;
            if (s < n_keys) {
                const float4 k0 = kf[rd][0], k1 = kf[rd][1];
                part = q0.x * k0.x + q0.y * k0.y + q0.z * k0.z + q0.w * k0.w + q1.x * k1.x + q1.y * k1.y + q1.z * k1.z + q1.w * k1.w;
            }
            part += __shfl_xor_sync(0xffffffffu, part, 1);
            part += __shfl_xor_sync(0xffffffffu, part, 2);
            part += __shfl_xor_sync(0xffffffffu, part, 4);
            if (s < n_keys) { sc[rd] = part * 0.125f; mloc = fmaxf(mloc, sc[rd]); }
        }
    }
    mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 8));
    mloc = fmaxf(mloc, __shfl_xor_sync(0xffffffffu, mloc, 16));
    float lsum = 0.f;
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
#pragma unroll
    for (int rd = 0; rd < ROUNDS; ++rd) {
        const int s = rd * 4 + g;
        if (rd * 4 < n_keys && s < n_keys) {
            const float p = expf(sc[rd] - mloc);
            lsum += p;
            const float4 v0 = vf[rd][0], v1 = vf[rd][1];
            a0.x = fmaf(p, v0.x, a0.x); a0.y = fmaf(p, v0.y, a0.y); a0.z = fmaf(p, v0.z, a0.z); a0.w = fmaf(p, v0.w, a0.w);
            a1.x = fmaf(p, v1.x, a1.x); a1.y = fmaf(p, v1.y, a1.y); a1.z = fmaf(p, v1.z, a1.z); a1.w = fmaf(p, v1.w, a1.w);
        }
    }
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {                        // sum the four key groups
        lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        a0.x += __shfl_xor_sync(0xffffffffu, a0.x, o); a0.y += __shfl_xor_sync(0xffffffffu, a0.y, o);
        a0.z += __shfl_xor_sync(0xffffffffu, a0.z, o); a0.w += __shfl_xor_sync(0xffffffffu, a0.w, o);
        a1.x += __shfl_xor_sync(0xffffffffu, a1.x, o); a1.y += __shfl_xor_sync(0xffffffffu, a1.y, o);
        a1.z += __shfl_xor_sync(0xffffffffu, a1.z, o); a1.w += __shfl_xor_sync(0xffffffffu, a1.w, o);
    }
    const float inv = 1.0f / lsum;
    o0 = make_float4(a0.x * inv, a0.y * inv, a0.z * inv, a0.w * inv);
    o1 = make_float4(a1.x * inv, a1.y * inv, a1.z * inv, a1.w * inv);
}

template <int ROUNDS, class SO>
__global__ void __launch_bounds__(512, ROUNDS <= 3 ? 2 : 1) dec_self_attn_kernel(int64_t R, int d, int heads, int cur_pos, int T,
                                                               const float* __restrict__ qkv, float* kc, float* vc,
                                                               const int32_t* __restrict__ anc,
                                                               float* __restrict__ out, SO so, int row_mul, int bcast) {
    // row_mul / bcast: at the first decode step all beams of a query are the same row (same start token, same
    // source), so the step runs on one row per query: compact row r stands for physical rows r*row_mul ..
    // r*row_mul + bcast - 1, whose cache entries all receive this row's k / v (any of them may become the
    // ancestor of a later beam).  Every other step: row_mul = bcast = 1.
    const int64_t r = blockIdx.x;
    const int64_t pr = r * row_mul;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 3, i8 = (lane & 7) * 8;
    const int n_keys = cur_pos + 1;                            // <= 32
    const int32_t* arow = anc + pr * T;
    for (int h = warp; h < heads; h += blockDim.x >> 5) {
        const int col = h * kHeadDim + i8;
        const float* qp = qkv + r * 3 * d + col;
        float4 o0, o1;
        // rows read from the cache are never the row written below (position cur_pos), so the
        // read-only path is safe
        self_attend_head<ROUNDS>(qp, kc, vc, arow, R, d, col, cur_pos, n_keys, g, o0, o1);
        if (g == 0) {
            const int64_t idx = r * d + col;
            if (out) { *reinterpret_cast<float4*>(out + idx) = o0; *reinterpret_cast<float4*>(out + idx + 4) = o1; }
            store_split4(so, idx, o0); store_split4(so, idx + 4, o1);
            // persist this position's k, v for the later steps
            const float* kcur = qp + d; const float* vcur = qp + 2 * d;
            const float4 k0 = __ldg(reinterpret_cast<const float4*>(kcur)), k1 = __ldg(reinterpret_cast<const float4*>(kcur + 4));
            const float4 v0 = __ldg(reinterpret_cast<const float4*>(vcur)), v1 = __ldg(reinterpret_cast<const float4*>(vcur + 4));
            for (int b2 = 0; b2 < bcast; ++b2) {
                float* kd = kc + ((int64_t)cur_pos * R + pr + b2) * d + col; float* vd = vc + ((int64_t)cur_pos * R + pr + b2) * d + col;
                *reinterpret_cast<float4*>(kd) = k0; *reinterpret_cast<float4*>(kd + 4) = k1;
                *reinterpret_cast<float4*>(vd) = v0; *reinterpret_cast<float4*>(vd + 4) = v1;
            }
        }
    }
}

// Decoder self-attention with the beams of a query processed TOGETHER (round 2).  The beams of a query share most of
// their ancestors -- at position s the B rows point at only a few distinct cache rows -- but dec_self_attn_kernel gives
// every row its own CTA and re-reads a shared ancestor's K / V once per beam (through L2; 1.36x the byte floor, and
// bound by the number of L2 requests rather than by HBM).  Here one CTA per (query, head) first de-duplicates the
// ancestor indices per position with warp match/ballot, stages each DISTINCT K / V head row (64 floats) once in shared
// memory, then warp b attends for beam b out of shared memory.  Same arithmetic order per row as the other kernels is
// not required (scores are summed per key in the same k order; softmax is the online form).
// grid (Q, heads), block 32 * B threads, dynamic smem self_attn_query_smem(P, B).
__host__ __device__ inline size_t self_attn_query_smem(int P, int B) { return (size_t)2 * P * B * kHeadDim * 4 + (size_t)2 * P * 32 * 4 + 128 * 4; }

template <class SO>
__global__ void __launch_bounds__(1024) dec_self_attn_query_kernel(int64_t R, int B, int d, int cur_pos, int T,
                                                                  const float* __restrict__ qkv, float* kc, float* vc,
                                                                  const int32_t* __restrict__ anc,
                                                                  float* __restrict__ out, SO so, SplitSrc qsrc) {
    extern __shared__ __align__(16) unsigned char sa_smem[];
    const int P = cur_pos + 1;
    float* Ks = reinterpret_cast<float*>(sa_smem);                       // [P][B][64]
    float* Vs = Ks + (size_t)P * B * kHeadDim;
    int32_t* row_of = reinterpret_cast<int32_t*>(Vs + (size_t)P * B * kHeadDim);   // [P][32] cache row of slot
    int32_t* slot_of = row_of + P * 32;                                 // [P][32] slot of beam
    int32_t* ucount = slot_of + P * 32;                                 // [P] (<= 128 positions)
    const int64_t qi = blockIdx.x;
    const int col = blockIdx.y * kHeadDim;
    const int64_t r0 = qi * B;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // ---- 1. distinct ancestors per position
    for (int s = warp; s < P; s += B) {
        const bool act = lane < B;
        const unsigned amask = __ballot_sync(0xffffffffu, act);
        if (act) {
            const int a = (s == cur_pos) ? lane : anc[(r0 + lane) * T + s];        // the current position: every beam has its own k / v
            const unsigned same = __match_any_sync(amask, a);
            const int leader = __ffs(same) - 1;
            const unsigned leaders = __ballot_sync(amask, leader == lane);
            slot_of[s * 32 + lane] = __popc(leaders & ((1u << leader) - 1u));
            if (leader == lane) row_of[s * 32 + __popc(leaders & ((1u << lane) - 1u))] = a;
            if (lane == 0) ucount[s] = __popc(leaders);
        }
    }
    __syncthreads();
    // ---- 2. stage the distinct K / V head rows once; persist the current position's k / v
    const int per_pos = B * (kHeadDim / 4);
    for (int e = threadIdx.x; e < P * per_pos; e += blockDim.x) {
        const int s = e / per_pos, rem = e - s * per_pos, slot = rem / (kHeadDim / 4), i4 = rem - slot * (kHeadDim / 4);
        if (slot >= ucount[s]) continue;
        const int a = row_of[s * 32 + slot];
        float4 kk, vv;
        if (s == cur_pos) {
            const int64_t qoff = (r0 + a) * 3 * d + col + 4 * i4;
            kk = load_split4(qkv, qsrc, qoff + d, d + col + 4 * i4); vv = load_split4(qkv, qsrc, qoff + 2 * d, 2 * d + col + 4 * i4);
            const int64_t off = ((int64_t)cur_pos * R + r0 + a) * d + col + 4 * i4;
            *reinterpret_cast<float4*>(kc + off) = kk; *reinterpret_cast<float4*>(vc + off) = vv;
        } else {
            const int64_t off = ((int64_t)s * R + a) * d + col + 4 * i4;
            kk = *reinterpret_cast<const float4*>(kc + off); vv = *reinterpret_cast<const float4*>(vc + off);
        }
        *reinterpret_cast<float4*>(Ks + ((size_t)s * B + slot) * kHeadDim + 4 * i4) = kk;
        *reinterpret_cast<float4*>(Vs + ((size_t)s * B + slot) * kHeadDim + 4 * i4) = vv;
    }
    __syncthreads();
    // ---- 3. warp b = beam b
    if (warp < B) {
        const int64_t r = r0 + warp;
        const float2 q2 = load_split2(qkv, qsrc, r * 3 * d + col + 2 * lane, col + 2 * lane);
        float m = -INFINITY, l = 0.f, ax = 0.f, ay = 0.f;
        for (int s = 0; s < P; ++s) {
            const int slot = slot_of[s * 32 + warp];
            const float2 k2 = *reinterpret_cast<const float2*>(Ks + ((size_t)s * B + slot) * kHeadDim + 2 * lane);
            const float sc = warp_sum(q2.x * k2.x + q2.y * k2.y) * 0.125f;
            const float mn = fmaxf(m, sc);
            const float corr = (m == -INFINITY) ? 0.f : expf(m - mn);
            const float p = expf(sc - mn);
            const float2 v2 = *reinterpret_cast<const float2*>(Vs + ((size_t)s * B + slot) * kHeadDim + 2 * lane);
            l = l * corr + p;
            ax = fmaf(p, v2.x, ax * corr); ay = fmaf(p, v2.y, ay * corr);
            m = mn;
        }
        store_attn(make_float2(ax / l, ay / l), r * d + col + 2 * lane, out, so);
    }
}

// Decoder self-attention for positions beyond the 32-key register-resident fast path (max_length up to 128,
// README.md:209-216 decodes with max_length = 100): one warp per (row, head), lane = key inside a 32-key chunk,
// chunks merged with the online softmax of warp_attend.  Same ancestry indirection, same cache update.
struct AncestryKV {
    const float* kc; const float* vc; const int32_t* arow; const float* kcur; const float* vcur;
    int64_t R; int d; int col; int cur_pos;
    __device__ __forceinline__ bool valid(int) const { return true; }
    __device__ __forceinline__ const float* k(int s) const { return s == cur_pos ? kcur : kc + ((int64_t)s * R + arow[s]) * d + col; }
    __device__ __forceinline__ const float* v(int s) const { return s == cur_pos ? vcur : vc + ((int64_t)s * R + arow[s]) * d + col; }
};

template <class SO>
__global__ void __launch_bounds__(512) dec_self_attn_long_kernel(int64_t R, int d, int heads, int cur_pos, int T,
                                                                 const float* __restrict__ qkv, float* kc, float* vc,
                                                                 const int32_t* __restrict__ anc,
                                                                 float* __restrict__ out, SO so) {
    __shared__ __align__(16) float q_s[16][kHeadDim];
    const int64_t r = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t* arow = anc + r * T;
    for (int h = warp; h < heads; h += blockDim.x >> 5) {
        const int col = h * kHeadDim;
        const float* qp = qkv + r * 3 * d + col;
        AncestryKV kv{kc, vc, arow, qp + d, qp + 2 * d, R, d, col, cur_pos};
        const float2 o = warp_attend(qp, cur_pos + 1, kv, q_s[warp]);
        store_attn(o, r * d + col + 2 * lane, out, so);
        const float2 k2 = *reinterpret_cast<const float2*>(qp + d + 2 * lane);
        const float2 v2 = *reinterpret_cast<const float2*>(qp + 2 * d + 2 * lane);
        *reinterpret_cast<float2*>(kc + ((int64_t)cur_pos * R + r) * d + col + 2 * lane) = k2;
        *reinterpret_cast<float2*>(vc + ((int64_t)cur_pos * R + r) * d + col + 2 * lane) = v2;
    }
}

// Grouped attention: the `rows` query rows of group g (the beams of one query for cross attention,
// the tokens of one query for the encoder) all attend to the same n_keys keys, so one CTA per
// (group, head) stages each 32-key K/V chunk in shared memory ONCE and every warp reuses it
// (the per-row version re-read K/V from L2 for each of the 15 beams: 3.4 GB per launch at R = 15 000).
// K chunk is stored transposed+padded (lane = key reads conflict-free), V row-major (lane = dims).
struct GroupAddr {
    const float* q; int64_t q_stride;        // query row r of the group: q + r * q_stride (+ head offset)
    const float* k; const float* v; int64_t kv_stride;   // key s: k + s * kv_stride (+ head offset)
    const int32_t* mask;                     // [n_keys], 0 = padded key; nullptr = every key valid (packed sources)
};

template <int NW, int MAXP, class SO>
__device__ __forceinline__ void grouped_attention(const GroupAddr& g, int rows, int n_keys, int head_off, int64_t out_base,
                                                  int64_t out_stride, float* __restrict__ out, const SO& so) {
    __shared__ float Kt[kHeadDim][33];
    __shared__ __align__(16) float Vs[32][kHeadDim];
    __shared__ __align__(16) float q_s[NW * MAXP][kHeadDim];
    __shared__ int32_t valid_s[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int rbase = 0; rbase < rows; rbase += NW * MAXP) {    // a group of NW*MAXP query rows per sweep over the keys
        float m[MAXP], l[MAXP], ax[MAXP], ay[MAXP];
        bool has[MAXP];
#pragma unroll
        for (int p = 0; p < MAXP; ++p) {
            const int r = rbase + p * NW + warp;
            has[p] = r < rows;
            m[p] = -INFINITY; l[p] = 0.f; ax[p] = 0.f; ay[p] = 0.f;
            if (has[p]) {
                const float2 q2 = *reinterpret_cast<const float2*>(g.q + r * g.q_stride + head_off + 2 * lane);
                q_s[warp * MAXP + p][2 * lane] = q2.x; q_s[warp * MAXP + p][2 * lane + 1] = q2.y;
            }
        }
        for (int s0 = 0; s0 < n_keys; s0 += 32) {
            __syncthreads();                                   // previous chunk fully consumed
            for (int e = threadIdx.x; e < 32 * (kHeadDim / 4); e += blockDim.x) {
                const int s = e / (kHeadDim / 4), i4 = e % (kHeadDim / 4);
                float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
                if (s0 + s < n_keys) {
                    kk = *reinterpret_cast<const float4*>(g.k + (int64_t)(s0 + s) * g.kv_stride + head_off + 4 * i4);
                    vv = *reinterpret_cast<const float4*>(g.v + (int64_t)(s0 + s) * g.kv_stride + head_off + 4 * i4);
                }
                Kt[4 * i4 + 0][s] = kk.x; Kt[4 * i4 + 1][s] = kk.y; Kt[4 * i4 + 2][s] = kk.z; Kt[4 * i4 + 3][s] = kk.w;
                *reinterpret_cast<float4*>(&Vs[s][4 * i4]) = vv;
            }
            if (threadIdx.x < 32) valid_s[threadIdx.x] = (s0 + threadIdx.x < n_keys) && (!g.mask || g.mask[s0 + threadIdx.x] != 0);
            __syncthreads();
            const bool ok = valid_s[lane] != 0;
            const int cnt = n_keys - s0 < 32 ? n_keys - s0 : 32;
#pragma unroll
            for (int p = 0; p < MAXP; ++p) {
                if (!has[p]) continue;                         // warp-uniform
                const float* qq = q_s[warp * MAXP + p];
                float sc = -INFINITY;
                if (ok) {
                    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
                    for (int i = 0; i < kHeadDim; i += 4) {
                        c0 = fmaf(qq[i], Kt[i][lane], c0); c1 = fmaf(qq[i + 1], Kt[i + 1][lane], c1);
                        c2 = fmaf(qq[i + 2], Kt[i + 2][lane], c2); c3 = fmaf(qq[i + 3], Kt[i + 3][lane], c3);
                    }
                    sc = ((c0 + c1) + (c2 + c3)) * 0.125f;
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
                    if (j < cnt) {                             // masked / missing keys have p == 0 and zero V rows
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
            if (has[p]) store_attn(make_float2(ax[p] / l[p], ay[p] / l[p]), out_base + r * out_stride + head_off + 2 * lane, out, so);
        }
        __syncthreads();                                       // q_s is rewritten by the next row group
    }
}

constexpr int kGAttnWarps = 8, kGAttnPasses = 2;               // 16 rows per sweep, 256 threads -> 8 CTAs / SM

// Cross attention: q [R][d]; ckv [Q*S][2d] (k | v) of the encoder states.  Group g (one CTA per
// group x head) = the rows that attend to the same source: by default the `beams` rows of query g;
// with grp_query/grp_start (ragged groups, teacher-forced re-scoring) rows grp_start[g]..grp_start[g+1]
// of query grp_query[g].
template <class SO>
__global__ void __launch_bounds__(kGAttnWarps * 32) cross_attn_kernel(int64_t G, int d, int heads, int beams, int S,
                                                         const float* __restrict__ q, const float* __restrict__ ckv,
                                                         const int32_t* __restrict__ src_mask,
                                                         const int32_t* __restrict__ grp_query,
                                                         const int32_t* __restrict__ grp_start, float* __restrict__ out,
                                                         SO so, const int32_t* __restrict__ src_off) {
    // src_off (packed sources): query qi's encoder states are rows src_off[qi] .. src_off[qi+1] of ckv, all valid
    const int64_t gi = blockIdx.x;
    const int h = blockIdx.y;
    const int64_t qi = grp_query ? grp_query[gi] : gi;
    const int64_t row0 = grp_start ? grp_start[gi] : gi * beams;
    const int rows = grp_start ? grp_start[gi + 1] - grp_start[gi] : beams;
    const int64_t k0 = src_off ? src_off[qi] : qi * S;
    const int Sq = src_off ? src_off[qi + 1] - src_off[qi] : S;
    GroupAddr g{q + row0 * d, d, ckv + k0 * 2 * d, ckv + k0 * 2 * d + d, 2 * d, src_off ? nullptr : src_mask + qi * S};
    grouped_attention<kGAttnWarps, kGAttnPasses>(g, rows, Sq, h * kHeadDim, row0 * d, d, out, so);
}

// Cross attention for sources of at most 32 positions (every decode shape of the benchmark: S <= 28): one CTA of
// 128 threads per (group, head) stages K (padded rows: conflict-free 16-byte reads with lane = key), V, and
// blocks of 16 query rows in shared memory; scores are register-tiled 4 rows x 1 key per thread (one K read
// feeds four rows), the softmax runs over the lanes of a warp, and the P.V product is tiled 4 rows x 2 head
// dims per thread.  About half the instructions per (group, head) of grouped_attention, whose one-row-per-warp
// sweep spends two shared-memory reads per FMA.  Same ragged-group arguments as
// cross_attn_kernel.
constexpr int kXKeys = 32, kXRows = 16, kXPad = kHeadDim + 4;
template <class SO>
__global__ void __launch_bounds__(128) cross_attn_small_kernel(int64_t G, int d, int heads, int beams, int S_pad,
                                                               const float* __restrict__ q, const float* __restrict__ ckv,
                                                               const int32_t* __restrict__ src_mask,
                                                               const int32_t* __restrict__ grp_query,
                                                               const int32_t* __restrict__ grp_start, float* __restrict__ out,
                                                               SO so, const int32_t* __restrict__ src_off, SplitSrc qsrc) {
    __shared__ __align__(16) float Ks[kXKeys][kXPad];
    __shared__ __align__(16) float Vs[kXKeys][kHeadDim];
    __shared__ __align__(16) float Qs[kXRows][kHeadDim];
    __shared__ __align__(16) float Ps[kXRows][kXKeys];
    __shared__ float Ls[kXRows];
    const int64_t gi = blockIdx.x;
    const int head_off = blockIdx.y * kHeadDim;
    const int64_t qi = grp_query ? grp_query[gi] : gi;
    const int64_t row0 = grp_start ? grp_start[gi] : gi * beams;
    const int rows = grp_start ? grp_start[gi + 1] - grp_start[gi] : beams;
    // src_off (packed sources): this query's states are rows src_off[qi] .. src_off[qi+1], all valid
    const int S = src_off ? src_off[qi + 1] - src_off[qi] : S_pad;
    const float* kbase = ckv + (src_off ? (int64_t)src_off[qi] : qi * S_pad) * 2 * d + head_off;
    const float* vbase = kbase + d;
    const int tid = threadIdx.x, lane = tid & 31, rg = tid >> 5;
    for (int e = tid; e < kXKeys * (kHeadDim / 4); e += 128) {
        const int sidx = e / (kHeadDim / 4), i4 = e % (kHeadDim / 4);
        float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
        if (sidx < S) {
            kk = *reinterpret_cast<const float4*>(kbase + (int64_t)sidx * 2 * d + 4 * i4);
            vv = *reinterpret_cast<const float4*>(vbase + (int64_t)sidx * 2 * d + 4 * i4);
        }
        *reinterpret_cast<float4*>(&Ks[sidx][4 * i4]) = kk;
        *reinterpret_cast<float4*>(&Vs[sidx][4 * i4]) = vv;        // rows >= S stay zero: their weight is 0, never 0 * garbage
    }
    const bool key_ok = lane < S && (src_off || src_mask[qi * S_pad + lane] != 0);
    for (int rbase = 0; rbase < rows; rbase += kXRows) {
        __syncthreads();                                           // K/V staged; previous block's Qs / Ps consumed
        for (int e = tid; e < kXRows * (kHeadDim / 4); e += 128) {
            const int r = e / (kHeadDim / 4), i4 = e % (kHeadDim / 4);
            float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rbase + r < rows) qq = load_split4(q, qsrc, (row0 + rbase + r) * d + head_off + 4 * i4, head_off + 4 * i4);
            *reinterpret_cast<float4*>(&Qs[r][4 * i4]) = qq;
        }
        __syncthreads();
        // scores: this thread = key `lane` x rows rg*4 .. rg*4+3
        float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i4 = 0; i4 < kHeadDim / 4; ++i4) {
            const float4 kk = *reinterpret_cast<const float4*>(&Ks[lane][4 * i4]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float4 qq = *reinterpret_cast<const float4*>(&Qs[rg * 4 + u][4 * i4]);
                c[u] = fmaf(qq.x, kk.x, c[u]); c[u] = fmaf(qq.y, kk.y, c[u]);
                c[u] = fmaf(qq.z, kk.z, c[u]); c[u] = fmaf(qq.w, kk.w, c[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const float sc = key_ok ? c[u] * 0.125f : -INFINITY;
            const float mx = warp_max(sc);
            const float pr = (key_ok && mx != -INFINITY) ? expf(sc - mx) : 0.f;
            const float sum = warp_sum(pr);
            Ps[rg * 4 + u][lane] = pr;
            if (lane == 0) Ls[rg * 4 + u] = sum;
        }
        __syncthreads();
        // P.V: this thread = head dims 2*lane, 2*lane+1 x rows rg*4 .. rg*4+3
        float ax[4] = {0.f, 0.f, 0.f, 0.f}, ay[4] = {0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < S; j += 4) {                           // rows S..31 of Vs are zero, P there is zero
            float4 pp[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) pp[u] = *reinterpret_cast<const float4*>(&Ps[rg * 4 + u][j]);
            const float2 v0 = *reinterpret_cast<const float2*>(&Vs[j][2 * lane]);
            const float2 v1 = *reinterpret_cast<const float2*>(&Vs[j + 1][2 * lane]);
            const float2 v2 = *reinterpret_cast<const float2*>(&Vs[j + 2][2 * lane]);
            const float2 v3 = *reinterpret_cast<const float2*>(&Vs[j + 3][2 * lane]);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                ax[u] = fmaf(pp[u].x, v0.x, ax[u]); ay[u] = fmaf(pp[u].x, v0.y, ay[u]);
                ax[u] = fmaf(pp[u].y, v1.x, ax[u]); ay[u] = fmaf(pp[u].y, v1.y, ay[u]);
                ax[u] = fmaf(pp[u].z, v2.x, ax[u]); ay[u] = fmaf(pp[u].z, v2.y, ay[u]);
                ax[u] = fmaf(pp[u].w, v3.x, ax[u]); ay[u] = fmaf(pp[u].w, v3.y, ay[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int r = rbase + rg * 4 + u;
            if (r < rows) {
                const float l = Ls[rg * 4 + u];
                store_attn(make_float2(ax[u] / l, ay[u] / l), (row0 + r) * d + head_off + 2 * lane, out, so);
            }
        }
    }
}

// Encoder self attention over the S positions of the same query (bidirectional, key padding mask).
// qkv [Q*S][3d].  grid (Q, heads).
template <class SO>
__global__ void __launch_bounds__(kGAttnWarps * 32) enc_self_attn_kernel(int64_t Q, int d, int heads, int S,
                                                            const float* __restrict__ qkv,
                                                            const int32_t* __restrict__ src_mask,
                                                            float* __restrict__ out, SO so,
                                                            const int32_t* __restrict__ src_off) {
    const int64_t qi = blockIdx.x;
    const int h = blockIdx.y;
    const int64_t r0 = src_off ? src_off[qi] : qi * S;       // packed: only the real tokens of each query are rows
    const int n = src_off ? src_off[qi + 1] - src_off[qi] : S;
    const float* base = qkv + r0 * 3 * d;
    GroupAddr g{base, 3 * d, base + d, base + 2 * d, 3 * d, src_off ? nullptr : src_mask + qi * S};
    grouped_attention<kGAttnWarps, kGAttnPasses>(g, n, n, h * kHeadDim, r0 * d, d, out, so);
}

}  // namespace sealb200
