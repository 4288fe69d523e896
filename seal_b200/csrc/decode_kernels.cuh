// Constrained beam-search step on the device: full-vocabulary log-softmax, HF logits processors,
// FM-index mask and per-row top-(2*beam) (topk_rows_kernel, one CTA per row), then per query the merge,
// BeamSearchScorerWithMemory bookkeeping and LF-mapping of the surviving beams (select_merge_kernel); the
// successor sets of the new beams are expanded by the FM-index kernels (fm_kernels.cu) over all rows.
// Replaces seal/beam_search.py:244-332 + :614-703 and the CPU FM-index work of :62-140 without a single
// host synchronisation.
#pragma once
#include "bart_kernels.cuh"      // warp_sum, warp_max
#include "decode_types.cuh"
#include "fm_device.cuh"
#include "launch.cuh"

#include <cooperative_groups.h>
#include <cfloat>
#include <cstdint>

namespace sealb200 {

constexpr int kSelMaxK = 64;           // 2*num_beams <= 64
constexpr int kSelMaxBeams = 32;

struct StepCfg {
    int32_t num_beams, K;              // K = 2*num_beams
    int32_t V, ld;                     // vocab, logits leading dimension
    int32_t cur_len;                   // tokens per row so far (t); this step picks token t
    int32_t min_length, max_length;
    int32_t eos_token_id, pad_token_id, model_eos_token_id, forced_eos_token_id, forced_bos_token_id;
    int32_t stop_at_count, always_allow_eos, disable_fm_index, remove_invalid_values;
    int32_t shift;
    int32_t T;                         // token row stride (>= max_length)
    int32_t mask_words;                // words per bitmask row
    int32_t first_step_shared_mask;    // 1: every row uses occurring_mask (seal/beam_search.py:73-77)
    int32_t expand_next;               // 0 on the last step
    int32_t logits_shared;             // 1 (first step): one logits row per QUERY, shared by its beams (identical rows)
    int32_t logits_ignored;            // 1: a forcing processor overwrites every score of this step (apply_processors),
                                       //    so the model was not run and `logits` must not be read
    int64_t hyps_per_query;
    int32_t hyp_base;                  // index of this step's first hypothesis record
    int32_t num_groups;                // diverse beam groups G (1: constrained_beam_search; > 1: group_beam_search)
    float diversity_penalty;           // Hamming diversity penalty, 0 = no HammingDiversityLogitsProcessor
    int32_t head_tiles;                // > 0: the lm_head wrote per-(row, n tile) statistics (head_stats, HeadEpi) and the
                                       //    logits only at the row's read set; 0: dense logits, statistics streamed here
    int32_t top_k;                     // TopKLogitsWarper on the raw logits, 1 <= top_k < V; 0 = off (also for top_k >= V)
};

// Whether this step's logits go through the top-k warp: the forcing steps (forced BOS at cur_len 1, the forced-EOS step
// whose logits are ignored) overwrite every score in apply_processors, so the warp cannot change them and is skipped.
__host__ __device__ __forceinline__ bool topk_warp_step(const StepCfg& c) {
    return c.top_k > 0 && !c.logits_ignored && !(c.forced_bos_token_id >= 0 && c.cur_len == 1);
}

struct StepState {
    // per row (R = Q*num_beams), double-buffered by the caller
    const float* beam_scores_in;  float* beam_scores_out;
    const int32_t* tokens_in;     int32_t* tokens_out;        // [R][T]
    const uint64_t* lo_in;        uint64_t* lo_out;           // SA range [lo, hi) of tokens[1:]
    const uint64_t* hi_in;        uint64_t* hi_out;
    const uint64_t* pw_in;        uint64_t* pw_out;           // width of the range before the last token
    const int32_t* anc_in;        int32_t* anc_out;           // [R][T] KV ancestry
    const uint32_t* mask_in;      uint32_t* mask_out;         // [R][mask_words] allowed-token bitmasks
    const uint32_t* occurring_mask;                           // [mask_words]
    const float* logits;                                      // [R][ld]
    const float2* head_stats;                                 // [R][head_tiles] (max, sum exp(x - max)) per lm_head tile
    // hypothesis records
    float* hyp_score; int32_t* hyp_len; int32_t* hyp_tokens; uint8_t* hyp_valid; uint64_t* hyp_lo; uint64_t* hyp_hi;
    int32_t* error_flag;
};

__device__ __forceinline__ float block_reduce_max(float v, float* red) {
    v = warp_max(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = fmaxf(r, red[w]);
    __syncthreads();
    return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r += red[w];
    __syncthreads();
    return r;
}

// HF-4.13 processors applied to a log-probability (SURVEY.md §H3; order MinLength -> ForcedBOS ->
// ForcedEOS -> InfNanRemove), seal/beam_search.py:255.
__device__ __forceinline__ float apply_processors(const StepCfg& c, int v, float p) {
    if (c.min_length > -1 && c.cur_len < c.min_length && v == c.model_eos_token_id) p = -INFINITY;
    if (c.forced_bos_token_id >= 0 && c.cur_len == 1) p = (v == c.forced_bos_token_id) ? 0.f : -INFINITY;
    if (c.forced_eos_token_id >= 0 && c.cur_len == c.max_length - 1) p = (v == c.forced_eos_token_id) ? 0.f : -INFINITY;
    if (c.remove_invalid_values) {
        if (p != p) p = 0.f;
        if (p == INFINITY) p = FLT_MAX;
    }
    return p;
}

// better(a,b): a precedes b in the top-k order — larger score first, lower flat index on ties.
__device__ __forceinline__ bool cand_better(float sa, int ia, float sb, int ib) {
    return sa > sb || (sa == sb && ia < ib);
}

// Candidate staging + running top-K of one CTA of topk_rows_kernel.
template <int BUF>
struct SelSharedT {
    static constexpr int kBuf = BUF;
    float cval[BUF + kSelMaxK];
    int cidx[BUF + kSelMaxK];
    float tval[kSelMaxK];
    int tidx[kSelMaxK];
    float red[32];
    float rv[32]; int ri[32]; int rslot[32];
    int ccount, tcount, overflow;
    float thr; int thr_idx;
};

// Select the best min(K, n) of the n staged candidates (cval/cidx[0..n)) in order; result in
// tval/tidx[0..tcount).  K rounds of block-wide arg-best.
template <typename SH>
__device__ void sel_merge(SH& S, int K) {
    // current top list is appended to the staging area so one pass handles both
    __syncthreads();
    int n = S.ccount;
    for (int i = threadIdx.x; i < S.tcount; i += blockDim.x) { S.cval[n + i] = S.tval[i]; S.cidx[n + i] = S.tidx[i]; }
    __syncthreads();
    n += S.tcount;
    const int want = n < K ? n : K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int round = 0; round < want; ++round) {
        float bv = -INFINITY; int bi = 0x7fffffff; int bs = -1;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int id = S.cidx[i];
            if (id < 0) continue;                        // already taken
            const float v = S.cval[i];
            if (bs < 0 || cand_better(v, id, bv, bi)) { bv = v; bi = id; bs = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            const int os = __shfl_xor_sync(0xffffffffu, bs, o);
            if (os >= 0 && (bs < 0 || cand_better(ov, oi, bv, bi))) { bv = ov; bi = oi; bs = os; }
        }
        if (lane == 0) { S.rv[warp] = bv; S.ri[warp] = bi; S.rslot[warp] = bs; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float v = S.rv[0]; int id = S.ri[0]; int sl = S.rslot[0];
            for (int w = 1; w < nw; ++w)
                if (S.rslot[w] >= 0 && (sl < 0 || cand_better(S.rv[w], S.ri[w], v, id))) { v = S.rv[w]; id = S.ri[w]; sl = S.rslot[w]; }
            S.tval[round] = v; S.tidx[round] = id;
            S.cidx[sl] = -1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        S.tcount = want; S.ccount = 0;
        if (want == K) { S.thr = S.tval[K - 1]; S.thr_idx = S.tidx[K - 1]; }
    }
    __syncthreads();
}

// Per-row scratch between the two kernels of a step.
struct RowScratch {
    float* row_max; float* row_logsum; uint8_t* row_rule;     // [R]  log-softmax statistics / index rule of every row
    float* cand_val; int32_t* cand_idx; int32_t* cand_cnt;    // [Q * lists][K] sorted best candidates per candidate list, [Q * lists]
    float* row_thr;                                           // [logits rows][3] (max, log sum exp over x >= tau, tau) of the
                                                              // top-k warp (topk_threshold_kernel, or topk_threshold_cluster_kernel
                                                              // above kTopkMaxVocab); read on topk_warp_step only
};

// ---- top-k warp (transformers' TopKLogitsWarper before log_softmax, seal/beam_search.py:249-253) ----------------------
// One CTA per logits row: tau = the k-th largest value of the fp32 row (ties at tau kept, -inf entries count as values),
// the exact row max, and log(sum over x >= tau of exp(x - max)).  The row is staged once in shared memory as
// order-preserving uint32 keys (-0.0 canonicalised to +0.0, so that the two compare equal as floats do); the max is the
// largest key, tau comes out of an MSB-first radix select over 4 digits of 8 bits that counts ties, and the sum is taken
// over the staged keys in a fixed order (per thread strided, then the warp tree, then the warps in order).
constexpr int kTopkThreads = 512;
constexpr int kTopkWarps = kTopkThreads / 32;
constexpr int kTopkMaxVocab = 53248;   // V * 4 bytes of keys + the static arrays below fit the 227 KB a CTA can opt into

__device__ __forceinline__ uint32_t float_key(float x) {
    uint32_t u = __float_as_uint(x);
    if (u == 0x80000000u) u = 0u;                                 // -0.0 == +0.0
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// hist[d] += the number of lanes of this warp with digit d; every lane of the warp calls it, d = 256: no count
__device__ __forceinline__ void warp_hist_add(uint32_t* hist, uint32_t d) {
    const unsigned same = __match_any_sync(0xffffffffu, d);
    if (d < 256u && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(&hist[d], (uint32_t)__popc(same));
}

__global__ void __launch_bounds__(kTopkThreads, 1) topk_threshold_kernel(int V, int64_t ld, const float* __restrict__ logits,
                                                                         int top_k, float* __restrict__ row_thr) {
    extern __shared__ __align__(16) uint32_t keys[];
    __shared__ uint32_t hist[kTopkWarps][256];
    __shared__ uint32_t s_max[kTopkWarps];
    __shared__ float red[32];
    __shared__ uint32_t s_prefix, s_rem;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* lp = logits + (int64_t)blockIdx.x * ld;
    const int k = top_k < 1 ? 1 : (top_k > V ? V : top_k);
    for (int i = tid; i < kTopkWarps * 256; i += kTopkThreads) (&hist[0][0])[i] = 0u;
    if (tid == 0) { s_prefix = 0u; s_rem = (uint32_t)k; }
    __syncthreads();
    // Stage the keys, taking the max and the histogram of the top digit in the same pass.  Every loop below runs the
    // same number of iterations in all lanes of a warp (warp_hist_add is a warp-wide operation).
    uint32_t mk = 0u;
    auto stage = [&](int v, float x, bool in) {
        uint32_t d = 256u;
        if (in) {
            const uint32_t key = float_key(x);
            keys[v] = key;
            mk = key > mk ? key : mk;
            d = key >> 24;
        }
        warp_hist_add(hist[warp], d);
    };
    int v0 = 0;
    if ((ld & 3) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
        const int V4 = V >> 2;
        for (int i0 = 0; i0 < V4; i0 += kTopkThreads) {
            const int i = i0 + tid;
            const bool in = i < V4;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in) x = reinterpret_cast<const float4*>(lp)[i];
            const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) stage(4 * i + j, xs[j], in);
        }
        v0 = V4 * 4;
    }
    for (int b = v0; b < V; b += kTopkThreads) stage(b + tid, b + tid < V ? lp[b + tid] : 0.f, b + tid < V);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const uint32_t t = __shfl_xor_sync(0xffffffffu, mk, o); mk = t > mk ? t : mk; }
    if (lane == 0) s_max[warp] = mk;
    __syncthreads();
    uint32_t max_key = s_max[0];
    for (int w = 1; w < kTopkWarps; ++w) max_key = s_max[w] > max_key ? s_max[w] : max_key;
    // Radix select, most significant digit first: with rem = the rank still wanted among the keys matching the prefix,
    // take the digit d where (keys above d) < rem <= (keys above d) + (keys with digit d), and continue with rem minus the
    // keys above d.  Ties at tau are counted, so after the last digit the prefix is the k-th largest key.
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (pass > 0) {
            const uint32_t prefix = s_prefix;
            const uint32_t hmask = 0xffffffffu << (shift + 8);
            for (int b = 0; b < V; b += kTopkThreads) {
                const int v = b + tid;
                uint32_t d = 256u;
                if (v < V) {
                    const uint32_t key = keys[v];
                    if ((key & hmask) == prefix) d = (key >> shift) & 0xffu;
                }
                warp_hist_add(hist[warp], d);
            }
            __syncthreads();
        }
        if (warp == 0) {
            // lane l owns digits 255 - 8l down to 248 - 8l; counts summed over the warp histograms
            uint32_t cnt[8], tot = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int d = 255 - 8 * lane - j;
                uint32_t c = 0;
                for (int w = 0; w < kTopkWarps; ++w) c += hist[w][d];
                cnt[j] = c; tot += c;
            }
            uint32_t incl = tot;                                 // inclusive prefix over the lanes (higher digits first)
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
            const uint32_t rem = s_rem, excl = incl - tot;
            __syncwarp();                                        // every lane has read s_rem before one lane writes it
            if (excl < rem && rem <= incl) {
                uint32_t above = excl;
                int j = 0;
                while (above + cnt[j] < rem) { above += cnt[j]; ++j; }
                s_prefix |= (uint32_t)(255 - 8 * lane - j) << shift;
                s_rem = rem - above;
            }
        }
        __syncthreads();
        for (int i = tid; i < kTopkWarps * 256; i += kTopkThreads) (&hist[0][0])[i] = 0u;
        __syncthreads();
    }
    const uint32_t tau_key = s_prefix;
    const float mx = key_float(max_key);
    float se = 0.f;
    if (mx > -INFINITY)
        for (int v = tid; v < V; v += kTopkThreads) {
            const uint32_t key = keys[v];
            if (key >= tau_key) se += expf(key_float(key) - mx);
        }
    se = block_reduce_sum(se, red);
    if (tid == 0) {
        float* o = row_thr + (int64_t)blockIdx.x * 3;
        o[0] = mx; o[1] = logf(se); o[2] = key_float(tau_key);
    }
}

// Rows of V > kTopkMaxVocab (mT5: 250 112): one cluster of n = ceil(V / kTopkMaxVocab) CTAs per logits row, n <= 8 (the
// portable cluster size), so V <= kTopkClusterMaxVocab.  It returns what topk_threshold_kernel returns.  CTA `rank`
// stages the contiguous slice [rank * chunk, min(V, (rank + 1) * chunk)) of the row, chunk = ceil(V / n) rounded up to
// a multiple of 4 (<= kTopkMaxVocab), as the same keys in its own shared memory; the row is read from HBM once.  Each
// radix pass sums the CTA's warp histograms into tot[pass & 1], and after a cluster barrier every CTA adds the n totals
// over DSMEM and takes the same digit decision from the same integer counts, so no broadcast is needed.  tot is double
// buffered: a CTA overwrites tot[b] two passes after it was read, and every CTA finished that read before the barrier in
// between.  The max is the largest of the n per-CTA maxima.
// Summation order of log sum (fixed, independent of scheduling): each CTA sums its slice as topk_threshold_kernel sums
// a row (per thread strided over ceil(len / 512) keys, the warp's 5-level shuffle tree, the 16 warps in order), then
// rank 0 adds the n CTA sums in rank order, ((s_0 + s_1) + s_2) + ...: at most ceil(chunk / 512) + 5 + 16 + (n - 1)
// additions on any term's path.
constexpr int kTopkClusterMax = 8;
constexpr int kTopkClusterMaxVocab = kTopkClusterMax * kTopkMaxVocab;   // 425 984

__host__ __device__ __forceinline__ int topk_cluster_ctas(int V) { return (V + kTopkMaxVocab - 1) / kTopkMaxVocab; }
__host__ __device__ __forceinline__ int topk_cluster_chunk(int V) {
    const int n = topk_cluster_ctas(V);
    return ((V + n - 1) / n + 3) / 4 * 4;
}

__global__ void __launch_bounds__(kTopkThreads, 1) topk_threshold_cluster_kernel(int V, int64_t ld,
                                                                                 const float* __restrict__ logits,
                                                                                 int top_k, float* __restrict__ row_thr) {
    namespace cg = cooperative_groups;
    extern __shared__ __align__(16) uint32_t keys[];
    __shared__ uint32_t hist[kTopkWarps][256];
    __shared__ uint32_t tot[2][256];
    __shared__ uint32_t s_max[kTopkWarps];
    __shared__ float red[32];
    __shared__ uint32_t s_prefix, s_rem, s_cta_max;
    __shared__ float s_se;
    cg::cluster_group cluster = cg::this_cluster();
    const int n = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int chunk = topk_cluster_chunk(V);
    const int v_begin = rank * chunk < V ? rank * chunk : V;
    const int len = (v_begin + chunk < V ? v_begin + chunk : V) - v_begin;
    const float* lp = logits + (int64_t)(blockIdx.x / n) * ld + v_begin;
    const int k = top_k < 1 ? 1 : (top_k > V ? V : top_k);
    for (int i = tid; i < kTopkWarps * 256; i += kTopkThreads) (&hist[0][0])[i] = 0u;
    if (tid == 0) { s_prefix = 0u; s_rem = (uint32_t)k; }
    __syncthreads();
    uint32_t mk = 0u;
    auto stage = [&](int v, float x, bool in) {
        uint32_t d = 256u;
        if (in) {
            const uint32_t key = float_key(x);
            keys[v] = key;
            mk = key > mk ? key : mk;
            d = key >> 24;
        }
        warp_hist_add(hist[warp], d);
    };
    int v0 = 0;
    if ((ld & 3) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {        // v_begin is a multiple of 4
        const int L4 = len >> 2;
        for (int i0 = 0; i0 < L4; i0 += kTopkThreads) {
            const int i = i0 + tid;
            const bool in = i < L4;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in) x = reinterpret_cast<const float4*>(lp)[i];
            const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) stage(4 * i + j, xs[j], in);
        }
        v0 = L4 * 4;
    }
    for (int b = v0; b < len; b += kTopkThreads) stage(b + tid, b + tid < len ? lp[b + tid] : 0.f, b + tid < len);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const uint32_t t = __shfl_xor_sync(0xffffffffu, mk, o); mk = t > mk ? t : mk; }
    if (lane == 0) s_max[warp] = mk;
    __syncthreads();
    if (tid == 0) {
        uint32_t m = s_max[0];
        for (int w = 1; w < kTopkWarps; ++w) m = s_max[w] > m ? s_max[w] : m;
        s_cta_max = m;
    }
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        if (pass > 0) {
            const uint32_t prefix = s_prefix;
            const uint32_t hmask = 0xffffffffu << (shift + 8);
            for (int b = 0; b < len; b += kTopkThreads) {
                const int v = b + tid;
                uint32_t d = 256u;
                if (v < len) {
                    const uint32_t key = keys[v];
                    if ((key & hmask) == prefix) d = (key >> shift) & 0xffu;
                }
                warp_hist_add(hist[warp], d);
            }
            __syncthreads();
        }
        uint32_t* const my_tot = tot[pass & 1];
        if (tid < 256) {
            uint32_t c = 0;
            for (int w = 0; w < kTopkWarps; ++w) c += hist[w][tid];
            my_tot[tid] = c;
        }
        cluster.sync();                                          // every CTA's totals (and, pass 0, its max) are visible
        if (tid < 256) {                                         // the cluster's count of digit tid, into hist[0]
            uint32_t c = 0;
            for (int r = 0; r < n; ++r) c += cluster.map_shared_rank(my_tot, r)[tid];
            hist[0][tid] = c;
        }
        __syncthreads();
        if (warp == 0) {                                         // the decision of topk_threshold_kernel, same counts
            uint32_t cnt[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { cnt[j] = hist[0][255 - 8 * lane - j]; sum += cnt[j]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
            const uint32_t rem = s_rem, excl = incl - sum;
            __syncwarp();
            if (excl < rem && rem <= incl) {
                uint32_t above = excl;
                int jd = 7;
                bool found = false;
#pragma unroll
                for (int j = 0; j < 8; ++j) {                    // constant indices: cnt stays in registers
                    if (found) continue;
                    if (above + cnt[j] >= rem) { jd = j; found = true; }
                    else above += cnt[j];
                }
                s_prefix |= (uint32_t)(255 - 8 * lane - jd) << shift;
                s_rem = rem - above;
            }
        }
        __syncthreads();
        for (int i = tid; i < kTopkWarps * 256; i += kTopkThreads) (&hist[0][0])[i] = 0u;
        __syncthreads();
    }
    uint32_t max_key = 0u;
    for (int r = 0; r < n; ++r) { const uint32_t m = *cluster.map_shared_rank(&s_cta_max, r); max_key = m > max_key ? m : max_key; }
    const uint32_t tau_key = s_prefix;
    const float mx = key_float(max_key);
    float se = 0.f;
    if (mx > -INFINITY)
        for (int v = tid; v < len; v += kTopkThreads) {
            const uint32_t key = keys[v];
            if (key >= tau_key) se += expf(key_float(key) - mx);
        }
    se = block_reduce_sum(se, red);
    if (tid == 0) s_se = se;
    cluster.sync();                                              // every CTA's sum is visible
    if (rank == 0 && tid == 0) {
        float total = s_se;
        for (int r = 1; r < n; ++r) total += *cluster.map_shared_rank(&s_se, r);
        float* o = row_thr + (int64_t)(blockIdx.x / n) * 3;
        o[0] = mx; o[1] = logf(total); o[2] = key_float(tau_key);
    }
    cluster.sync();                                              // no CTA exits while rank 0 reads its shared memory
}

// ---- step kernel 1 of 2: row statistics + the best K constrained candidates of a run of beams -----------------------
// grid = Q * lists CTAs; list g of query q covers beams [g * rows_per_cta, ...).  After the first step a list is ONE
// row (lists = num_beams): 15 000 CTAs stream the 3 GB of logits in parallel (a CTA per whole query -- 15 rows,
// 3 MB -- stayed far from the byte floor and kept only 20 SMs busy at batch 20).  At the first step a
// list is the whole query (lists = 1): beams 1.. carry -1e9 and are pruned exactly against the running K-th best.
// Full-vocabulary log-softmax (seal/beam_search.py:251), HF processors (:255), FM-index mask (:260-262), top-2B of
// the constrained scores restricted to the list's rows (:302-307) -- exact: the query's top-K is the top-K of its lists' top-Ks.
// Diverse beam groups (num_groups > 1) always use one row per list: see select_merge_kernel for why that is exact.
template <int THREADS, int BUF>
__global__ void __launch_bounds__(THREADS, THREADS >= 512 ? 2 : 4) topk_rows_kernel(StepCfg c, StepState st, RowScratch rs, int lists, int rows_per_cta) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    using SH = SelSharedT<BUF>;
    SH& S = *reinterpret_cast<SH*>(smem_raw);
    const int B = c.num_beams, K = c.K, V = c.V;
    const int64_t qi = blockIdx.x / lists;
    const int g = blockIdx.x - (int)(qi * lists);
    const int64_t r0 = qi * B;
    const int tid = threadIdx.x;
    if (tid == 0) { S.ccount = 0; S.tcount = 0; S.overflow = 0; S.thr = -INFINITY; S.thr_idx = 0x7fffffff; }
    __syncthreads();
    const int b_end = (g + 1) * rows_per_cta < B ? (g + 1) * rows_per_cta : B;
    for (int b = g * rows_per_cta; b < b_end; ++b) {
        const int64_t r = r0 + b;
        const float* lp = st.logits + (c.logits_shared ? qi : r) * c.ld;
        // Exact pruning: every candidate of this row scores <= beam_score (log-probs <= 0, forced tokens
        // add 0).  Once K candidates are held and the row's beam score is below the K-th best, nothing
        // in the row can enter the top-K and no fill-in will be needed -> skip the row entirely,
        // including its 200 KB of logits.  (First step: beams 1..B-1 start at -1e9, :214-216.)
        if (S.tcount == K && st.beam_scores_in[r] < S.thr) continue;
        // ---- full-vocabulary log-softmax statistics (seal/beam_search.py:251), ONE streaming pass:
        // per-thread running (max, sum exp(x - max)), merged across the block.
        float mx = -INFINITY, se = 0.f;
        float tau = -INFINITY;                                   // top-k warp: logits below tau score -inf
        const bool warp_k = topk_warp_step(c);
        if (c.logits_ignored) { mx = 0.f; se = 1.f; }           // log-softmax statistics are never used (uniform branch)
        else if (warp_k) {                                       // statistics of the warped row (topk_threshold_kernel)
            const float* t3 = rs.row_thr + (c.logits_shared ? qi : r) * 3;
            mx = t3[0]; tau = t3[2];
        } else {
        if (c.head_tiles > 0) {                                  // the lm_head's partials, a fixed order per thread
            const float2* ps = st.head_stats + r * c.head_tiles;
            for (int i = tid; i < c.head_tiles; i += THREADS) {
                const float2 p = ps[i];
                if (p.x > mx) { se = se * expf(mx - p.x) + p.y; mx = p.x; }
                else if (p.x > -INFINITY) se += p.y * expf(p.x - mx);
            }
        } else {
        // four 16-byte loads in flight per thread, one running-max update per 16 values
        constexpr int kStride = THREADS * 4;
        int v = tid * 4;
        for (; v + 3 * kStride + 3 < V; v += 4 * kStride) {
            const float4 a = *reinterpret_cast<const float4*>(lp + v);
            const float4 b4 = *reinterpret_cast<const float4*>(lp + v + kStride);
            const float4 c4 = *reinterpret_cast<const float4*>(lp + v + 2 * kStride);
            const float4 d4 = *reinterpret_cast<const float4*>(lp + v + 3 * kStride);
            const float m16 = fmaxf(fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)), fmaxf(fmaxf(b4.x, b4.y), fmaxf(b4.z, b4.w))),
                                    fmaxf(fmaxf(fmaxf(c4.x, c4.y), fmaxf(c4.z, c4.w)), fmaxf(fmaxf(d4.x, d4.y), fmaxf(d4.z, d4.w))));
            if (m16 > mx) { se *= expf(mx - m16); mx = m16; }
            if (mx > -INFINITY) {
                const float s0 = (expf(a.x - mx) + expf(a.y - mx)) + (expf(a.z - mx) + expf(a.w - mx));
                const float s1 = (expf(b4.x - mx) + expf(b4.y - mx)) + (expf(b4.z - mx) + expf(b4.w - mx));
                const float s2 = (expf(c4.x - mx) + expf(c4.y - mx)) + (expf(c4.z - mx) + expf(c4.w - mx));
                const float s3 = (expf(d4.x - mx) + expf(d4.y - mx)) + (expf(d4.z - mx) + expf(d4.w - mx));
                se += (s0 + s1) + (s2 + s3);
            }
        }
        for (; v < V; v += kStride) {
            float x0, x1 = -INFINITY, x2 = -INFINITY, x3 = -INFINITY;
            if (v + 3 < V) {
                const float4 x = *reinterpret_cast<const float4*>(lp + v);
                x0 = x.x; x1 = x.y; x2 = x.z; x3 = x.w;
            } else {
                x0 = lp[v];
                if (v + 1 < V) x1 = lp[v + 1];
                if (v + 2 < V) x2 = lp[v + 2];
            }
            const float m4 = fmaxf(fmaxf(x0, x1), fmaxf(x2, x3));
            if (m4 > mx) { se *= expf(mx - m4); mx = m4; }          // mx = -inf: se is 0, expf(-inf) = 0
            if (mx > -INFINITY) se += expf(x0 - mx) + expf(x1 - mx) + expf(x2 - mx) + expf(x3 - mx);
        }
        }
        {
            const float bm = block_reduce_max(mx, S.red);
            const float scaled = (mx > -INFINITY) ? se * expf(mx - bm) : 0.f;
            se = block_reduce_sum(scaled, S.red);
            mx = bm;
        }
        }
        const float logsum = warp_k ? rs.row_thr[(c.logits_shared ? qi : r) * 3 + 1] : logf(se);
        // ---- which tokens does the index allow on this row (seal/beam_search.py:87-135) ----------
        const int32_t* trow = st.tokens_in + r * c.T;
        const int last = trow[c.cur_len - 1];
        int rule = 0;
        const uint32_t* mrow = c.first_step_shared_mask ? st.occurring_mask : st.mask_in + r * c.mask_words;
        const bool fm_step = !c.disable_fm_index && !(c.forced_bos_token_id >= 0 && c.cur_len == 1);
        // with forced_bos the reference drops the first column before looking at lengths (:66-71)
        const int eff_len = c.cur_len - (c.forced_bos_token_id >= 0 ? 1 : 0);
        if (fm_step && eff_len > 1) {
            const bool ended = (last == c.eos_token_id || last == c.pad_token_id);
            const uint64_t count = ended ? 0 : st.pw_in[r];
            if (c.stop_at_count > 0 && count <= (uint64_t)c.stop_at_count) rule = 1;
            else if (ended) rule = 2;
        }
        if (tid == 0) { rs.row_max[r] = mx; rs.row_logsum[r] = logsum; rs.row_rule[r] = (uint8_t)rule; }
        const float bs = st.beam_scores_in[r];
        // ---- stage candidates whose constrained score is finite and not below the running k-th best.
        // Fast path: one barrier-free sweep over the row's mask words (rows allow a handful of tokens
        // after the first step); if the staging buffer would overflow (first step: ~47 k allowed
        // tokens) the row is redone in bounded sub-rounds with a merge between them.
        auto row_bits = [&](int w) -> uint32_t {
            uint32_t bits;
            if (c.disable_fm_index) bits = 0xffffffffu;
            else if (c.forced_bos_token_id >= 0 && c.cur_len == 1) bits = (c.forced_bos_token_id >> 5) == w ? 1u << (c.forced_bos_token_id & 31) : 0u;
            else if (rule == 1) bits = (c.eos_token_id >> 5) == w ? 1u << (c.eos_token_id & 31) : 0u;
            else if (rule == 2) bits = (c.pad_token_id >> 5) == w ? 1u << (c.pad_token_id & 31) : 0u;
            else bits = mrow[w];
            if (c.always_allow_eos && !c.disable_fm_index && !(c.forced_bos_token_id >= 0 && c.cur_len == 1) &&
                (c.eos_token_id >> 5) == w) bits |= 1u << (c.eos_token_id & 31);
            if (w == c.mask_words - 1 && (V & 31)) bits &= (1u << (V & 31)) - 1;
            return bits;
        };
        auto consider = [&](int v, bool guarded) {
            float p = c.logits_ignored ? 0.f : (lp[v] - mx) - logsum;
            if (warp_k && lp[v] < tau) p = -INFINITY;
            p = apply_processors(c, v, p);
            const float s = p + bs;
            const int flat = b * V + v;
            if (s > -INFINITY && (S.tcount < K || cand_better(s, flat, S.thr, S.thr_idx))) {
                const int slot = atomicAdd(&S.ccount, 1);
                if (!guarded || slot < BUF) { S.cval[slot] = s; S.cidx[slot] = flat; }
                else S.overflow = 1;
            }
        };
        __syncthreads();
        const int count_before = S.ccount;
        for (int w = tid; w < c.mask_words; w += THREADS) {
            uint32_t bits = row_bits(w);
            while (bits) {
                const int bit = __ffs(bits) - 1; bits &= bits - 1;
                consider(w * 32 + bit, true);
            }
        }
        __syncthreads();
        const bool overflow = S.overflow != 0;                   // uniform: read between two barriers
        const int staged_fast = S.ccount;
        __syncthreads();
        if (!overflow) {
            if (staged_fast > BUF / 2) sel_merge(S, K);          // keep room for the next rows
        } else {
            if (tid == 0) { S.ccount = count_before; S.overflow = 0; }
            __syncthreads();
            if (count_before > 0) sel_merge(S, K);
            for (int w0 = 0; w0 < c.mask_words; w0 += THREADS) {
                const int w = w0 + tid;
                const uint32_t bits = w < c.mask_words ? row_bits(w) : 0u;
                for (int sub = 0; sub < 4; ++sub) {
                    uint32_t part = (bits >> (8 * sub)) & 0xffu;
                    while (part) {
                        const int bit = __ffs(part) - 1; part &= part - 1;
                        consider(w * 32 + 8 * sub + bit, false);
                    }
                    __syncthreads();
                    const int staged = S.ccount;                 // read between two barriers:
                    __syncthreads();                             // the branch below is uniform
                    if (staged > BUF - THREADS * 8) sel_merge(S, K);
                }
            }
        }
    }
    sel_merge(S, K);
    static_assert(BUF >= THREADS * 16, "a sub-round stages up to 8 candidates per thread on top of a half-full buffer");
    const int64_t gidx = qi * lists + g;
    for (int k = tid; k < S.tcount; k += THREADS) { rs.cand_val[gidx * K + k] = S.tval[k]; rs.cand_idx[gidx * K + k] = S.tidx[k]; }
    if (tid == 0) rs.cand_cnt[gidx] = S.tcount;
}

constexpr int kMergeThreads = 128;

struct MergeShared {
    float cval[kSelMaxBeams * kSelMaxK];
    int cidx[kSelMaxBeams * kSelMaxK];
    float tval[kSelMaxK];
    int tidx[kSelMaxK];
    uint8_t tvalid[kSelMaxK];
    float rv[kMergeThreads / 32]; int ri[kMergeThreads / 32]; int rslot[kMergeThreads / 32];
    int nbeam_src[kSelMaxBeams];          // candidate index feeding each new beam
    int n_noneos;
    int new_tok[kSelMaxBeams];            // token of every new beam of this step so far (4.13's `current_tokens`)
    int pen_tok[kSelMaxBeams]; int pen_cnt[kSelMaxBeams]; int n_pen;   // (token, count) of the earlier groups' new beams
};

// ---- step kernel 2 of 2, one CTA per query: merge the candidate lists into the top-2B (:302-307), -inf fill-ins
// (SURVEY.md H4), BeamSearchScorerWithMemory.process (:614-703), hypothesis records, and the LF step (incremental
// get_range) of every record and new beam.  The successor sets of the new beams (next step's masks) are expanded by the
// FM-index kernels right after (fm_kernels.cu launch_expand_masks), over all rows of the batch.
//
// Diverse beam groups (c.num_groups = G > 1, transformers 4.13 group_beam_search as fm_index_generate calls it,
// seal/beam_search.py:447-469,523-532): the groups of gs = B / G beams are handled in order, each like a query of its
// own -- top-2gs over its [gs * V] view, process with group_size = gs, 2gs records, gs new beams -- except that
//   * the index mask is an ordinary logits processor there, so the recorded and carried scores are the CONSTRAINED
//     ones: a tie-filled pick scores -inf (and drops out of the reference's output, :555);
//   * HammingDiversityLogitsProcessor runs between the HF processors and the index mask: group g's score of token v is
//     (p - penalty * count(v)) + beam_score, count(v) = how often v is the new token of a beam of groups < g.
// Exactness of the per-row lists (topk_rows_kernel, K = 2B per row): the penalty lowers only tokens earlier groups
// chose, at most (G-1) * gs distinct ones, so a candidate of the group's penalised top-2gs is among its row's
// unpenalised top 2gs + (G-1)gs = B + gs <= 2B.  (A list over several rows would need (G-1)gs more per row.)
// At the first step every group leader is the same row (same logits, start token, mask and score 0), and so is every
// other beam (score -1e9): topk_rows_kernel lists rows 0 and 1 only (lists = 2, or 1 if gs = 1), and here a leader
// takes row 0's list and statistics, a non-leader row 1's -- exactly the per-row lists of all rows, relabelled.
__global__ void __launch_bounds__(kMergeThreads) select_merge_kernel(FmView fm, StepCfg c, StepState st, RowScratch rs, int lists) {
    __shared__ MergeShared S;
    const int B = c.num_beams, K = c.K, V = c.V;
    const int G = c.num_groups, gs = B / G, Kg = 2 * gs;
    const bool grouped = G > 1;
    const int64_t qi = blockIdx.x;
    const int64_t r0 = qi * B;
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    // grouped path: which candidate list / row statistics stand for row b of group [b0, b0 + gs)
    auto src_row = [&](int b, int b0) -> int { return lists == B ? b : (b == b0 ? 0 : 1); };
    const bool warp_k = topk_warp_step(c);
    auto row_logprob = [&](int64_t r, int64_t stat_r, int v) -> float {
        const int64_t lr = c.logits_shared ? qi : r;
        float p = c.logits_ignored ? 0.f : (st.logits[lr * c.ld + v] - rs.row_max[stat_r]) - rs.row_logsum[stat_r];
        if (warp_k && st.logits[lr * c.ld + v] < rs.row_thr[lr * 3 + 2]) p = -INFINITY;    // top-k warp (single group only)
        return apply_processors(c, v, p);
    };
    for (int g = 0; g < G; ++g) {
        const int b0 = g * gs;
        // ---- (token, count) table of the new tokens of groups < g (HammingDiversityLogitsProcessor) ----------------
        if (tid == 0) {
            int np = 0;
            if (c.diversity_penalty > 0.f)
                for (int j = 0; j < b0; ++j) {
                    const int t = S.new_tok[j];
                    if (t < 0) continue;
                    int i = 0;
                    while (i < np && S.pen_tok[i] != t) ++i;
                    if (i == np) { S.pen_tok[np] = t; S.pen_cnt[np] = 0; ++np; }
                    S.pen_cnt[i] += 1;
                }
            S.n_pen = np;
        }
        __syncthreads();
        // ---- gather the candidate lists of the group's rows ----------------------------------------------------------
        int n = 0;
        if (!grouped) {
            for (int l = 0; l < lists; ++l) {
                const int cnt = rs.cand_cnt[qi * lists + l];
                for (int k = tid; k < cnt; k += kMergeThreads) { S.cval[n + k] = rs.cand_val[(qi * lists + l) * K + k]; S.cidx[n + k] = rs.cand_idx[(qi * lists + l) * K + k]; }
                n += cnt;
            }
        } else {
            const int np = S.n_pen;
            for (int b = b0; b < b0 + gs; ++b) {
                const int64_t li = qi * lists + src_row(b, b0);
                const int64_t r = r0 + b, stat_r = r0 + src_row(b, b0);
                const int cnt = rs.cand_cnt[li];
                for (int k = tid; k < cnt; k += kMergeThreads) {
                    const int f = rs.cand_idx[li * K + k];
                    const int v = f - (f / V) * V;
                    float s = rs.cand_val[li * K + k];
                    int count = 0;
                    for (int i = 0; i < np; ++i) count += S.pen_tok[i] == v ? S.pen_cnt[i] : 0;
                    if (count) {
                        // recomputed in the reference's order: (p - penalty * count) + beam_score, no contraction
                        const float p = __fsub_rn(row_logprob(r, stat_r, v), __fmul_rn(c.diversity_penalty, (float)count));
                        s = __fadd_rn(p, st.beam_scores_in[r]);
                    }
                    S.cval[n + k] = s; S.cidx[n + k] = b * V + v;
                }
                n += cnt;
            }
        }
        __syncthreads();
        // ---- top-Kg, score descending then lower flat index -----------------------------------------------------------
        const int want = n < Kg ? n : Kg;
        for (int round = 0; round < want; ++round) {
            float bv = -INFINITY; int bi = 0x7fffffff; int bs = -1;
            for (int i = tid; i < n; i += kMergeThreads) {
                const int id = S.cidx[i];
                if (id < 0) continue;
                const float v = S.cval[i];
                if (bs < 0 || cand_better(v, id, bv, bi)) { bv = v; bi = id; bs = i; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                const int os = __shfl_xor_sync(0xffffffffu, bs, o);
                if (os >= 0 && (bs < 0 || cand_better(ov, oi, bv, bi))) { bv = ov; bi = oi; bs = os; }
            }
            if (lane == 0) { S.rv[warp] = bv; S.ri[warp] = bi; S.rslot[warp] = bs; }
            __syncthreads();
            if (tid == 0) {
                float v = S.rv[0]; int id = S.ri[0]; int sl = S.rslot[0];
                for (int w = 1; w < kMergeThreads / 32; ++w)
                    if (S.rslot[w] >= 0 && (sl < 0 || cand_better(S.rv[w], S.ri[w], v, id))) { v = S.rv[w]; id = S.ri[w]; sl = S.rslot[w]; }
                S.tval[round] = v; S.tidx[round] = id;
                S.cidx[sl] = -1;
            }
            __syncthreads();
        }
        if (tid < kSelMaxK) S.tvalid[tid] = tid < want ? 1 : 0;
        __syncthreads();

        // ---- fewer than Kg finite constrained candidates: fill with masked ones (SURVEY.md §H4) -------
        // torch.topk's choice among -inf ties is unspecified; ours: lowest flat index first.  The single-group path
        // records the unconstrained score of a fill-in (:258,:304-307), the grouped path the constrained one, -inf.
        if (tid == 0 && want < Kg) {                                 // `want` is the same register value in every thread
            int have = want;
            for (int flat = b0 * V; have < Kg && flat < (b0 + gs) * V; ++flat) {
                const int b = flat / V, v = flat - b * V;
                const int64_t r = r0 + b;
                const int64_t stat_r = grouped ? r0 + src_row(b, b0) : r;
                const float s = row_logprob(r, stat_r, v) + st.beam_scores_in[r];
                // was it a finite constrained candidate (then it is already in the list)?
                bool allowed;
                if (c.disable_fm_index) allowed = true;
                else if (c.forced_bos_token_id >= 0 && c.cur_len == 1) allowed = v == c.forced_bos_token_id;
                else {
                    const uint32_t* mrow = c.first_step_shared_mask ? st.occurring_mask : st.mask_in + r * c.mask_words;
                    const int rule = rs.row_rule[stat_r];
                    allowed = rule == 1 ? v == c.eos_token_id : rule == 2 ? v == c.pad_token_id : ((mrow[v >> 5] >> (v & 31)) & 1);
                    if (c.always_allow_eos && v == c.eos_token_id) allowed = true;
                }
                if (allowed && s > -INFINITY) continue;
                S.tval[have] = grouped ? -INFINITY : s; S.tidx[have] = flat; S.tvalid[have] = 0; ++have;
            }
        }
        __syncthreads();

        // ---- BeamSearchScorerWithMemory.process (seal/beam_search.py:642-695), group_size = gs -----------------------
        if (tid == 0) {
            int nb = 0;
            for (int k = 0; k < Kg; ++k) {
                const int tok = S.tidx[k] % V;
                if (tok != c.eos_token_id && nb < gs) S.nbeam_src[nb++] = k;     // :673-681
            }
            S.n_noneos = nb;
            if (nb < gs) atomicExch(st.error_flag, 1);                          // :687-690 ValueError
        }
        __syncthreads();
        const int new_len = c.cur_len + 1;
        if (tid < Kg) {
            const int k = tid;
            const int flat = S.tidx[k];
            const int pb = flat / V, tok = flat - pb * V;                        // :309-310
            const int64_t pr = r0 + pb;
            const int64_t h = qi * c.hyps_per_query + c.hyp_base + 2 * b0 + k;  // group-major, rank order
            st.hyp_score[h] = S.tval[k];                                         // :662-668
            st.hyp_len[h] = new_len;
            st.hyp_valid[h] = S.tvalid[k];
            int32_t* ht = st.hyp_tokens + h * c.T;
            const int32_t* pt = st.tokens_in + pr * c.T;
            for (int i = 0; i < c.cur_len; ++i) ht[i] = pt[i];
            ht[c.cur_len] = tok;
            for (int i = new_len; i < c.T; ++i) ht[i] = c.pad_token_id;
            if (st.hyp_lo) {
                uint64_t l = 0, r = 0;
                if (!c.disable_fm_index && S.tvalid[k] && !(c.forced_bos_token_id >= 0 && c.cur_len == 1)) {
                    uint64_t rr;
                    lf_step(fm, (uint64_t)tok + c.shift, st.lo_in[pr], st.hi_in[pr] - 1, l, rr);
                    r = rr + 1;
                }
                st.hyp_lo[h] = l; st.hyp_hi[h] = r;
            }
        }
        // ---- next beams: state of row b0 + j comes from candidate nbeam_src[j] (threads Kg .. Kg+gs-1: other warps
        // than the record writers where possible) ---------------------------------------------------------------------
        const int jt = tid - (Kg + gs <= kMergeThreads ? Kg : 0);
        if (jt >= 0 && jt < gs) {
            const int j = jt;
            const int64_t nr = r0 + b0 + j;
            if (j < S.n_noneos) {
                const int k = S.nbeam_src[j];
                const int flat = S.tidx[k];
                const int pb = flat / V, tok = flat - pb * V;
                const int64_t pr = r0 + pb;
                S.new_tok[b0 + j] = tok;
                st.beam_scores_out[nr] = S.tval[k];
                const int32_t* pt = st.tokens_in + pr * c.T;
                int32_t* nt = st.tokens_out + nr * c.T;
                for (int i = 0; i < c.cur_len; ++i) nt[i] = pt[i];
                nt[c.cur_len] = tok;
                for (int i = new_len; i < c.T; ++i) nt[i] = c.pad_token_id;
                const int32_t* pa = st.anc_in + pr * c.T;
                int32_t* na = st.anc_out + nr * c.T;
                for (int i = 0; i + 1 < c.cur_len; ++i) na[i] = pa[i];
                na[c.cur_len - 1] = (int32_t)pr;                                // KV of position cur_len-1 lives in the parent's slot
                uint64_t l = 0, rr = 0;
                if (c.forced_bos_token_id >= 0 && c.cur_len == 1) {
                    // the forced BOS is not part of the FM-index query (the reference drops it, :71)
                    l = st.lo_in[pr]; rr = st.hi_in[pr];
                } else if (!c.disable_fm_index) {
                    // incremental get_range: one backward_search_step on the parent's range
                    // (seal/index.py:102-111 recomputed from scratch by the reference, :96-101)
                    lf_step(fm, (uint64_t)tok + c.shift, st.lo_in[pr], st.hi_in[pr] - 1, l, rr);
                    rr += 1;
                }
                st.lo_out[nr] = l; st.hi_out[nr] = rr;
                st.pw_out[nr] = (c.forced_bos_token_id >= 0 && c.cur_len == 1) ? st.pw_in[pr] : st.hi_in[pr] - st.lo_in[pr];
            } else {
                S.new_tok[b0 + j] = -1;
                st.beam_scores_out[nr] = 0.f;
                st.lo_out[nr] = 0; st.hi_out[nr] = 0; st.pw_out[nr] = 0;
            }
        }
        __syncthreads();                                                         // S is reused by the next group
    }
}

// BeamSearchScorerWithMemory.finalize (seal/beam_search.py:705-725): the live beams are recorded
// once more with their running scores.
__global__ void finalize_kernel(int64_t Q, StepCfg c, const float* __restrict__ beam_scores,
                                const int32_t* __restrict__ tokens, const uint64_t* __restrict__ lo,
                                const uint64_t* __restrict__ hi, StepState st) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= Q * c.num_beams) return;
    const int64_t qi = i / c.num_beams; const int j = (int)(i - qi * c.num_beams);
    const int64_t h = qi * c.hyps_per_query + c.hyp_base + j;
    st.hyp_score[h] = beam_scores[i];
    st.hyp_len[h] = c.cur_len;
    st.hyp_valid[h] = 2;
    for (int t = 0; t < c.T; ++t) st.hyp_tokens[h * c.T + t] = tokens[i * c.T + t];
    if (st.hyp_lo) { st.hyp_lo[h] = lo[i]; st.hyp_hi[h] = hi[i]; }
}

// ---- stateless logits-processor path (seal/beam_search.py:62-140) -------------------------------

// rows -> (lo, hi, rule) from scratch, like the reference: fold of force_decoding_from + sent[1:]
__global__ void __launch_bounds__(128) rows_fold_kernel(FmView fm, int64_t R, int t, const int64_t* __restrict__ ids,
                                                        int skip_first, int eos, int pad, int stop_at_count,
                                                        const uint64_t* __restrict__ force_syms, int n_force,
                                                        int shift, uint64_t* __restrict__ lo_out,
                                                        uint64_t* __restrict__ hi_out, uint8_t* __restrict__ rule_out) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= R) return;
    const int64_t* sent = ids + r * t + skip_first;
    const int n = t - skip_first;
    const int64_t last = sent[n - 1];
    uint64_t l = 0, h = 0, count = 0;
    const bool ended = (last == eos || last == pad);
    if (!ended) {
        uint64_t rr = fm.m, prev_l = 0, prev_r = fm.m;        // get_range starts from (0, size()) (:106-107)
        for (int i = 0; i < n_force; ++i) { prev_l = l; prev_r = rr; lf_step(fm, force_syms[i], l, rr, l, rr); }
        for (int i = 1; i < n; ++i) { prev_l = l; prev_r = rr; lf_step(fm, (uint64_t)sent[i] + shift, l, rr, l, rr); }
        h = rr + 1;
        count = prev_r + 1 - prev_l;                          // get_count(prefix without the last token) (:97,:101)
    }
    uint8_t rule = 0;
    if (stop_at_count > 0 && count <= (uint64_t)stop_at_count) rule = 1;
    else if (ended) rule = 2;
    lo_out[r] = l; hi_out[r] = h; rule_out[r] = rule;
}

// scores_out = scores_in + mask, mask in {0,-inf}
__global__ void __launch_bounds__(256) apply_mask_kernel(int64_t R, int V, int64_t ld, const float* __restrict__ in,
                                                         float* __restrict__ out, const uint32_t* __restrict__ masks,
                                                         int mask_words, int shared_mask,
                                                         const uint8_t* __restrict__ rule, int eos, int pad,
                                                         int always_allow_eos, int only_token) {
    const int64_t r = blockIdx.x;
    const uint32_t* mrow = shared_mask ? masks : masks + r * mask_words;
    const int ru = rule ? rule[r] : 0;
    for (int v = blockIdx.y * blockDim.x + threadIdx.x; v < V; v += gridDim.y * blockDim.x) {
        bool allowed;
        if (only_token >= 0) allowed = v == only_token;
        else {
            allowed = ru == 1 ? v == eos : ru == 2 ? v == pad : ((mrow[v >> 5] >> (v & 31)) & 1);
            if (always_allow_eos && v == eos) allowed = true;
        }
        const float x = in[r * ld + v];
        out[r * ld + v] = allowed ? x + 0.0f : x + (-INFINITY);
    }
}


// ---- teacher-forced scoring (seal/keys.py:64-141 rescore_keys, :145-176 compute_unigram_scores) ------
// out[r] = log_softmax(logits[r] / temperature)[target[r]]   (full-vocabulary normalisation);
// optionally the whole log-prob row.  One CTA per row, single streaming pass for the statistics.
__global__ void __launch_bounds__(256) target_logprob_kernel(int64_t R, int V, int64_t ld, const float* __restrict__ logits,
                                                             const int64_t* __restrict__ targets, int64_t tgt_stride,
                                                             float temperature, float* __restrict__ out,
                                                             int64_t out_stride, float* __restrict__ full, int64_t full_ld) {
    __shared__ float red[8];
    const int64_t r = blockIdx.x;
    const float* lp = logits + r * ld;
    float mx = -INFINITY, se = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const float x = lp[v] / temperature;              // the reference divides the logits (seal/keys.py:167)
        if (x > mx) { se *= expf(mx - x); mx = x; }
        if (mx > -INFINITY) se += expf(x - mx);
        else if (isnan(x)) se = x;                        // a NaN ahead of the thread's first finite entry
    }
    const float bm = block_reduce_max(mx, red);
    // se is 0 while mx = -inf unless a NaN was seen: it then makes the whole row NaN, as torch's log_softmax does
    const float scaled = (mx > -INFINITY) ? se * expf(mx - bm) : se;
    const float tot = block_reduce_sum(scaled, red);
    const float logsum = logf(tot);
    if (out && threadIdx.x == 0) {
        const int64_t t = targets[r * tgt_stride];
        out[r * out_stride] = (t >= 0 && t < V) ? (lp[t] / temperature - bm) - logsum : 0.f;
    }
    if (full)
        for (int v = threadIdx.x; v < V; v += blockDim.x) full[r * full_ld + v] = (lp[v] / temperature - bm) - logsum;
}
}  // namespace sealb200
