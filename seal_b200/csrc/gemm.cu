// GEMM dispatch of the decode library: C = A W^T + b on the tensor cores (wgmma_gemm.cuh) in the model's gemm_mode --
// operand formats, split-K, L2 bands, the lm_head statistics epilogue -- and the weights' operand splits.
#include "decode_model.hpp"
#include "wgmma_gemm.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

namespace {

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

// the n values of x times scale split into format T's pieces p0, p1 (, p2) on stream s; 3xFP16 raises *ovf for a value
// past the fp16 range
template <typename T> void split_into(cudaStream_t s, const float* x, float scale, int64_t n, T* p0, T* p1, T* p2, int* ovf) {
    const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8);
    split_kernel<T><<<std::max(blocks, 1), 256, 0, s>>>(n, x, scale, p0, p1, p2, ovf);
    CUDA_CHECK(cudaGetLastError());
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

// K slices of a 3xFP16 / 3xBF16 GEMM of `tiles` output tiles: skinny problems (a few tiles for the whole GPU) split K
// so that the serial K loop of a tile is spread over up to 8 CTAs, then sum the partial tiles in a fixed order
int split_k_slices(int tiles, int kblocks) {
    int k_slices = 1;
    if (tiles * 2 <= sm_count() && kblocks >= 4) {
        k_slices = std::min(8, std::min(kblocks / 2, sm_count() / tiles));
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

// The x3 GEMM's operand formats, by element type T: the Lin fields of W's pieces, whether the epilogue unscales W by
// l.w_unscale, whether split-K, L2 bands and the lm_head statistics epilogue apply (tuned), and the last_paths bits of
// every call and of the whole-tile launch.  3xBF16's W is one piece; its kernel reads A's third piece in the W lo slot.
template <typename T> using LinField = T* Lin::*;
template <typename T> struct X3Format;
template <> struct X3Format<__half> {                 // 3xFP16 (modes 3, 5): A = h1 + h2, W * 2^s = w_h1 + w_h2
    static constexpr LinField<__half> w = &Lin::w_h1, w2 = &Lin::w_h2;
    static constexpr bool scaled_w = true, tuned = true;
    static constexpr uint32_t path_call = 0, path_tile = kPathGemmFullTile;
};
template <> struct X3Format<__nv_bfloat16> {          // 3xBF16 (mode 6): A = b1 + b2 + b3, W once in bf16
    static constexpr LinField<__nv_bfloat16> w = &Lin::w_bf;
    static constexpr bool scaled_w = false, tuned = true;
    static constexpr uint32_t path_call = kPathGemmBf16, path_tile = 0;
};
template <> struct X3Format<float> {                  // 3xTF32 (mode 2): A = hi + lo, W = w_hi + w_lo; band 0, gemm_band ignored
    static constexpr LinField<float> w = &Lin::w_hi, w2 = &Lin::w_lo;
    static constexpr bool scaled_w = false, tuned = false;    // unscaled: after an overflow fallback l.w_unscale is 3xFP16's
    static constexpr uint32_t path_call = 0, path_tile = kPathGemmTf32;
};

// x (n fp32 values) split into format T's pieces in buf, grown to 8 bytes per element and viewed as split_view.
// 3xFP16 raises *ovf for a value past the fp16 range.
template <typename T> Act split_act(cudaStream_t s, float* x, int64_t n, Buf& buf, int* ovf) {
    buf.ensure((size_t)n * 8);
    const Act a = split_view<T>(x, buf);
    split_into(s, x, 1.0f, n, a.piece<T>(0), a.piece<T>(1), a.piece<T>(2), ovf);
    return a;
}

template <typename T>
void gemm_x3(Ctx& cx, int64_t M, int N, int K, const Act& A, Lin& l, const Act& C, int ldc, int act, int64_t defer_rows) {
    using F = X3Format<T>;
    constexpr int pieces = kPieces<T>;
    sealbart* m = cx.m;
    const int tiles = (int)(((N + GN - 1) / GN) * ((M + GM - 1) / GM));
    const int n_fastest = ((int64_t)M >= (int64_t)N) ? 1 : 0;     // stream the larger operand once
    Act a = A;
    if (!a.p[0]) {
        a = split_act<T>(cx.s, A.x, M * K, cx.slice ? m->a_split1 : m->a_split, m->ovf);
        m->launches++;
    }
    CUtensorMap ma[3];
    for (int i = 0; i < pieces; ++i) make_map(&ma[i], a.piece<T>(i), M, K, K, GM);
    if (!l.maps_ready) {
        make_map(&l.map_hi, l.*F::w, N, K, K, GN);
        if constexpr (pieces == 2) make_map(&l.map_lo, l.*F::w2, N, K, K, GN);
        l.maps_ready = true;
    }
    const CUtensorMap& w_lo = pieces == 3 ? ma[2] : l.map_lo;
    T* const c1 = C.piece<T>(0); T* const c2 = C.piece<T>(1); T* const c3 = C.piece<T>(2);
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
            if (M <= defer_rows && act == kActNone && !C.p[0] && ldc == N && l.b) {     // C has no split output: summed by the consumer kernel
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

void gemm_impl(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act, int64_t defer_rows) {
    if (M == 0) return;
    if (act == kActRelu) cx.m->last_paths |= kPathT5Relu;
    with_format(cx.m->cfg.gemm_mode, [&](auto t) {
        using T = decltype(t);
        if (K % GemmElem<T>::KE || lda != K || !(l.*X3Format<T>::w))
            throw ApiError(SEALFM_EINVAL, "GEMM: K must be a multiple of 64 (3xFP16, 3xBF16) / 32 (3xTF32) with contiguous operands");
        gemm_x3<T>(cx, M, N, K, A, l, C, ldc, act, defer_rows);
    });
}

// 3xTF32 operand copies of l (gemm_mode 2): W = w_hi + w_lo, allocated here and owned by m (split_allocs)
void split_lin_tf32(sealbart* m, Lin& l) {
    const uint64_t n = (uint64_t)l.out * l.in;
    CUDA_CHECK(cudaMalloc(&l.w_hi, n * 4)); m->split_allocs.push_back(l.w_hi);
    CUDA_CHECK(cudaMalloc(&l.w_lo, n * 4)); m->split_allocs.push_back(l.w_lo);
    split_into<float>(nullptr, l.w, 1.0f, (int64_t)n, l.w_hi, l.w_lo, nullptr, nullptr);
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
    split_into<__half>(nullptr, l.w, std::ldexp(1.0f, sexp), (int64_t)n, l.w_h1, l.w_h2, nullptr, m->err.as<int>() + 1);
    l.maps_ready = false;
}

}  // namespace

namespace sealb200 {

void gemm(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act, int64_t defer_rows) {
    sealbart* m = cx.m;
    if (!m->profile_gemm || M == 0) { gemm_impl(cx, M, N, K, A, lda, l, C, ldc, act, defer_rows); return; }
    cudaEvent_t a, b;
    CUDA_CHECK(cudaEventCreate(&a)); CUDA_CHECK(cudaEventCreate(&b));
    CUDA_CHECK(cudaEventRecord(a, cx.s));
    gemm_impl(cx, M, N, K, A, lda, l, C, ldc, act, defer_rows);
    CUDA_CHECK(cudaEventRecord(b, cx.s));
    m->gemm_events.emplace_back(a, b);
    m->gemm_flops += 2.0 * (double)M * N * K;
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

void check_gemm_mode(int mode) {
    if (mode != kGemmTf32 && !is_3xfp16(mode) && mode != kGemmBf16)
        throw ApiError(SEALFM_EINVAL, "gemm_mode must be 3 (3xFP16, one CTA per tile, default), 5 (3xFP16 on 2-CTA clusters), 2 (3xTF32) "
                                      "or 6 (3xBF16, bf16 weights)");
}

}  // namespace sealb200

// ---- test hooks ------------------------------------------------------------------------------------------------

extern "C" {

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

}  // extern "C"

namespace {

// The lm_head statistics epilogue of sealdec_debug_head: the row masks [M][ceil(N/32)] (host), eos / pad, and where
// the statistics [Mpad][ceil(N/128)] go (host; Mpad = M rounded up to 128 rows) and whether the epilogue ran.
struct DebugHead { const uint32_t* mask; int eos, pad; float* stats; int32_t* fused; };

// The other outputs of sealdec_debug_gemm_split (host pointers): the operand split of the next GEMM into s[0..2] when
// `split` is set, the epilogue's overflow flag, defer_rows with the deferred slices, and the call's last_paths bits.
struct DebugSplit {
    bool split; void* s[3]; int32_t* overflow; int64_t defer_rows; float* slices; int32_t* k_slices; float* unscale; uint32_t* paths;
};

// presplit: 3xFP16 and 3xBF16 split the activations once, outside the timed calls (as the decoder's producers do)
// act: kActNone, kActGelu or kActRelu
int debug_gemm(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias, float* C,
               int32_t act, int32_t iters, double* avg_us, int32_t band, int32_t store, bool presplit,
               const DebugHead* head = nullptr, const DebugSplit* so = nullptr) {
    return guarded([&] {
        if (!A || !W || (store && !C) || M <= 0 || N <= 0 || K <= 0 || band < -1 || act < kActNone || act > kActRelu)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (head && (!head_stats_mode(mode) || !store || act || iters > 0 || !head->mask || !head->stats || !head->fused))
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (so && (head || iters > 0 || (!store && !so->split) || (so->split && (!so->s[0] || !so->s[1] || (mode == kGemmBf16 && !so->s[2]))) ||
                   !so->overflow || !so->paths || !so->k_slices || so->defer_rows < 0 || (so->defer_rows > 0 && (!so->slices || !so->unscale))))
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
        Buf dA, dC, dA_split, dC_split;
        const int ldc = (N + 3) / 4 * 4;
        dA.ensure((size_t)M * K * 4); dC.ensure((size_t)M * ldc * 4);
        CUDA_CHECK(cudaMemcpy(dA.p, A, (size_t)M * K * 4, cudaMemcpyHostToDevice));
        Act a{dA.as<float>()};
        if (presplit && mode != kGemmTf32)
            with_format(mode, [&](auto t) { a = split_act<decltype(t)>(nullptr, a.x, M * K, dA_split, fake.ovf); });
        Act c{store ? dC.as<float>() : nullptr};
        size_t elem = 4;
        if (so) {
            // only the epilogue's flag is reported: clear what the input split raised.  Every output starts poisoned
            // (all-ones bits: NaN in fp32, fp16 and bf16), so an element the GEMM does not write comes back as NaN.
            CUDA_CHECK(cudaDeviceSynchronize());
            CUDA_CHECK(cudaMemset(fake.ovf, 0, sizeof(int)));
            CUDA_CHECK(cudaMemset(dC.p, 0xFF, (size_t)M * ldc * 4));
            if (so->split) {
                dC_split.ensure((size_t)M * ldc * 8);
                CUDA_CHECK(cudaMemset(dC_split.p, 0xFF, (size_t)M * ldc * 8));
                with_format(mode, [&](auto t) { c = split_view<decltype(t)>(c.x, dC_split); elem = sizeof(t); });
            }
        }
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
        gemm(cx, M, N, K, a, K, l, head ? Act{dC.as<float>()} : c, ldc, act, so ? so->defer_rows : 0);
        CUDA_CHECK(cudaDeviceSynchronize());
        if (so) {
            CUDA_CHECK(cudaMemcpy(so->overflow, fake.ovf, sizeof(int32_t), cudaMemcpyDeviceToHost));
            *so->paths = fake.last_paths;
            const SplitSrc& p = cx.pending;
            *so->k_slices = p.ks;
            if (p.ks > 0) {                                    // deferred: [k_slices][M][ldc] raw slices (ldc == N)
                CUDA_CHECK(cudaMemcpy(so->slices, p.part, (size_t)p.ks * p.stride * 4, cudaMemcpyDeviceToHost));
                *so->unscale = p.unscale;
            }
            for (int i = 0; i < 3; ++i)
                if (c.p[i]) CUDA_CHECK(cudaMemcpy2D(so->s[i], (size_t)N * elem, c.p[i], (size_t)ldc * elem, (size_t)N * elem, M, cudaMemcpyDeviceToHost));
        }
        if (head) {
            *head->fused = cx.head_fused ? 1 : 0;
            CUDA_CHECK(cudaMemcpy2D(C, (size_t)N * 4, dC.p, (size_t)ldc * 4, (size_t)N * 4, m_pad, cudaMemcpyDeviceToHost));
            CUDA_CHECK(cudaMemcpy(head->stats, dstats.p, (size_t)m_pad * n_tiles * 8, cudaMemcpyDeviceToHost));
            return;
        }
        if (iters > 0 && avg_us) {
            cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
            CUDA_CHECK(cudaEventRecord(e0, nullptr));
            for (int i = 0; i < iters; ++i) gemm(cx, M, N, K, a, K, l, c, ldc, act);
            CUDA_CHECK(cudaEventRecord(e1, nullptr));
            CUDA_CHECK(cudaEventSynchronize(e1));
            float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
            *avg_us = (double)ms * 1e3 / iters;
            cudaEventDestroy(e0); cudaEventDestroy(e1);
        }
        if (store) CUDA_CHECK(cudaMemcpy2D(C, (size_t)N * 4, dC.p, (size_t)ldc * 4, (size_t)N * 4, M, cudaMemcpyDeviceToHost));
    });
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

int sealdec_debug_gemm_split(int mode, int64_t M, int32_t N, int32_t K, const float* A, const float* W, const float* bias,
                             int32_t act, int32_t outputs, float* C, void* s1, void* s2, void* s3, int32_t* overflow,
                             int64_t defer_rows, float* slices, int32_t* k_slices, float* unscale, uint32_t* paths) {
    if (outputs < 1 || outputs > 3) return guarded([] { throw ApiError(SEALFM_EINVAL, "outputs must be 1, 2 or 3"); });
    const DebugSplit so{(outputs & 2) != 0, {s1, s2, s3}, overflow, defer_rows, slices, k_slices, unscale, paths};
    return debug_gemm(mode, M, N, K, A, W, bias, C, act, 0, nullptr, -1, outputs & 1, true, nullptr, &so);
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

}  // extern "C"
