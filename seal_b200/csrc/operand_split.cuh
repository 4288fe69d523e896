// The operand splits of the error-compensated x3 GEMMs (wgmma_gemm.cuh), one per GEMM element type T: how an fp32
// value becomes T's pieces and how the pieces of consecutive values are stored.  The producers (bart_kernels.cuh
// SplitOut / SplitBf16), the GEMM epilogue, the split-K finish pass and the stand-alone split kernel all split through
// here, and the host sizes and views split buffers with kPieces.  No kernel: any unit may include it.
//   float (3xTF32, gemm_mode 2):        hi = x with the 13 low mantissa bits cleared, lo = x - hi (exact).
//   __half (3xFP16, gemm_mode 3 / 5):   h1 = rn_half(x), h2 = rn_half(x - h1), x saturated at +-65504 first, which
//                                       raises the caller's overflow flag.
//   __nv_bfloat16 (3xBF16, gemm_mode 6): x = b1 + b2 + b3, each piece the round-to-nearest bf16 of what the previous
//     pieces leave.  Each residual is exact in fp32 and has at most 16, then 8 significant bits, so the three pieces
//     carry x exactly for every 2^-100 <= |x| < (2 - 2^-8) 2^127 (below, b3 may be a bf16 subnormal; from the upper
//     bound on, which only the last 2^-8 of fp32's range reaches, b1 rounds to infinity); bf16 has fp32's exponent
//     range, so nothing saturates.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>
#include <utility>

namespace sealb200 {

// pieces per value of format T
template <typename T> constexpr int kPieces = 2;
template <> constexpr int kPieces<__nv_bfloat16> = 3;

// x -> its pieces p in format T.  Only the fp16 split can overflow: it sets ov (no atomic; the caller publishes it).
__device__ __forceinline__ void split_value(float x, float (&p)[2], int&) {
    p[0] = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    p[1] = x - p[0];
}
__device__ __forceinline__ void split_value(float x, __half (&p)[2], int& ov) {
    if (fabsf(x) > 65504.f) { ov = 1; x = copysignf(65504.f, x); }
    p[0] = __float2half_rn(x);
    p[1] = __float2half_rn(x - __half2float(p[0]));
}
__device__ __forceinline__ void split_value(float x, __nv_bfloat16 (&p)[3], int&) {
    p[0] = __float2bfloat16_rn(x);
    const float r = x - __bfloat162float(p[0]);
    p[1] = __float2bfloat16_rn(r);
    p[2] = __float2bfloat16_rn(r - __bfloat162float(p[1]));
}

__device__ __forceinline__ uint32_t pack2(__half a, __half b) { return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16); }
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// The V consecutive values v (V = 1, 2 or 4) split into format T: q[e][i] is piece i of v[e].  ov as split_value.
// (The index sequences keep every array index a constant, so the arrays live in registers from the start.)
template <typename T, int V, int... E>
__device__ __forceinline__ void split_values(const float (&v)[V], T (&q)[V][kPieces<T>], int& ov, std::integer_sequence<int, E...>) {
    (split_value(v[E], q[E], ov), ...);
}
template <typename T, int V> __device__ __forceinline__ void split_values(const float (&v)[V], T (&q)[V][kPieces<T>], int& ov) {
    split_values(v, q, ov, std::make_integer_sequence<int, V>{});
}

// piece I of the V values q (split_values) to dst with one access of V elements (dst aligned to it)
template <int I, typename T, int V> __device__ __forceinline__ void store_piece(T* dst, const T (&q)[V][kPieces<T>]) {
    static_assert(V == 1 || V == 2 || V == 4, "vector width");
    if constexpr (V == 1) *dst = q[0][I];
    else if constexpr (std::is_same<T, float>::value) {
        if constexpr (V == 2) *reinterpret_cast<float2*>(dst) = make_float2(q[0][I], q[1][I]);
        else *reinterpret_cast<float4*>(dst) = make_float4(q[0][I], q[1][I], q[2][I], q[3][I]);
    } else if constexpr (V == 2) *reinterpret_cast<uint32_t*>(dst) = pack2(q[0][I], q[1][I]);
    else *reinterpret_cast<uint2*>(dst) = make_uint2(pack2(q[0][I], q[1][I]), pack2(q[2][I], q[3][I]));
}

// every piece i of the V values q stored at s[i] + off with one vector access
template <typename T, int V, int... I>
__device__ __forceinline__ void store_pieces(T* const* s, int64_t off, const T (&q)[V][kPieces<T>], std::integer_sequence<int, I...>) {
    (store_piece<I>(s[I] + off, q), ...);
}
template <typename T, int V> __device__ __forceinline__ void store_pieces(T* const* s, int64_t off, const T (&q)[V][kPieces<T>]) {
    store_pieces(s, off, q, std::make_integer_sequence<int, kPieces<T>>{});
}

// split_values, then store_pieces
template <typename T, int V> __device__ __forceinline__ void store_split(T* const* s, int64_t off, const float (&v)[V], int& ov) {
    T q[V][kPieces<T>];
    split_values(v, q, ov);
    store_pieces(s, off, q);
}

}  // namespace sealb200
