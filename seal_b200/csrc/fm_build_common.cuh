// Pieces shared by the two GPU index builders: fm_build.cu (in-memory, 32-bit ranks) and fm_build_large.cu (64-bit
// positions, streamed suffix array).  Each translation unit gets its own copy (anonymous namespace).
#pragma once
#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace sealb200 {
namespace {

constexpr int kBT = 256;

inline int blocks_for(uint64_t n) {
    uint64_t b = (n + kBT - 1) / kBT;
    const uint64_t cap = (uint64_t)sm_count() * 16;          // grid-stride loops; multiple of the SM count
    return (int)std::max<uint64_t>(1, std::min(b, cap));
}

#define GRID_STRIDE(i, n) \
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < (n); i += (uint64_t)gridDim.x * blockDim.x)

// Level k of the wavelet tree: `keys` holds the BWT stably sorted by its k leading bits (node order); bit
// L-k-1 of element i goes to global bit position k*m + i of the level-concatenated tree
// (sdsl/wt_int.hpp:202-242).  One warp packs 32 consecutive global positions with a ballot; levels meet
// inside a word, hence atomicOr on the (zero-initialised) 32-bit halves.
__global__ void __launch_bounds__(kBT) pack_level_kernel(const uint32_t* __restrict__ keys, uint32_t* __restrict__ tree32,
                                                          uint64_t m, uint32_t k, uint32_t L) {
    const uint64_t first = (uint64_t)k * m, last = first + m;       // global bit range of this level
    const uint64_t w0 = first >> 5, w1 = (last + 31) >> 5;          // 32-bit words touched
    const uint32_t shift = L - k - 1;
    for (uint64_t w = w0 + (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) / 32; w < w1; w += (uint64_t)gridDim.x * blockDim.x / 32) {
        const uint64_t pos = (w << 5) + (threadIdx.x & 31);
        const bool in = pos >= first && pos < last;
        const uint32_t bit = in ? ((keys[pos - first] >> shift) & 1u) : 0u;
        const uint32_t word = __ballot_sync(0xffffffffu, bit);
        if ((threadIdx.x & 31) == 0 && word) atomicOr(tree32 + w, word);
    }
}

// grid of pack_level_kernel for a text of m symbols
inline int pack_blocks_for(uint64_t m) {
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((m / 32 + kBT / 32) / (kBT / 32) + 1, (uint64_t)sm_count() * 16));
}

template <typename T>
struct Dev {
    T* p = nullptr;
    uint64_t n = 0;
    explicit Dev(uint64_t count) : n(count) { if (count) CUDA_CHECK(cudaMalloc(&p, count * sizeof(T))); }
    ~Dev() { if (p) cudaFree(p); }
    Dev(const Dev&) = delete;
    Dev& operator=(const Dev&) = delete;
};

inline uint32_t hi_bit64(uint64_t x) { uint32_t r = 0; while (x >>= 1) ++r; return r; }

}  // namespace
}  // namespace sealb200
