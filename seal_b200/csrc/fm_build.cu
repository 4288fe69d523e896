// Index construction on the GPU (SURVEY.md §8f rank 3): symbols -> suffix array -> BWT -> level-wise
// wavelet-tree bits -> SA / ISA samples, producing exactly the HostIndex the host builder (fm_host.cpp:
// SA-IS) produces -- the sections sdsl's construct() would write (sdsl/construct.hpp:120-166,
// sdsl/wt_int.hpp:169-256, sdsl/csa_sampling_strategy.hpp:85-99,626-641) -- so that save / to_device and
// every query kernel are unchanged.  tests/test_fm_gpu.py compares the two builders section by section.
//
// Suffix sorting is prefix doubling on dense ranks: round h sorts the m = n+1 suffixes by the 64-bit key
// (rank_h[i] << 32 | rank_h[i+h]) and re-ranks; ceil(log2(longest repeat)) + 1 rounds, each one radix sort
// of m (key, position) pairs plus three streaming kernels.  The unique sentinel (symbol 0 at position n)
// makes every suffix distinct before it can run off the end, so "past the end" is simply rank 0.
// Device-wide radix sort and prefix sum are CUB's (CUDA toolkit primitives, like cuBLAS for a plain
// GEMM); everything specific to the index is written here.  Memory: 40 bytes per symbol.
//
// Limit: m < 2^32 (32-bit ranks and positions, 64-bit keys, 64-bit item counts in the CUB calls) AND 40 B x m of free
// device memory: ~1.9e9 symbols on an 80 GB H100, so NQ-sized (~3.2e9) and KILT-sized (~5.5e9, 33-bit rows) texts go
// through the host SA-IS builder; the query kernels are 64-bit throughout.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <stdexcept>
#include <vector>

#include "common.cuh"
#include "fm_build_common.cuh"
#include "fm_host.hpp"
#include "../../include/sealfm.h"

namespace sealb200 {
namespace {

__global__ void __launch_bounds__(kBT) iota_kernel(uint32_t* v, uint64_t m) { GRID_STRIDE(i, m) v[i] = (uint32_t)i; }

// flag[j] = 1 where the sorted key changes (j = 0 included)
template <typename K>
__global__ void __launch_bounds__(kBT) boundary_kernel(const K* __restrict__ key, uint32_t* __restrict__ flag, uint64_t m) {
    GRID_STRIDE(j, m) flag[j] = (j == 0 || key[j] != key[j - 1]) ? 1u : 0u;
}

// rank[sa[j]] = dense rank of the group sorted position j belongs to (1-based)
__global__ void __launch_bounds__(kBT) scatter_rank_kernel(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ grp,
                                                            uint32_t* __restrict__ rank, uint64_t m) {
    GRID_STRIDE(j, m) rank[sa[j]] = grp[j];
}

__global__ void __launch_bounds__(kBT) pair_key_kernel(const uint32_t* __restrict__ rank, uint64_t* __restrict__ key,
                                                        uint32_t* __restrict__ pos, uint64_t m, uint64_t h) {
    GRID_STRIDE(i, m) {
        const uint64_t hi = rank[i];
        const uint64_t lo = (i + h < m) ? rank[i + h] : 0;
        key[i] = (hi << 32) | lo;
        pos[i] = (uint32_t)i;
    }
}

// alphabet[c] = symbol of group c, C[c] = its first sorted position  (csa_alphabet_strategy.hpp:494-534)
__global__ void __launch_bounds__(kBT) alphabet_kernel(const uint32_t* __restrict__ sorted_sym, const uint32_t* __restrict__ flag,
                                                        const uint32_t* __restrict__ grp, uint64_t* __restrict__ alphabet,
                                                        uint64_t* __restrict__ C, uint64_t m) {
    GRID_STRIDE(j, m) if (flag[j]) { alphabet[grp[j] - 1] = sorted_sym[j]; C[grp[j] - 1] = j; }
}

// BWT in real symbols + the two sample arrays, one pass over the suffix array
__global__ void __launch_bounds__(kBT) bwt_samples_kernel(const uint32_t* __restrict__ sa, const uint32_t* __restrict__ text,
                                                           uint32_t* __restrict__ bwt, uint64_t* __restrict__ sa_samples,
                                                           uint64_t* __restrict__ isa_samples, uint64_t m) {
    GRID_STRIDE(i, m) {
        const uint32_t p = sa[i];
        bwt[i] = p ? text[p - 1] : text[m - 1];
        if ((i & 31) == 0) sa_samples[i >> 5] = p;
        if ((p & 63) == 0) isa_samples[p >> 6] = i;
    }
}

}  // namespace

void build_index_gpu(const uint64_t* symbols, uint64_t n, int device, HostIndex& o) {
    o = HostIndex();
    const uint64_t m = n + 1;
    if (m >= (1ULL << 32) - 8) throw ApiError(SEALFM_EINVAL, "GPU index construction handles texts below 2^32 symbols (32-bit ranks); use sealfm_build");
    {
        size_t free_b = 0, total_b = 0;
        CUDA_CHECK(cudaSetDevice(device));
        CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
        if ((double)m * 42.0 + (double)(1ull << 30) > (double)free_b)
            throw ApiError(SEALFM_ENOMEM, "GPU index construction needs ~40 bytes of device memory per symbol; use sealfm_build");
    }
    std::vector<uint32_t> text(m);
    for (uint64_t i = 0; i < n; ++i) {
        if (symbols[i] == 0) throw ApiError(SEALFM_EINVAL, "symbol 0 is reserved for the sentinel");
        if (symbols[i] >= (1ULL << 32)) throw ApiError(SEALFM_EINVAL, "symbols must be < 2^32");
        text[i] = (uint32_t)symbols[i];
    }
    text[n] = 0;
    CUDA_CHECK(cudaSetDevice(device));
    cudaStream_t st = nullptr;

    Dev<uint32_t> d_text(m), d_rank(m), d_pos_a(m), d_pos_b(m), d_flag(m), d_grp(m);
    Dev<uint64_t> d_key_a(m), d_key_b(m);
    CUDA_CHECK(cudaMemcpyAsync(d_text.p, text.data(), m * 4, cudaMemcpyHostToDevice, st));

    // one temp buffer big enough for every CUB call below
    size_t tmp_sort64 = 0, tmp_sort32 = 0, tmp_scan = 0, tmp_keys32 = 0;
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort64, d_key_a.p, d_key_b.p, d_pos_a.p, d_pos_b.p, (int64_t)m, 0, 64, st));
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort32, d_flag.p, d_grp.p, d_pos_a.p, d_pos_b.p, (int64_t)m, 0, 32, st));
    CUDA_CHECK(cub::DeviceRadixSort::SortKeys(nullptr, tmp_keys32, d_flag.p, d_grp.p, (int64_t)m, 0, 32, st));
    CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, d_flag.p, d_grp.p, (int64_t)m, st));
    const size_t tmp_bytes = std::max(std::max(tmp_sort64, tmp_sort32), std::max(tmp_scan, tmp_keys32));
    Dev<uint8_t> d_tmp(tmp_bytes);
    size_t tb;

    const int G = blocks_for(m);
    auto rerank = [&](auto* sorted_key, const uint32_t* sorted_pos) -> uint32_t {
        boundary_kernel<<<G, kBT, 0, st>>>(sorted_key, d_flag.p, m);
        tb = tmp_bytes;
        CUDA_CHECK(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, d_flag.p, d_grp.p, (int64_t)m, st));
        scatter_rank_kernel<<<G, kBT, 0, st>>>(sorted_pos, d_grp.p, d_rank.p, m);
        CUDA_CHECK(cudaGetLastError());
        uint32_t groups = 0;
        CUDA_CHECK(cudaMemcpyAsync(&groups, d_grp.p + (m - 1), 4, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        return groups;
    };

    // round 0: sort by the symbol itself -> alphabet, C, ranks of the 1-symbol prefixes
    iota_kernel<<<G, kBT, 0, st>>>(d_pos_a.p, m);
    const int sym_bits = (int)hi_bit64(std::max<uint32_t>(1, *std::max_element(text.begin(), text.end()))) + 1;
    uint32_t* d_sym_sorted = reinterpret_cast<uint32_t*>(d_key_b.p);           // scratch: key_b is free in round 0
    tb = tmp_bytes;
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(d_tmp.p, tb, d_text.p, d_sym_sorted, d_pos_a.p, d_pos_b.p, (int64_t)m, 0, sym_bits, st));
    uint32_t groups = rerank(d_sym_sorted, d_pos_b.p);
    o.size = m;
    o.sigma = groups;
    {
        Dev<uint64_t> d_alpha(groups), d_C(groups);
        alphabet_kernel<<<G, kBT, 0, st>>>(d_sym_sorted, d_flag.p, d_grp.p, d_alpha.p, d_C.p, m);
        CUDA_CHECK(cudaGetLastError());
        o.alphabet.resize(groups); o.C.resize(groups + 1);
        CUDA_CHECK(cudaMemcpyAsync(o.alphabet.data(), d_alpha.p, groups * 8ull, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(o.C.data(), d_C.p, groups * 8ull, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
        o.C[groups] = m;
    }
    o.max_level = hi_bit64(std::max<uint64_t>(o.alphabet.back(), 1)) + 1;      // sdsl/wt_int.hpp:182-193

    // prefix doubling
    const uint32_t* d_sa = d_pos_b.p;
    const int rank_bits = (int)hi_bit64(m) + 1;                                 // ranks are <= m
    for (uint64_t h = 1; groups < m; h <<= 1) {
        pair_key_kernel<<<G, kBT, 0, st>>>(d_rank.p, d_key_a.p, d_pos_a.p, m, h);
        tb = tmp_bytes;
        CUDA_CHECK(cub::DeviceRadixSort::SortPairs(d_tmp.p, tb, d_key_a.p, d_key_b.p, d_pos_a.p, d_pos_b.p, (int64_t)m, 0, 32 + rank_bits, st));
        groups = rerank(d_key_b.p, d_pos_b.p);
        if (h > m) throw ApiError(SEALFM_ECUDA, "suffix sort did not converge");
    }

    // BWT + samples
    Dev<uint32_t>& d_bwt = d_flag;                                              // flag / grp are free from here on
    const uint64_t n_sa = (m + 31) / 32, n_isa = (m - 1) / 64 + 1;
    {
        Dev<uint64_t> d_sas(n_sa), d_isas(n_isa);
        bwt_samples_kernel<<<G, kBT, 0, st>>>(d_sa, d_text.p, d_bwt.p, d_sas.p, d_isas.p, m);
        CUDA_CHECK(cudaGetLastError());
        o.sa_samples.resize(n_sa); o.isa_samples.resize(n_isa);
        CUDA_CHECK(cudaMemcpyAsync(o.sa_samples.data(), d_sas.p, n_sa * 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaMemcpyAsync(o.isa_samples.data(), d_isas.p, n_isa * 8, cudaMemcpyDeviceToHost, st));
        CUDA_CHECK(cudaStreamSynchronize(st));
    }

    // wavelet tree, level by level: level k+1's order = level k's order stably sorted by one more leading bit
    const uint32_t L = o.max_level;
    const uint64_t words = (m * L + 63) >> 6;
    Dev<uint64_t> d_tree(words);
    CUDA_CHECK(cudaMemsetAsync(d_tree.p, 0, words * 8, st));
    uint32_t* cur = d_bwt.p;
    uint32_t* nxt = d_grp.p;
    const int PG = pack_blocks_for(m);
    for (uint32_t k = 0; k < L; ++k) {
        if (k > 0) {                                                            // order by the k leading bits
            tb = tmp_bytes;
            CUDA_CHECK(cub::DeviceRadixSort::SortKeys(d_tmp.p, tb, cur, nxt, (int64_t)m, (int)(L - k), (int)L, st));
            // always re-sort from the BWT order: radix sort on bits [L-k, L) is stable, so this IS the node order
            pack_level_kernel<<<PG, kBT, 0, st>>>(nxt, reinterpret_cast<uint32_t*>(d_tree.p), m, k, L);
        } else {
            pack_level_kernel<<<PG, kBT, 0, st>>>(cur, reinterpret_cast<uint32_t*>(d_tree.p), m, k, L);
        }
        CUDA_CHECK(cudaGetLastError());
    }
    o.tree.resize(words);
    CUDA_CHECK(cudaMemcpyAsync(o.tree.data(), d_tree.p, words * 8, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
}

}  // namespace sealb200
