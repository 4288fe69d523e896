// CUDA kernels + C ABI (include/sealfm.h) of the FM-index path.  sm_90a only.
#include "../../include/sealfm.h"
#include "fm_device.cuh"
#include "fm_host.hpp"
#include "fm_layout.hpp"
#include "fm_expand.cuh"
#include "fm_handle.hpp"
#include "common.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

using namespace sealb200;

// ------------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------------
struct sealfm {
    HostIndex host;
    int device = -1;
    FmView view{};                 // device pointers
    void* d_blocks = nullptr;
    uint64_t* d_csym = nullptr;
    NodeEntry* d_node_tab = nullptr;
    uint64_t* d_sa = nullptr;
    uint64_t* d_isa = nullptr;
    uint64_t* d_beginnings = nullptr;
    uint64_t device_bytes = 0;
    std::vector<uint64_t> beginnings;
    // Host-pointer entry points: per-handle staging instead of a cudaMalloc / cudaFree pair per call.  Small calls
    // (seal/retrieval.py:91 issues one get_count per key: 285 k per 1 000 queries) go through MAPPED pinned memory --
    // the kernel reads its arguments from and writes its results to host memory directly: one launch + one stream
    // synchronisation, no copies.  Larger calls use a grow-only device buffer.  Guarded by a mutex: re-entrant.
    mutable std::mutex stage_mu;
    mutable cudaStream_t stage_stream = nullptr;
    mutable void* pin_h = nullptr; mutable void* pin_d = nullptr; mutable size_t pin_bytes = 0;
    mutable void* dev_p = nullptr; mutable size_t dev_bytes = 0;
};

namespace {

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------

// Two LF steps walked in lockstep: four dependent rank chains (i, j of both symbols) are in flight per level, and the
// next level's node entries are fetched with them.  One triple per thread (two chains) left the kernel latency-bound
// beyond L2, with low issue activity.
__device__ __forceinline__ void lf_step_pair(const FmView& v, uint64_t c0, uint64_t l0, uint64_t r0, uint64_t c1, uint64_t l1, uint64_t r1,
                                             uint64_t& ol0, uint64_t& or0, uint64_t& ol1, uint64_t& or1) {
    const uint32_t L = v.L;
    const bool p0 = sym_present(v, c0), p1 = sym_present(v, c1);
    const bool w0 = p0 && l0 == 0 && r0 + 1 == v.m, w1 = p1 && l1 == 0 && r1 + 1 == v.m;      // whole-range shortcut (:181-183)
    const bool walk0 = p0 && !w0, walk1 = p1 && !w1;
    const uint32_t s0 = walk0 ? (uint32_t)c0 : 0u, s1 = walk1 ? (uint32_t)c1 : 0u;
    uint64_t i0 = walk0 ? l0 : 0, j0 = walk0 ? r0 + 1 : 0, i1 = walk1 ? l1 : 0, j1 = walk1 ? r1 + 1 : 0;
    NodeEntry e0 = load_node(v, 1), e1 = e0;
    for (uint32_t k = 0; k < L && (i0 | j0 | i1 | j1); ++k) {
        NodeEntry n0 = e0, n1 = e1;
        if (k + 1 < L) { n0 = load_node(v, (2u << k) + (s0 >> (L - 1 - k))); n1 = load_node(v, (2u << k) + (s1 >> (L - 1 - k))); }
        const uint64_t a0 = rank1(v, e0.base + i0) - e0.ones, b0 = rank1(v, e0.base + j0) - e0.ones;
        const uint64_t a1 = rank1(v, e1.base + i1) - e1.ones, b1 = rank1(v, e1.base + j1) - e1.ones;
        if ((s0 >> (L - 1 - k)) & 1) { i0 = a0; j0 = b0; } else { i0 -= a0; j0 -= b0; }
        if ((s1 >> (L - 1 - k)) & 1) { i1 = a1; j1 = b1; } else { i1 -= a1; j1 -= b1; }
        e0 = n0; e1 = n1;
    }
    if (!p0) { ol0 = 1; or0 = 0; } else if (w0) { ol0 = v.csym[c0]; or0 = v.csym[c0 + 1] - 1; } else { const uint64_t cb = v.csym[c0]; ol0 = cb + i0; or0 = cb + j0 - 1; }
    if (!p1) { ol1 = 1; or1 = 0; } else if (w1) { ol1 = v.csym[c1]; or1 = v.csym[c1 + 1] - 1; } else { const uint64_t cb = v.csym[c1]; ol1 = cb + i1; or1 = cb + j1 - 1; }
}

// Batched LF step (FMIndex::backward_search_step, fm_index.cpp:67-76): two triples per thread.
__global__ void __launch_bounds__(256) lf_step_kernel(FmView v, uint64_t n, const uint64_t* __restrict__ sym,
                                                      const uint64_t* __restrict__ lo,
                                                      const uint64_t* __restrict__ hi,
                                                      uint64_t* __restrict__ out_lo,
                                                      uint64_t* __restrict__ out_hi) {
    const uint64_t half = (n + 1) / 2;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < half; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t u = t + half;
        uint64_t l0, r0, l1, r1;
        if (u < n) {
            lf_step_pair(v, sym[t], lo[t], hi[t], sym[u], lo[u], hi[u], l0, r0, l1, r1);
            out_lo[u] = l1; out_hi[u] = r1;
        } else {
            lf_step(v, sym[t], lo[t], hi[t], l0, r0);
        }
        out_lo[t] = l0; out_hi[t] = r0;
    }
}

// FMIndex::backward_search_multi (fm_index.cpp:55-65): fold from (0, size()), return {l, r+1}.
__global__ void __launch_bounds__(128) lf_fold_kernel(FmView v, uint64_t nq, const uint64_t* __restrict__ symbols,
                                                      const uint64_t* __restrict__ offsets,
                                                      uint64_t* __restrict__ out_lo,
                                                      uint64_t* __restrict__ out_hi) {
    for (uint64_t q = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < nq; q += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t l = 0, r = v.m;
        for (uint64_t t = offsets[q]; t < offsets[q + 1]; ++t) lf_step(v, symbols[t], l, r, l, r);
        out_lo[q] = l;
        out_hi[q] = r + 1;
    }
}

constexpr int kExpandWarps = 4;
constexpr int kWideThreads = 256;

// dynamic shared memory of the two kernel shapes for a tree of height L
size_t narrow_smem(uint32_t L) { return kExpandWarps * warp_expand_smem(L); }

__device__ __forceinline__ WarpFrontier& warp_frontier(unsigned char* smem, uint32_t L, uint32_t warp, uint64_t*& stk) {
    unsigned char* base = smem + warp * warp_expand_smem(L);
    stk = reinterpret_cast<uint64_t*>(base + sizeof(WarpFrontier));
    return *reinterpret_cast<WarpFrontier*>(base);
}

// What a batch of SA ranges is expanded INTO: bitmask rows (the decode's allowed-token masks) or (symbol, count) pair lists.
struct MaskRows {
    uint32_t* mask; uint32_t ld_words, vocab, shift;
    __device__ void clear(uint64_t r, uint32_t lane) const { uint32_t* row = mask + r * ld_words; for (uint32_t w = lane; w < ld_words; w += 32) row[w] = 0; }
    __device__ MaskSink sink(uint64_t r) const { return MaskSink{mask + r * ld_words, vocab, shift}; }
};
struct PairRows {
    uint64_t* list; const uint64_t* list_off; unsigned int* counters; uint32_t* present; uint32_t present_words;
    __device__ void clear(uint64_t, uint32_t) const {}                      // counters / bitmaps are zeroed by one memset
    __device__ PairSink sink(uint64_t r) const { return PairSink{list + list_off[r], counters + r, present + r * (uint64_t)present_words}; }
};

// One warp per range; wide ranges are deferred to the block-cooperative kernel through a device-side list:
// wide_list[0] = number of wide rows found, [1] = work cursor of the wide kernel, [2..] = their indices.
template <typename Rows>
__global__ void __launch_bounds__(kExpandWarps * 32) expand_rows_kernel(FmView v, uint64_t R, const uint64_t* __restrict__ lo,
                                                                      const uint64_t* __restrict__ hi, Rows rows,
                                                                      unsigned long long* wide_list) {
    extern __shared__ __align__(16) unsigned char expand_smem[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t* stk;
    WarpFrontier& F = warp_frontier(expand_smem, v.L, warp, stk);
    for (uint64_t r = blockIdx.x * (uint64_t)kExpandWarps + warp; r < R; r += (uint64_t)gridDim.x * kExpandWarps) {
        rows.clear(r, lane);
        __syncwarp();
        const uint64_t l = lo[r], h = hi[r];
        if (h > l && h - l >= kWideRange) {
            if (lane == 0) { const unsigned long long k = atomicAdd(wide_list, 1ULL); wide_list[2 + k] = r; }
            continue;
        }
        auto sink = rows.sink(r);
        warp_expand(v, l, h, sink, F, stk);
        __syncwarp();
    }
}

// Persistent CTAs pull the wide rows found by expand_rows_kernel (no host sync) and expand each level-synchronously
// (block_expand_bfs); `scratch` = gridDim.x regions of global_frontier_bytes(L).
template <typename Rows>
__global__ void __launch_bounds__(kWideThreads) expand_rows_wide_kernel(FmView v, const uint64_t* __restrict__ lo,
                                                                       const uint64_t* __restrict__ hi, Rows rows,
                                                                       unsigned long long* wide_list, unsigned char* scratch) {
    __shared__ BlockFrontier F;
    __shared__ unsigned long long pick;
    const uint32_t cap = 1u << (v.L - 1);
    unsigned char* mine = scratch + (size_t)blockIdx.x * global_frontier_bytes(v.L);
    GlobalFrontier G;
    G.cap = cap;
    G.i = reinterpret_cast<uint64_t*>(mine); G.j = G.i + 2 * (size_t)cap; G.prefix = reinterpret_cast<uint32_t*>(G.j + 2 * (size_t)cap);
    const unsigned long long n = wide_list[0];
    for (;;) {
        if (threadIdx.x == 0) pick = atomicAdd(wide_list + 1, 1ULL);
        __syncthreads();
        const unsigned long long k = pick;
        __syncthreads();
        if (k >= n) break;
        const uint64_t r = wide_list[2 + k];
        auto sink = rows.sink(r);
        block_expand_bfs(v, lo[r], hi[r], sink, F, G);
    }
}

// Unordered (symbol, count) pairs + presence bitmap -> ascending-symbol pairs: the position of a symbol is the number
// of present symbols below it.  One CTA per range: block scan of the bitmap's popcounts, then a scatter.  The scan goes
// to `prefix`, global scratch of the bitmap's size (2^L / 8 bytes per range: beyond shared memory from L = 19 on).
__global__ void __launch_bounds__(256) order_pairs_kernel(uint32_t present_words, const uint32_t* __restrict__ present,
                                                          const unsigned int* __restrict__ counters,
                                                          const uint64_t* __restrict__ list, const uint64_t* __restrict__ list_off,
                                                          uint32_t* __restrict__ prefix,
                                                          uint64_t* __restrict__ out, uint64_t* __restrict__ out_len) {
    __shared__ uint32_t warp_tot[8];
    __shared__ uint32_t carry;
    const uint64_t r = blockIdx.x;
    const uint32_t* bm = present + r * (uint64_t)present_words;
    uint32_t* pre = prefix + r * (uint64_t)present_words;      // exclusive prefix of popcounts, present_words entries
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t w0 = 0; w0 < present_words; w0 += blockDim.x) {
        const uint32_t w = w0 + threadIdx.x;
        const uint32_t c = w < present_words ? __popc(bm[w]) : 0u;
        uint32_t incl = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (uint32_t)d) incl += t; }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        uint32_t woff = 0, tot = 0;
        for (uint32_t x = 0; x < blockDim.x / 32; ++x) { if (x < warp) woff += warp_tot[x]; tot += warp_tot[x]; }
        if (w < present_words) pre[w] = carry + woff + incl - c;
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
    const unsigned int k = counters[r];
    const uint64_t* src = list + list_off[r];
    uint64_t* dst = out + list_off[r];
    for (unsigned int p = threadIdx.x; p < k; p += blockDim.x) {
        const uint64_t sym = src[2ull * p], cnt = src[2ull * p + 1];
        const uint32_t pos = pre[sym >> 5] + __popc(bm[sym >> 5] & ((1u << (sym & 31)) - 1u));
        dst[2ull * pos] = sym; dst[2ull * pos + 1] = cnt;
    }
    if (threadIdx.x == 0) out_len[r] = 2ull * k;
}

// Measurement aid (sealfm_debug_sector_probe): independent random 32-byte sector reads over a buffer, eight in flight
// per thread -- the memory system's ceiling for the access pattern of a rank query, the denominator the LF kernel's
// beyond-L2 rate is compared with (a streaming-copy peak is not reachable with 32-byte random accesses).
__global__ void __launch_bounds__(256) sector_probe_kernel(const uint4* __restrict__ buf, uint64_t n_sectors, uint64_t n_loads,
                                                           uint64_t seed, unsigned long long* __restrict__ sink) {
    auto mix = [](uint64_t x) { x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31); };
    uint32_t acc = 0;
    // index = hash * n_sectors >> 64 (no 64-bit division: the probe must be bound by the loads, not by the index arithmetic)
    for (uint64_t t = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) * 8; t < n_loads; t += (uint64_t)gridDim.x * blockDim.x * 8) {
        uint4 a[8], b[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const uint64_t i = __umul64hi(mix(t + u + seed), n_sectors);
            a[u] = __ldg(buf + 2 * i); b[u] = __ldg(buf + 2 * i + 1);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) acc ^= a[u].x ^ b[u].w;
    }
    if (acc == 0xDEADBEEFu) atomicAdd(sink, 1ULL);              // keeps the loads alive
}

__global__ void __launch_bounds__(128) locate_kernel(FmView v, uint64_t n, const uint64_t* __restrict__ rows,
                                                     uint64_t* __restrict__ out, int want_doc) {
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t pos = locate_row(v, rows[t]);
        if (want_doc) pos = doc_of_pos(v, pos);
        out[t] = pos;
    }
}

__global__ void __launch_bounds__(64) extract_kernel(FmView v, uint64_t n, const uint64_t* __restrict__ begins,
                                                     const uint64_t* __restrict__ ends,
                                                     const uint64_t* __restrict__ offs, uint64_t* __restrict__ out) {
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x)
        extract_text(v, begins[t], ends[t], out + offs[t]);
}

// ------------------------------------------------------------------------------------------------
// host helpers
// ------------------------------------------------------------------------------------------------
int grid_for(uint64_t work_items, int per_block, int max_waves = 8) {
    uint64_t blocks = (work_items + per_block - 1) / per_block;
    uint64_t cap = (uint64_t)sm_count() * max_waves;       // multiples of the SM count (132 on H100 SXM)
    if (blocks > cap) blocks = cap;
    if (blocks == 0) blocks = 1;
    return (int)blocks;
}

template <typename T>
struct DevBuf {
    T* p = nullptr;
    explicit DevBuf(uint64_t n) { if (n) CUDA_CHECK(cudaMalloc(&p, n * sizeof(T))); }
    ~DevBuf() { if (p) cudaFree(p); }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
};

// Per-call view of the handle's staging area (see struct sealfm): a bump allocator over the mapped pinned buffer
// (small calls: the kernels read / write host memory directly, no copies) or the grow-only device buffer.
class Stage {
public:
    static constexpr size_t kMappedMax = 96 * 1024;
    // device_only: the kernels use atomics on the staged memory (not guaranteed on mapped host memory)
    Stage(const sealfm_t* h, size_t bytes_needed, bool device_only = false) : h_(h), lk_(h->stage_mu) {
        bytes_needed += 256;
        if (!h->stage_stream) CUDA_CHECK(cudaStreamCreateWithFlags(&h->stage_stream, cudaStreamNonBlocking));
        mapped_ = !device_only && bytes_needed <= kMappedMax;
        if (mapped_) {
            if (!h->pin_h) {
                CUDA_CHECK(cudaHostAlloc(&h->pin_h, kMappedMax, cudaHostAllocMapped));
                CUDA_CHECK(cudaHostGetDevicePointer(&h->pin_d, h->pin_h, 0));
                h->pin_bytes = kMappedMax;
            }
            cap_ = h->pin_bytes;
        } else {
            if (h->dev_bytes < bytes_needed) {
                if (h->dev_p) { CUDA_CHECK(cudaStreamSynchronize(h->stage_stream)); cudaFree(h->dev_p); h->dev_p = nullptr; h->dev_bytes = 0; }
                const size_t want = std::max(bytes_needed, (size_t)1 << 20);
                CUDA_CHECK(cudaMalloc(&h->dev_p, want));
                h->dev_bytes = want;
            }
            cap_ = h->dev_bytes;
        }
    }
    cudaStream_t stream() const { return h_->stage_stream; }
    // device-usable region of `bytes` (16-byte aligned); *host_alias (mapped mode only) is the same memory seen from the host
    void* reserve(size_t bytes, void** host_alias = nullptr) {
        const size_t off = used_;
        used_ = (used_ + bytes + 15) / 16 * 16;
        if (used_ > cap_) throw ApiError(SEALFM_ENOMEM, "internal: staging area too small");
        if (host_alias) *host_alias = mapped_ ? static_cast<char*>(h_->pin_h) + off : nullptr;
        return static_cast<char*>(mapped_ ? h_->pin_d : h_->dev_p) + off;
    }
    // input: a device-usable copy of src[0..bytes)
    void* put(const void* src, size_t bytes) {
        void* alias = nullptr;
        void* d = reserve(bytes, &alias);
        if (!bytes) return d;
        if (mapped_) std::memcpy(alias, src, bytes);
        else CUDA_CHECK(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, stream()));
        return d;
    }
    void zero(void* d, size_t bytes) {
        if (!bytes) return;
        if (mapped_) std::memset(static_cast<char*>(h_->pin_h) + (static_cast<char*>(d) - static_cast<char*>(h_->pin_d)), 0, bytes);
        else CUDA_CHECK(cudaMemsetAsync(d, 0, bytes, stream()));
    }
    // output: after sync(), dst holds the `bytes` at device-usable pointer d
    void get(void* dst, const void* d, size_t bytes) {
        if (!bytes) return;
        if (mapped_) pending_.push_back({dst, static_cast<const char*>(h_->pin_h) + (static_cast<const char*>(d) - static_cast<const char*>(h_->pin_d)), bytes});
        else CUDA_CHECK(cudaMemcpyAsync(dst, d, bytes, cudaMemcpyDeviceToHost, stream()));
    }
    void sync() {
        CUDA_CHECK(cudaStreamSynchronize(stream()));
        for (auto& p : pending_) std::memcpy(p.dst, p.src, p.bytes);
        pending_.clear();
    }
private:
    struct Pending { void* dst; const void* src; size_t bytes; };
    const sealfm_t* h_;
    std::unique_lock<std::mutex> lk_;
    bool mapped_ = false;
    size_t cap_ = 0, used_ = 0;
    std::vector<Pending> pending_;
};

void require_device(const sealfm_t* h) {
    if (!h) throw ApiError(SEALFM_EINVAL, "null handle");
    if (h->device < 0) throw ApiError(SEALFM_ENODEVICE, "index not bound to a CUDA device (call sealfm_to_device)");
    CUDA_CHECK(cudaSetDevice(h->device));
}

void upload(sealfm_t* h, int device) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        cudaGetLastError();
        throw ApiError(SEALFM_ENODEVICE, std::string("no CUDA device available: ") + cudaGetErrorString(e));
    }
    if (device < 0 || device >= count) throw ApiError(SEALFM_EINVAL, "bad device id");
    CUDA_CHECK(cudaSetDevice(device));
    const HostIndex& H = h->host;
    const uint32_t L = H.max_level;
    const uint64_t m = H.size;
    DeviceArrays A;
    make_device_arrays(H, A);
    const std::vector<uint64_t>& blk = A.blocks;
    const std::vector<uint64_t>& csym = A.csym;
    const std::vector<NodeEntry>& node_tab = A.node_tab;

    auto put = [&](const void* src, uint64_t bytes) -> void* {
        void* d = nullptr;
        CUDA_CHECK(cudaMalloc(&d, bytes ? bytes : 8));
        if (bytes) CUDA_CHECK(cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice));
        h->device_bytes += bytes;
        return d;
    };
    h->device_bytes = 0;
    h->d_blocks = put(blk.data(), blk.size() * 8);
    h->d_csym = (uint64_t*)put(csym.data(), csym.size() * 8);
    h->d_node_tab = (NodeEntry*)put(node_tab.data(), node_tab.size() * sizeof(NodeEntry));
    h->d_sa = (uint64_t*)put(H.sa_samples.data(), H.sa_samples.size() * 8);
    h->d_isa = (uint64_t*)put(H.isa_samples.data(), H.isa_samples.size() * 8);
    FmView& v = h->view;
    v.blocks = (const uint4*)h->d_blocks;
    v.csym = h->d_csym; v.node_tab = h->d_node_tab;
    v.sa_samples = h->d_sa; v.isa_samples = h->d_isa;
    v.n_isa = H.isa_samples.size();
    v.beginnings = nullptr; v.n_beginnings = 0;
    v.m = m; v.L = L;
    h->device = device;
    if (!h->beginnings.empty()) {
        h->d_beginnings = (uint64_t*)put(h->beginnings.data(), h->beginnings.size() * 8);
        v.beginnings = h->d_beginnings; v.n_beginnings = h->beginnings.size();
    }
}

void release_device(sealfm_t* h) {
    if (h->device < 0) return;
    cudaSetDevice(h->device);
    cudaFree(h->d_blocks); cudaFree(h->d_csym); cudaFree(h->d_node_tab);
    cudaFree(h->d_sa); cudaFree(h->d_isa); cudaFree(h->d_beginnings);
    h->d_blocks = nullptr; h->d_csym = nullptr; h->d_node_tab = nullptr;       // a later re-bind must not see (or free) these again
    h->d_sa = nullptr; h->d_isa = nullptr; h->d_beginnings = nullptr;
    h->view = FmView{};
    if (h->stage_stream) { cudaStreamSynchronize(h->stage_stream); cudaStreamDestroy(h->stage_stream); h->stage_stream = nullptr; }
    if (h->pin_h) { cudaFreeHost(h->pin_h); h->pin_h = nullptr; h->pin_d = nullptr; h->pin_bytes = 0; }
    if (h->dev_p) { cudaFree(h->dev_p); h->dev_p = nullptr; h->dev_bytes = 0; }
    h->device = -1;
}

}  // namespace

namespace sealb200 {
// CTAs of the wide kernel: four per SM, fewer when their global frontiers (global_frontier_bytes(L) each) would pass
// 1 GiB in all, and at least one (528 at L = 16 on 132 SMs; 3 at L = 24, whose frontiers take 320 MiB each)
static int wide_ctas_for(uint64_t R, uint32_t L) {
    const uint64_t by_mem = std::max<uint64_t>(1, ((uint64_t)1 << 30) / global_frontier_bytes(L));
    return (int)std::max<uint64_t>(1, std::min<uint64_t>(R, std::min<uint64_t>((uint64_t)sm_count() * 4, by_mem)));
}
// device scratch launch_expand_masks needs for R ranges on a tree of height L: the wide-row work list, then one global
// frontier per wide CTA
size_t expand_scratch_bytes(uint32_t L, uint64_t R) { return ((R + 2 + 1) / 2 * 2) * 8 + (size_t)wide_ctas_for(R, L) * global_frontier_bytes(L); }

// Bitmask rows of R SA ranges: narrow ranges by one warp each, wide ones (>= kWideRange rows) by whole CTAs pulling
// from a device-side work list.  `wide`: expand_scratch_bytes(L, R) of device scratch (work list + the wide CTAs' global
// frontiers).  Stream-ordered, no host synchronisation; also the tail of every decode step (generate.cu).
void launch_expand_masks(const FmView& v, cudaStream_t s, uint64_t R, const uint64_t* lo_d, const uint64_t* hi_d, uint32_t* mask_d,
                         uint32_t ld_words, uint32_t vocab, uint32_t shift, unsigned long long* wide) {
    if (v.L > kMaxLevels) throw ApiError(SEALFM_EINVAL, "wavelet tree higher than kMaxLevels");
    CUDA_CHECK(cudaMemsetAsync(wide, 0, 2 * sizeof(unsigned long long), s));
    const int ns = (int)narrow_smem(v.L);
    static int ns_set = 0;
    if (ns > ns_set) { CUDA_CHECK(cudaFuncSetAttribute(expand_rows_kernel<MaskRows>, cudaFuncAttributeMaxDynamicSharedMemorySize, ns)); ns_set = ns; }
    const MaskRows rows{mask_d, ld_words, vocab, shift};
    expand_rows_kernel<MaskRows><<<grid_for(R, kExpandWarps, 16), kExpandWarps * 32, ns, s>>>(v, R, lo_d, hi_d, rows, wide);
    CUDA_CHECK(cudaGetLastError());
    expand_rows_wide_kernel<MaskRows><<<wide_ctas_for(R, v.L), kWideThreads, 0, s>>>(v, lo_d, hi_d, rows, wide,
                                                                              reinterpret_cast<unsigned char*>(wide + (R + 2 + 1) / 2 * 2));
    CUDA_CHECK(cudaGetLastError());
}

FmView sealfm_view(const sealfm_t* h) {
    if (!h) throw ApiError(SEALFM_EINVAL, "null handle");
    if (h->device < 0) throw ApiError(SEALFM_ENODEVICE, "index not bound to a CUDA device (call sealfm_to_device)");
    return h->view;
}

cudaStream_t sealfm_stream(const sealfm_t* h) {
    require_device(h);
    std::lock_guard<std::mutex> lk(h->stage_mu);
    if (!h->stage_stream) CUDA_CHECK(cudaStreamCreateWithFlags(&h->stage_stream, cudaStreamNonBlocking));
    return h->stage_stream;
}

const std::vector<uint64_t>& sealfm_beginnings(const sealfm_t* h) {
    if (!h) throw ApiError(SEALFM_EINVAL, "null handle");
    return h->beginnings;
}
}  // namespace sealb200

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

const char* sealfm_last_error(void) { return last_error().c_str(); }
int sealfm_abi_version(void) { return 3; }

int sealfm_build(const uint64_t* symbols, uint64_t n, sealfm_t** out) {
    return guarded([&] {
        if (!out || (!symbols && n)) throw ApiError(SEALFM_EINVAL, "null argument");
        std::unique_ptr<sealfm> h(new sealfm());
        build_index(symbols, n, h->host);
        *out = h.release();
    });
}
int sealfm_build_gpu(const uint64_t* symbols, uint64_t n, int device, sealfm_t** out) {
    return guarded([&] {
        if (!out || (!symbols && n)) throw ApiError(SEALFM_EINVAL, "null argument");
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
            cudaGetLastError();
            throw ApiError(SEALFM_ENODEVICE, "no such CUDA device");
        }
        std::unique_ptr<sealfm> h(new sealfm());
        build_index_gpu(symbols, n, device, h->host);
        *out = h.release();
    });
}
int sealfm_build_gpu_ex(const void* symbols, uint64_t n, int width_bytes, int device, const sealfm_build_opts_t* opts,
                        sealfm_t** out) {
    return guarded([&] {
        if (!out) throw ApiError(SEALFM_EINVAL, "null argument");
        *out = nullptr;
        if (!symbols && n) throw ApiError(SEALFM_EINVAL, "null argument");
        if (width_bytes != 4 && width_bytes != 8) throw ApiError(SEALFM_EINVAL, "width must be 4 or 8 bytes");
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
            cudaGetLastError();
            throw ApiError(SEALFM_ENODEVICE, "no such CUDA device");
        }
        std::unique_ptr<sealfm> h(new sealfm());
        build_index_gpu_large(symbols, n, width_bytes, device, opts, h->host);
        *out = h.release();
    });
}
int sealfm_build_gpu_ex_stats(sealfm_build_stats_t* out) {
    return guarded([&] {
        if (!out) throw ApiError(SEALFM_EINVAL, "null argument");
        *out = build_gpu_large_last_stats();
    });
}
int sealfm_build_from_file(const char* path, int width_bytes, sealfm_t** out) {
    return guarded([&] {
        if (!out || !path) throw ApiError(SEALFM_EINVAL, "null argument");
        std::unique_ptr<sealfm> h(new sealfm());
        try { build_index_from_file(path, width_bytes, h->host); }
        catch (const std::runtime_error& e) { throw ApiError(SEALFM_EIO, e.what()); }
        *out = h.release();
    });
}
int sealfm_load(const char* path, sealfm_t** out) {
    return guarded([&] {
        if (!out || !path) throw ApiError(SEALFM_EINVAL, "null argument");
        std::unique_ptr<sealfm> h(new sealfm());
        try { load_index(path, h->host); }
        catch (const std::runtime_error& e) { throw ApiError(SEALFM_EIO, e.what()); }
        *out = h.release();
    });
}
int sealfm_save(const sealfm_t* h, const char* path) {
    return guarded([&] {
        if (!h || !path) throw ApiError(SEALFM_EINVAL, "null argument");
        try { save_index_native(h->host, path); }
        catch (const std::runtime_error& e) { throw ApiError(SEALFM_EIO, e.what()); }
    });
}
int sealfm_save_sdsl(const sealfm_t* h, const char* path) {
    return guarded([&] {
        if (!h || !path) throw ApiError(SEALFM_EINVAL, "null argument");
        try { save_index_sdsl(h->host, path); }
        catch (const std::runtime_error& e) { throw ApiError(SEALFM_EIO, e.what()); }
    });
}
void sealfm_free(sealfm_t* h) {
    if (!h) return;
    release_device(h);
    delete h;
}
uint64_t sealfm_size(const sealfm_t* h) { return h ? h->host.size : 0; }
uint64_t sealfm_sigma(const sealfm_t* h) { return h ? h->host.sigma : 0; }
uint32_t sealfm_max_level(const sealfm_t* h) { return h ? h->host.max_level : 0; }

int sealfm_section(const sealfm_t* h, int which, const uint64_t** ptr, uint64_t* n_words) {
    return guarded([&] {
        if (!h || !ptr || !n_words) throw ApiError(SEALFM_EINVAL, "null argument");
        const std::vector<uint64_t>* v = nullptr;
        switch (which) {
            case 0: v = &h->host.tree; break;
            case 1: v = &h->host.alphabet; break;
            case 2: v = &h->host.C; break;
            case 3: v = &h->host.sa_samples; break;
            case 4: v = &h->host.isa_samples; break;
            default: throw ApiError(SEALFM_EINVAL, "unknown section");
        }
        *ptr = v->data(); *n_words = v->size();
    });
}

int sealfm_to_device(sealfm_t* h, int device) {
    return guarded([&] {
        if (!h) throw ApiError(SEALFM_EINVAL, "null handle");
        if (h->device >= 0) release_device(h);
        upload(h, device);
    });
}
int sealfm_device(const sealfm_t* h) { return h ? h->device : -1; }
uint64_t sealfm_device_bytes(const sealfm_t* h) { return h ? h->device_bytes : 0; }

int sealfm_set_beginnings(sealfm_t* h, const uint64_t* beginnings, uint64_t n) {
    return guarded([&] {
        if (!h || (!beginnings && n)) throw ApiError(SEALFM_EINVAL, "null argument");
        h->beginnings.assign(beginnings, beginnings + n);
        if (h->device >= 0) {
            CUDA_CHECK(cudaSetDevice(h->device));
            if (h->d_beginnings) { cudaFree(h->d_beginnings); h->d_beginnings = nullptr; }
            CUDA_CHECK(cudaMalloc(&h->d_beginnings, (n ? n : 1) * 8));
            CUDA_CHECK(cudaMemcpy(h->d_beginnings, beginnings, n * 8, cudaMemcpyHostToDevice));
            h->view.beginnings = h->d_beginnings; h->view.n_beginnings = n;
        }
    });
}

int sealfm_backward_search_step_d(const sealfm_t* h, sealfm_stream_t stream, uint64_t n,
                                  const uint64_t* sym_d, const uint64_t* lo_d, const uint64_t* hi_d,
                                  uint64_t* out_lo_d, uint64_t* out_hi_d) {
    return guarded([&] {
        require_device(h);
        if (!n) return;
        lf_step_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(h->view, n, sym_d, lo_d, hi_d, out_lo_d, out_hi_d);
        CUDA_CHECK(cudaGetLastError());
    });
}

int sealfm_expand_mask_d(const sealfm_t* h, sealfm_stream_t stream, uint64_t R, const uint64_t* lo_d,
                         const uint64_t* hi_d, uint32_t* mask_d, uint32_t ld_words, uint32_t vocab,
                         uint32_t shift) {
    return guarded([&] {
        require_device(h);
        if (!R) return;
        if ((uint64_t)ld_words * 32 < vocab) throw ApiError(SEALFM_EINVAL, "ld_words too small for vocab");
        cudaStream_t s = (cudaStream_t)stream;
        unsigned long long* wide = nullptr;                    // [count, cursor, rows...] + the wide CTAs' global frontiers
        // the scratch is hundreds of MB for large R: keep freed blocks in the device's stream-ordered pool instead of
        // returning them to the driver at every synchronisation (the default release threshold is 0)
        static bool pool_kept = false;
        if (!pool_kept) {
            cudaMemPool_t pool = nullptr;
            if (cudaDeviceGetDefaultMemPool(&pool, h->device) == cudaSuccess) {
                uint64_t keep = ~0ull;
                cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
            }
            cudaGetLastError();
            pool_kept = true;
        }
        CUDA_CHECK(cudaMallocAsync(&wide, expand_scratch_bytes(h->view.L, R), s));
        struct Free { unsigned long long* p; cudaStream_t s; ~Free() { cudaFreeAsync(p, s); } } guard{wide, s};
        launch_expand_masks(h->view, s, R, lo_d, hi_d, mask_d, ld_words, vocab, shift, wide);
    });
}

int sealfm_backward_search_step(const sealfm_t* h, uint64_t n, const uint64_t* sym, const uint64_t* lo,
                                const uint64_t* hi, uint64_t* out_lo, uint64_t* out_hi) {
    return guarded([&] {
        require_device(h);
        if (!n) return;
        Stage st(h, 5 * n * 8 + 128);
        const uint64_t* ds = (const uint64_t*)st.put(sym, n * 8);
        const uint64_t* dl = (const uint64_t*)st.put(lo, n * 8);
        const uint64_t* dh = (const uint64_t*)st.put(hi, n * 8);
        uint64_t* ol = (uint64_t*)st.reserve(n * 8); uint64_t* oh = (uint64_t*)st.reserve(n * 8);
        lf_step_kernel<<<grid_for((n + 1) / 2, 256), 256, 0, st.stream()>>>(h->view, n, ds, dl, dh, ol, oh);
        CUDA_CHECK(cudaGetLastError());
        st.get(out_lo, ol, n * 8); st.get(out_hi, oh, n * 8);
        st.sync();
    });
}

int sealfm_backward_search_multi(const sealfm_t* h, uint64_t nq, const uint64_t* symbols,
                                 const uint64_t* offsets, uint64_t* out_lo, uint64_t* out_hi) {
    return guarded([&] {
        require_device(h);
        if (!nq) return;
        const uint64_t tot = offsets[nq];
        Stage st(h, (tot + 3 * nq + 1) * 8 + 128);
        const uint64_t* ds = (const uint64_t*)st.put(symbols, tot * 8);
        const uint64_t* doff = (const uint64_t*)st.put(offsets, (nq + 1) * 8);
        uint64_t* ol = (uint64_t*)st.reserve(nq * 8); uint64_t* oh = (uint64_t*)st.reserve(nq * 8);
        lf_fold_kernel<<<grid_for(nq, 128), 128, 0, st.stream()>>>(h->view, nq, ds, doff, ol, oh);
        CUDA_CHECK(cudaGetLastError());
        st.get(out_lo, ol, nq * 8); st.get(out_hi, oh, nq * 8);
        st.sync();
    });
}

int sealfm_distinct_count_multi(const sealfm_t* h, uint64_t n, const uint64_t* lows, const uint64_t* highs,
                                uint64_t* out_offsets, uint64_t* out, uint64_t out_cap) {
    return guarded([&] {
        require_device(h);
        if (!out_offsets || (!lows && n) || (!highs && n)) throw ApiError(SEALFM_EINVAL, "null argument");
        const uint32_t L = h->host.max_level;
        if (L > kMaxLevels) throw ApiError(SEALFM_EINVAL, "wavelet tree higher than kMaxLevels");
        const uint64_t nsym = 1ULL << L;
        const uint32_t words = (uint32_t)((nsym + 31) / 32);
        // upper bound on the pairs of a range: its width, or the alphabet (hi == size()+1 is reachable through the
        // reference's first-step quirk, SURVEY.md H1; the arithmetic below is the reference's own for such a range)
        std::vector<uint64_t> ub(n + 1, 0);
        for (uint64_t i = 0; i < n; ++i) {
            if (highs[i] > h->host.size + 1) throw ApiError(SEALFM_EINVAL, "range end beyond size()+1");
            const uint64_t k = highs[i] > lows[i] ? std::min<uint64_t>(highs[i] - lows[i], nsym) : 0;
            ub[i + 1] = ub[i] + 2 * k;
        }
        std::vector<uint64_t> lens(n, 0), tmp;
        out_offsets[0] = 0;
        const uint64_t kChunkPairs = 1ULL << 24;                // u64 of list scratch per pass (2 x 128 MB at most)
        // presence bitmaps per pass (2^L / 8 bytes per range, and as much again for their prefix): 4 096 ranges up to
        // L = 18, 64 at L = 24
        const uint64_t kChunkBitmapBytes = 1ULL << 27;
        const int ns = (int)narrow_smem(L);
        CUDA_CHECK(cudaFuncSetAttribute(expand_rows_kernel<PairRows>, cudaFuncAttributeMaxDynamicSharedMemorySize, ns));
        uint64_t written = 0;
        for (uint64_t c0 = 0; c0 < n;) {
            uint64_t c1 = c0 + 1;
            while (c1 < n && ub[c1 + 1] - ub[c0] <= kChunkPairs && c1 - c0 < 4096 && (c1 + 1 - c0) * words * 4 <= kChunkBitmapBytes) ++c1;
            const uint64_t cn = c1 - c0, pairs = ub[c1] - ub[c0];
            std::vector<uint64_t> off(cn + 1);
            for (uint64_t i = 0; i <= cn; ++i) off[i] = ub[c0 + i] - ub[c0];
            const size_t cnt_bytes = (cn * 4 + 15) / 16 * 16, present_bytes = ((size_t)cn * words * 4 + 15) / 16 * 16;     // 16-byte aligned regions
            const size_t wide_bytes = ((cn + 2 + 1) / 2 * 2) * 8;
            const size_t zero_bytes = cnt_bytes + present_bytes + wide_bytes;
            const size_t bfs_bytes = (size_t)wide_ctas_for(cn, L) * global_frontier_bytes(L);
            Stage st(h, (2 * cn + cn + 1 + 2 * pairs + cn) * 8 + zero_bytes + present_bytes + bfs_bytes + 512, true);
            const uint64_t* dlo = (const uint64_t*)st.put(lows + c0, cn * 8);
            const uint64_t* dhi = (const uint64_t*)st.put(highs + c0, cn * 8);
            const uint64_t* doff = (const uint64_t*)st.put(off.data(), (cn + 1) * 8);
            uint64_t* dlist = (uint64_t*)st.reserve(pairs * 8); uint64_t* dout = (uint64_t*)st.reserve(pairs * 8);
            uint64_t* dlen = (uint64_t*)st.reserve(cn * 8);
            char* z = (char*)st.reserve(zero_bytes);
            st.zero(z, zero_bytes);
            unsigned int* dcnt = (unsigned int*)z;
            uint32_t* dpresent = (uint32_t*)(z + cnt_bytes);
            unsigned long long* dwide = (unsigned long long*)(z + cnt_bytes + present_bytes);
            const PairRows rows{dlist, doff, dcnt, dpresent, words};
            expand_rows_kernel<PairRows><<<grid_for(cn, kExpandWarps, 16), kExpandWarps * 32, ns, st.stream()>>>(h->view, cn, dlo, dhi, rows, dwide);
            CUDA_CHECK(cudaGetLastError());
            unsigned char* dbfs = (unsigned char*)st.reserve(bfs_bytes);
            expand_rows_wide_kernel<PairRows><<<wide_ctas_for(cn, L), kWideThreads, 0, st.stream()>>>(h->view, dlo, dhi, rows, dwide, dbfs);
            CUDA_CHECK(cudaGetLastError());
            uint32_t* dprefix = (uint32_t*)st.reserve(present_bytes);
            order_pairs_kernel<<<(unsigned)cn, 256, 0, st.stream()>>>(words, dpresent, dcnt, dlist, doff, dprefix, dout, dlen);
            CUDA_CHECK(cudaGetLastError());
            st.get(lens.data() + c0, dlen, cn * 8);
            if (out) { tmp.resize(pairs); st.get(tmp.data(), dout, pairs * 8); }
            st.sync();
            for (uint64_t i = 0; i < cn; ++i) {
                const uint64_t len = lens[c0 + i];
                out_offsets[c0 + i + 1] = out_offsets[c0 + i] + len;
                if (out && len) {
                    if (written + len > out_cap) throw ApiError(SEALFM_ECAPACITY, "output buffer too small");
                    std::memcpy(out + written, tmp.data() + off[i], len * 8);
                }
                written += len;
            }
            c0 = c1;
        }
    });
}

static int locate_impl(const sealfm_t* h, uint64_t n, const uint64_t* rows, uint64_t* out, int want_doc) {
    return guarded([&] {
        require_device(h);
        if (!n) return;
        if (want_doc && !h->view.beginnings) throw ApiError(SEALFM_EINVAL, "sealfm_set_beginnings not called");
        Stage st(h, 2 * n * 8 + 128);
        const uint64_t* dr = (const uint64_t*)st.put(rows, n * 8);
        uint64_t* dout = (uint64_t*)st.reserve(n * 8);
        locate_kernel<<<grid_for(n, 128), 128, 0, st.stream()>>>(h->view, n, dr, dout, want_doc);
        CUDA_CHECK(cudaGetLastError());
        st.get(out, dout, n * 8);
        st.sync();
    });
}
int sealfm_locate(const sealfm_t* h, uint64_t n, const uint64_t* rows, uint64_t* out_pos) {
    return locate_impl(h, n, rows, out_pos, 0);
}
int sealfm_doc_index_from_rows(const sealfm_t* h, uint64_t n, const uint64_t* rows, uint64_t* out_doc) {
    return locate_impl(h, n, rows, out_doc, 1);
}

int sealfm_extract_text(const sealfm_t* h, uint64_t n, const uint64_t* begins, const uint64_t* ends,
                        uint64_t* out_offsets, uint64_t* out, uint64_t out_cap) {
    return guarded([&] {
        require_device(h);
        if (!out_offsets) throw ApiError(SEALFM_EINVAL, "null argument");
        out_offsets[0] = 0;
        for (uint64_t i = 0; i < n; ++i) {
            if (ends[i] >= h->host.size || begins[i] > ends[i]) throw ApiError(SEALFM_EINVAL, "bad text interval");
            out_offsets[i + 1] = out_offsets[i] + (ends[i] - begins[i]);
        }
        if (!out || !n) return;
        const uint64_t tot = out_offsets[n];
        if (tot > out_cap) throw ApiError(SEALFM_ECAPACITY, "output buffer too small");
        Stage st(h, (3 * n + 1 + tot) * 8 + 128);
        const uint64_t* db = (const uint64_t*)st.put(begins, n * 8);
        const uint64_t* de = (const uint64_t*)st.put(ends, n * 8);
        const uint64_t* doff = (const uint64_t*)st.put(out_offsets, (n + 1) * 8);
        uint64_t* dout = (uint64_t*)st.reserve(tot * 8);
        extract_kernel<<<grid_for(n, 64), 64, 0, st.stream()>>>(h->view, n, db, de, doff, dout);
        CUDA_CHECK(cudaGetLastError());
        st.get(out, dout, tot * 8);
        st.sync();
    });
}

/* Measurement aid: `n_loads` independent random 32-byte sector reads over a zero-filled device buffer of `buffer_bytes`
 * (8 in flight per thread); average device time per pass over `iters` passes (CUDA events). */
int sealfm_debug_sector_probe(uint64_t buffer_bytes, uint64_t n_loads, int iters, double* avg_us) {
    return guarded([&] {
        if (!avg_us || buffer_bytes < 64 || !n_loads || iters < 1) throw ApiError(SEALFM_EINVAL, "bad argument");
        int count = 0;
        if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) { cudaGetLastError(); throw ApiError(SEALFM_ENODEVICE, "no CUDA device available"); }
        DevBuf<uint8_t> buf(buffer_bytes);
        DevBuf<unsigned long long> sink(1);
        CUDA_CHECK(cudaMemset(buf.p, 0, buffer_bytes));
        CUDA_CHECK(cudaMemset(sink.p, 0, 8));
        const uint64_t n_sectors = buffer_bytes / 32;
        const int grid = sm_count() * 8;                       // 2 048 threads per SM x 8 sectors each in flight
        sector_probe_kernel<<<grid, 256>>>((const uint4*)buf.p, n_sectors, n_loads, 1, sink.p);
        cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0));
        for (int i = 0; i < iters; ++i) sector_probe_kernel<<<grid, 256>>>((const uint4*)buf.p, n_sectors, n_loads, 7919ull * (i + 2), sink.p);
        CUDA_CHECK(cudaEventRecord(e1));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *avg_us = (double)ms * 1e3 / iters;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    });
}

/* An index whose sections were computed elsewhere (same content sealfm_section hands out). */
int sealfm_from_sections(uint64_t size, uint32_t max_level, uint64_t sigma, const uint64_t* tree, uint64_t n_tree,
                         const uint64_t* alphabet, const uint64_t* C, const uint64_t* sa_samples, uint64_t n_sa,
                         const uint64_t* isa_samples, uint64_t n_isa, sealfm_t** out) {
    return guarded([&] {
        if (!out || !tree || !alphabet || !C || !sa_samples || !isa_samples) throw ApiError(SEALFM_EINVAL, "null argument");
        if (!size || !max_level || max_level > kMaxLevels || !sigma) throw ApiError(SEALFM_EINVAL, "bad size / max_level / sigma");
        const uint64_t bits = size * (uint64_t)max_level;
        if (n_tree != (bits + 63) / 64) throw ApiError(SEALFM_EINVAL, "tree must hold size * max_level bits");
        if (n_sa != (size + 31) / 32 || n_isa != (size - 1) / 64 + 1) throw ApiError(SEALFM_EINVAL, "sample arrays have the wrong length");
        std::unique_ptr<sealfm> h(new sealfm());
        HostIndex& H = h->host;
        H.size = size; H.max_level = max_level; H.sigma = sigma;
        H.tree.assign(tree, tree + n_tree);
        H.alphabet.assign(alphabet, alphabet + sigma);
        H.C.assign(C, C + sigma + 1);
        H.sa_samples.assign(sa_samples, sa_samples + n_sa);
        H.isa_samples.assign(isa_samples, isa_samples + n_isa);
        *out = h.release();
    });
}

}  // extern "C"
