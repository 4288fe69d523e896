// Index construction on the GPU for texts beyond fm_build.cu's reach (m = n + 1 up to 2^40 - 1): the same HostIndex
// the host SA-IS builder returns, with the suffix array streamed through pinned host memory.
//
// Suffix sort: in-place prefix doubling with Larsson-Sadakane labels.  A suffix's label is the first suffix-array row
// of its group; the inverse suffix array (ISA = labels) stays on the device, the suffix array (SA) in pinned host
// memory.  Round 0 sorts by the first symbol; the round with step h sorts every unsorted group by ISA[i + h].  Keys
// may read labels refined earlier in the same round: labels only refine (a new label lies inside its old group's row
// interval), so any order of keys seen at some moment of the round is consistent with the true suffix order, and
// equal keys still mean an equal 2h-prefix.  Since every suffix is unique, the groups end as singletons, ISA = rank,
// and the SA is the one SA-IS computes.
//
// Each round walks a host list of unsorted ranges (runs of groups of size > 1, merged across short sorted gaps) in
// windows of W rows.  A window starts on a group's first row and is cut before a group that crosses its far edge; it
// is sorted on the device by (label - window start, key) with one radix sort, relabelled, scattered into the ISA and
// written back.  A group larger than W is split by key range in place, on a snapshot of its keys: a min/max and a
// histogram pass pick a splitter, a streamed two-way partition moves the rows to their side, and each side is split
// again until it fits a window or holds a single key (a new group as a whole: relabelled, not sorted).
//
// Then BWT[i] = text[SA[i] - 1] and the SA samples stream out of the host SA once, the ISA samples come from the
// final labels, and the wavelet tree is built level by level as in fm_build.cu.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <chrono>
#include <cstring>
#include <thread>
#include <vector>

#include "common.cuh"
#include "fm_build_common.cuh"
#include "fm_host.hpp"
#include "../../include/sealfm.h"

namespace sealb200 {
namespace {

constexpr int kBins = 2048;                 // histogram bins of a key-range split
constexpr uint64_t kMergeGap = 64;          // sorted rows between two unsorted ranges that are re-sorted rather than skipped
constexpr uint32_t kMaxRounds = 48;         // round 0 + at most 41 doublings for m < 2^40
constexpr uint64_t kMaxM = 1ULL << 40;

struct DevTracker { uint64_t cur = 0, peak = 0; };

// device buffer whose bytes count towards the builder's peak; cudaMalloc failures are SEALFM_ENOMEM
template <typename T>
struct Buf {
    T* p = nullptr;
    uint64_t n = 0;
    DevTracker* tr = nullptr;
    void alloc(DevTracker& t, uint64_t count) {
        release();
        tr = &t;
        if (!count) return;
        cudaError_t e = cudaMalloc(&p, count * sizeof(T));
        if (e != cudaSuccess) {
            cudaGetLastError(); p = nullptr;
            throw ApiError(SEALFM_ENOMEM, std::string("device allocation failed: ") + cudaGetErrorString(e));
        }
        n = count;
        t.cur += bytes(); t.peak = std::max(t.peak, t.cur);
    }
    uint64_t bytes() const { return n * sizeof(T); }
    void release() {
        if (p) { cudaFree(p); tr->cur -= bytes(); }
        p = nullptr; n = 0;
    }
    ~Buf() { release(); }
};

struct Pinned {
    void* p = nullptr;
    ~Pinned() { if (p) cudaFreeHost(p); }
};

// sort key of suffix x in the current round: its first symbol in round 0 (h = 0), else the label of suffix x + h
// ("past the end" only happens for singleton groups, whose order does not matter)
template <typename T>
struct KeySrc {
    const T* isa;
    const void* text;
    int text16;
    uint64_t m, h;
    uint64_t flo, fhi;                 // labels in [flo, fhi) read as flo: the key snapshot of a group being split
    __device__ __forceinline__ uint64_t operator()(uint64_t x) const {
        if (h == 0) return text16 ? (uint64_t)static_cast<const uint16_t*>(text)[x] : (uint64_t)static_cast<const uint32_t*>(text)[x];
        const uint64_t k = x + h < m ? (uint64_t)isa[x + h] : 0;
        return k >= flo && k < fhi ? flo : k;
    }
};

template <typename T>
__global__ void __launch_bounds__(kBT) window_keys_kernel(const T* __restrict__ sa, uint64_t n, KeySrc<T> ks, int by_group,
                                                           uint64_t a, uint32_t kb, uint64_t* __restrict__ key) {
    GRID_STRIDE(j, n) {
        const uint64_t x = sa[j];
        uint64_t k = ks(x);
        if (by_group) k |= ((uint64_t)ks.isa[x] - a) << kb;
        key[j] = k;
    }
}

// start[j] candidates: j where the sorted key changes, else 0 (an inclusive max-scan turns them into group starts)
__global__ void __launch_bounds__(kBT) group_head_kernel(const uint64_t* __restrict__ key, uint64_t* __restrict__ head, uint64_t n) {
    GRID_STRIDE(j, n) head[j] = (j == 0 || key[j] != key[j - 1]) ? j : 0;
}

struct MaxOp {
    __device__ __forceinline__ uint64_t operator()(uint64_t a, uint64_t b) const { return a > b ? a : b; }
};

// new labels into the ISA; edge[j] (j in [0, n]) marks where membership of a group of size > 1 changes, so the
// selected edges alternate run start / run end; first[j] marks group starts (round 0: alphabet and C)
template <typename T>
__global__ void __launch_bounds__(kBT) relabel_kernel(const T* __restrict__ sa, const uint64_t* __restrict__ start, uint64_t n,
                                                       uint64_t a, T* __restrict__ isa, uint8_t* __restrict__ edge,
                                                       uint8_t* __restrict__ first) {
    GRID_STRIDE(j, n + 1) {
        auto multi = [&](uint64_t i) -> bool {            // row i's group has more than one row
            if (i >= n) return false;
            return start[i] != i || (i + 1 < n && start[i + 1] == i);
        };
        edge[j] = multi(j) != (j > 0 && multi(j - 1));
        if (j < n) {
            isa[sa[j]] = (T)(a + start[j]);
            first[j] = start[j] == j;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kBT) set_label_kernel(const T* __restrict__ sa, uint64_t n, T label, T* __restrict__ isa) {
    GRID_STRIDE(j, n) isa[sa[j]] = label;
}

__device__ __forceinline__ uint64_t warp_min(uint64_t v) {
    for (int o = 16; o; o >>= 1) { uint64_t w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
    return v;
}
__device__ __forceinline__ uint64_t warp_max(uint64_t v) {
    for (int o = 16; o; o >>= 1) { uint64_t w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
    return v;
}

// mm[0] = min, mm[1] = max of the keys of n rows
template <typename T>
__global__ void __launch_bounds__(kBT) minmax_kernel(const T* __restrict__ sa, uint64_t n, KeySrc<T> ks, unsigned long long* mm) {
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t j = base + threadIdx.x;
        const bool v = j < n;
        const uint64_t k = v ? ks(sa[j]) : 0;
        const uint64_t lo = warp_min(v ? k : ~0ULL), hi = warp_max(v ? k : 0);
        if ((threadIdx.x & 31) == 0) { atomicMin(mm, (unsigned long long)lo); atomicMax(mm + 1, (unsigned long long)hi); }
    }
}

// hist[b] += rows with (key - mn) / w == b; hist[nb] += rows with key == mn, hist[nb + 1] += rows with key == mx
template <typename T>
__global__ void __launch_bounds__(kBT) hist_kernel(const T* __restrict__ sa, uint64_t n, KeySrc<T> ks, uint64_t mn, uint64_t mx,
                                                    uint64_t w, uint32_t nb, unsigned long long* hist) {
    __shared__ uint32_t sh[kBins + 2];
    for (uint32_t i = threadIdx.x; i < nb + 2; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    for (uint64_t base = blockIdx.x * (uint64_t)blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t j = base + threadIdx.x;
        const bool v = j < n;
        const uint64_t k = v ? ks(sa[j]) : 0;
        if (v) atomicAdd(&sh[(k - mn) / w], 1u);
        const uint32_t bmin = __ballot_sync(0xffffffffu, v && k == mn), bmax = __ballot_sync(0xffffffffu, v && k == mx);
        if ((threadIdx.x & 31) == 0) {
            if (bmin) atomicAdd(&sh[nb], (uint32_t)__popc(bmin));
            if (bmax) atomicAdd(&sh[nb + 1], (uint32_t)__popc(bmax));
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nb + 2; i += blockDim.x)
        if (sh[i]) atomicAdd(hist + i, (unsigned long long)sh[i]);
}

template <typename T>
__global__ void __launch_bounds__(kBT) below_kernel(const T* __restrict__ sa, uint64_t n, KeySrc<T> ks, uint64_t t, int want,
                                                     uint8_t* __restrict__ flag) {
    GRID_STRIDE(j, n) flag[j] = (ks(sa[j]) < t) == (want != 0);
}

// exchanges the f misplaced rows of the left window (device copy, rows lpos - l0) with f rows of the right side,
// which are read and written in place in mapped host memory
template <typename T>
__global__ void __launch_bounds__(kBT) swap_kernel(T* __restrict__ lwin, const uint64_t* __restrict__ lpos, uint64_t l0,
                                                    const uint64_t* __restrict__ rpos, T* host_sa, uint64_t f) {
    GRID_STRIDE(i, f) {
        const uint64_t li = lpos[i] - l0, ri = rpos[i];
        const T r = host_sa[ri];
        host_sa[ri] = lwin[li];
        lwin[li] = r;
    }
}

template <typename T>
__global__ void __launch_bounds__(kBT) iota_window_kernel(T* v, uint64_t a, uint64_t n) { GRID_STRIDE(j, n) v[j] = (T)(a + j); }

template <typename S, typename D>
__global__ void __launch_bounds__(kBT) narrow_kernel(const S* __restrict__ src, D* __restrict__ dst, uint64_t n) {
    GRID_STRIDE(j, n) dst[j] = (D)src[j];
}

template <typename T, typename X>
__global__ void __launch_bounds__(kBT) bwt_window_kernel(const T* __restrict__ sa, uint64_t a, uint64_t n, const X* __restrict__ text,
                                                          uint32_t* __restrict__ bwt, uint64_t* __restrict__ sa_samples) {
    GRID_STRIDE(j, n) {
        const uint64_t i = a + j, p = sa[j];
        bwt[i] = p ? (uint32_t)text[p - 1] : 0u;          // SA[i] = 0: the sentinel, text[m - 1]
        if ((i & 31) == 0) sa_samples[i >> 5] = p;
    }
}

template <typename T>
__global__ void __launch_bounds__(kBT) isa_samples_kernel(const T* __restrict__ isa, uint64_t* __restrict__ out, uint64_t n_isa) {
    GRID_STRIDE(k, n_isa) out[k] = isa[k << 6];
}

using Clock = std::chrono::steady_clock;
inline double secs(Clock::time_point a) { return std::chrono::duration<double>(Clock::now() - a).count(); }

thread_local sealfm_build_stats_t g_last_stats{};

struct Range { uint64_t s, e; };

// bytes of the device window for W rows with positions of `w` bytes: sa x2, keys x2, two u64 scratch rows, two flag rows
inline uint64_t window_row_bytes(int w) { return 2ull * w + 4 * 8 + 2; }

template <typename T>
class LargeBuilder {
public:
    LargeBuilder(const void* sym, uint64_t n, int width, uint32_t max_sym, int device, uint64_t budget, uint64_t W,
                 sealfm_build_stats_t& st)
        : sym_(sym), n_(n), m_(n + 1), width_(width), max_sym_(max_sym), device_(device), budget_(budget), W_(W), st_(st) {
        text16_ = max_sym < (1u << 16);
        kb_ = std::max<uint32_t>(32, hi_bit64(m_) + 1);
    }

    void run(HostIndex& o) {
        o = HostIndex();
        CUDA_CHECK(cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking));
        try { build(o); } catch (...) { cudaStreamSynchronize(s_); cudaStreamDestroy(s_); throw; }
        CUDA_CHECK(cudaStreamSynchronize(s_));
        cudaStreamDestroy(s_);
    }

private:
    const void* sym_;
    uint64_t n_, m_;
    int width_;
    uint32_t max_sym_;
    int device_;
    uint64_t budget_, W_;
    sealfm_build_stats_t& st_;
    bool text16_;
    uint32_t kb_;                  // label bits of a composite window key
    cudaStream_t s_ = nullptr;
    DevTracker dt_;
    Pinned host_;
    T* sa_ = nullptr;              // host SA (mapped pinned memory)
    T* sa_dev_ = nullptr;          // its device alias
    Buf<T> isa_, w_sa_, w_sa2_;
    Buf<uint64_t> w_key_, w_key2_, w_aux_, w_aux2_, small_, hist_;
    Buf<uint8_t> w_flag_, w_flag2_, text_, tmp_;
    uint64_t h_ = 0;               // doubling step of the current round, 0 in round 0
    uint64_t freeze_lo_ = 0, freeze_hi_ = 0;   // labels in [lo, hi) read as lo (split_group)
    bool round0_ = true;
    std::vector<Range> next_;
    std::vector<uint64_t> alpha_, cstart_;        // round 0: symbol and first row of every group
    uint64_t windows_round_ = 0;

    KeySrc<T> ks() const { return KeySrc<T>{isa_.p, text_.p, text16_ ? 1 : 0, m_, h_, freeze_lo_, freeze_hi_}; }
    int G(uint64_t n) const { return blocks_for(n); }
    void sync() { CUDA_CHECK(cudaStreamSynchronize(s_)); }
    void check_launch() { CUDA_CHECK(cudaGetLastError()); }

    void load(T* dst, uint64_t a, uint64_t n) { CUDA_CHECK(cudaMemcpyAsync(dst, sa_ + a, n * sizeof(T), cudaMemcpyHostToDevice, s_)); }
    void store(const T* src, uint64_t a, uint64_t n) { CUDA_CHECK(cudaMemcpyAsync(sa_ + a, src, n * sizeof(T), cudaMemcpyDeviceToHost, s_)); }
    template <typename U> U fetch(const U* dptr) {
        U v; CUDA_CHECK(cudaMemcpyAsync(&v, dptr, sizeof(U), cudaMemcpyDeviceToHost, s_)); sync(); return v;
    }
    // label of SA row j (rows not yet processed in this round carry their group's first row)
    uint64_t label_at(uint64_t j) { sync(); return fetch(isa_.p + sa_[j]); }

    void emit(uint64_t s, uint64_t e) {
        if (!next_.empty() && s - next_.back().e < kMergeGap) next_.back().e = e;
        else next_.push_back({s, e});
    }

    // selects the positions a + j with flag[j] into out (ordered); returns how many
    uint64_t select_positions(const uint8_t* flag, uint64_t a, uint64_t n, uint64_t* out) {
        size_t tb = tmp_.n;
        CUDA_CHECK(cub::DeviceSelect::Flagged(tmp_.p, tb, thrust::counting_iterator<uint64_t>(a), flag, out,
                                              small_.p + 4, (int64_t)n, s_));
        return fetch(small_.p + 4);
    }

    size_t cub_bytes(uint64_t W) {
        size_t a = 0, b = 0, c = 0;
        CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, a, (uint64_t*)nullptr, (uint64_t*)nullptr, (T*)nullptr, (T*)nullptr,
                                                   (int64_t)W, 0, 64, s_));
        CUDA_CHECK(cub::DeviceScan::InclusiveScan(nullptr, b, (uint64_t*)nullptr, (uint64_t*)nullptr, MaxOp(), (int64_t)W, s_));
        CUDA_CHECK(cub::DeviceSelect::Flagged(nullptr, c, thrust::counting_iterator<uint64_t>(0), (uint8_t*)nullptr,
                                              (uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)W + 1, s_));
        return std::max(a, std::max(b, c));
    }
    size_t tree_cub_bytes() {
        size_t a = 0;
        CUDA_CHECK(cub::DeviceRadixSort::SortKeys(nullptr, a, (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)m_, 0, 32, s_));
        return a;
    }

    // device bytes of the largest phase for window W
    uint64_t need(uint64_t W, uint32_t L) {
        const uint64_t t = text16_ ? 2 : 4, w = sizeof(T);
        const uint64_t win = W * window_row_bytes((int)w) + cub_bytes(W) + (kBins + 8) * 8;
        const uint64_t rounds = w * m_ + t * m_ + win;
        const uint64_t bwt = t * m_ + 4 * m_ + (m_ + 31) / 32 * 8 + win;
        const uint64_t tree = 8 * m_ + (m_ * L + 63) / 64 * 8 + tree_cub_bytes();
        return std::max(rounds, std::max(bwt, tree));
    }

    void plan(uint32_t L) {
        const uint64_t cap = std::min<uint64_t>(m_, std::min<uint64_t>(1ULL << 31, 1ULL << (64 - kb_)));
        if (W_) {
            W_ = std::min(std::max<uint64_t>(W_, 16), cap);
        } else {                                              // largest window the budget allows, up to cap
            uint64_t lo = 16, hi = cap;
            if (need(std::min(lo, cap), L) <= budget_) {
                while (lo < hi) { const uint64_t mid = lo + (hi - lo + 1) / 2; if (need(mid, L) <= budget_) lo = mid; else hi = mid - 1; }
            }
            W_ = std::min(lo, cap);
        }
        const uint64_t nb = need(W_, L);
        if (nb > budget_)
            throw ApiError(SEALFM_ENOMEM, "GPU index construction needs " + std::to_string(nb) + " bytes of device memory (budget " +
                                              std::to_string(budget_) + ")");
    }

    void upload_text() {
        const uint64_t t = text16_ ? 2 : 4;
        text_.alloc(dt_, m_ * t);
        uint8_t* stage = reinterpret_cast<uint8_t*>(w_key_.p);             // W u64 rows: room for W symbols of either width
        for (uint64_t a = 0; a < n_; a += W_) {
            const uint64_t c = std::min(W_, n_ - a);
            CUDA_CHECK(cudaMemcpyAsync(stage, static_cast<const uint8_t*>(sym_) + a * width_, c * width_, cudaMemcpyHostToDevice, s_));
            if (width_ == 8) {
                if (text16_) narrow_kernel<<<G(c), kBT, 0, s_>>>((const uint64_t*)stage, (uint16_t*)text_.p + a, c);
                else narrow_kernel<<<G(c), kBT, 0, s_>>>((const uint64_t*)stage, (uint32_t*)text_.p + a, c);
            } else {
                if (text16_) narrow_kernel<<<G(c), kBT, 0, s_>>>((const uint32_t*)stage, (uint16_t*)text_.p + a, c);
                else narrow_kernel<<<G(c), kBT, 0, s_>>>((const uint32_t*)stage, (uint32_t*)text_.p + a, c);
            }
            check_launch();
            sync();                                                         // the stage is reused
        }
        CUDA_CHECK(cudaMemsetAsync(text_.p + n_ * t, 0, t, s_));           // sentinel
    }

    // ---- one window: rows [a, b), whole groups; by_group: rows carry their group labels (a window of a range), else
    // they are one part of a giant group's key split and all of it is sorted by key alone
    void sort_window(uint64_t a, uint64_t b, bool by_group) {
        const uint64_t n = b - a;
        ++st_.windows; ++windows_round_;
        load(w_sa_.p, a, n);
        window_keys_kernel<T><<<G(n), kBT, 0, s_>>>(w_sa_.p, n, ks(), by_group ? 1 : 0, a, kb_, w_key_.p);
        check_launch();
        size_t tb = tmp_.n;
        const int end_bit = by_group ? (int)std::min<uint32_t>(64, kb_ + hi_bit64(n) + 1) : (int)kb_;
        CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp_.p, tb, w_key_.p, w_key2_.p, w_sa_.p, w_sa2_.p, (int64_t)n, 0, end_bit, s_));
        group_head_kernel<<<G(n), kBT, 0, s_>>>(w_key2_.p, w_aux_.p, n);
        check_launch();
        tb = tmp_.n;
        CUDA_CHECK(cub::DeviceScan::InclusiveScan(tmp_.p, tb, w_aux_.p, w_aux2_.p, MaxOp(), (int64_t)n, s_));
        relabel_kernel<T><<<G(n + 1), kBT, 0, s_>>>(w_sa2_.p, w_aux2_.p, n, a, isa_.p, w_flag_.p, w_flag2_.p);
        check_launch();
        store(w_sa2_.p, a, n);
        const uint64_t ne = select_positions(w_flag_.p, a, n + 1, w_aux_.p);
        if (ne) {
            std::vector<uint64_t> edges(ne);
            CUDA_CHECK(cudaMemcpyAsync(edges.data(), w_aux_.p, ne * 8, cudaMemcpyDeviceToHost, s_));
            sync();
            for (uint64_t i = 0; i + 1 < ne; i += 2) emit(edges[i], edges[i + 1]);
        }
        if (round0_) {                                    // group starts and their symbols (composite keys: label part 0)
            const uint64_t ng = select_positions(w_flag2_.p, 0, n, w_aux_.p);
            size_t tb2 = tmp_.n;
            CUDA_CHECK(cub::DeviceSelect::Flagged(tmp_.p, tb2, w_key2_.p, w_flag2_.p, w_aux2_.p, small_.p + 4, (int64_t)n, s_));
            std::vector<uint64_t> pos(ng), sym(ng);
            CUDA_CHECK(cudaMemcpyAsync(pos.data(), w_aux_.p, ng * 8, cudaMemcpyDeviceToHost, s_));
            CUDA_CHECK(cudaMemcpyAsync(sym.data(), w_aux2_.p, ng * 8, cudaMemcpyDeviceToHost, s_));
            sync();
            for (uint64_t i = 0; i < ng; ++i) { cstart_.push_back(a + pos[i]); alpha_.push_back(sym[i]); }
        }
        sync();
    }

    // rows [s, e) become one group labelled s
    void set_label(uint64_t s, uint64_t e) {
        for (uint64_t a = s; a < e; a += W_) {
            const uint64_t c = std::min(W_, e - a);
            load(w_sa_.p, a, c);
            set_label_kernel<T><<<G(c), kBT, 0, s_>>>(w_sa_.p, c, (T)s, isa_.p);
            check_launch();
        }
        sync();
    }

    // ---- a group larger than the window: rows [gs, ge), all labelled gs.  Its keys are read as they were when its
    // split began: a label inside [gs, ge), set by a part of the group already resolved, reads as gs.  Only this
    // group's rows are relabelled meanwhile, so that is exactly the snapshot.  Live keys would let each part resolved
    // split the rest again (a run a^k peels one block of rows per partition); with the snapshot the dominant key of
    // a run becomes one bucket at once.  Key ranges are split depth first, left side first, so groups come out in
    // row order.
    void split_group(uint64_t gs, uint64_t ge) {
        freeze_lo_ = gs; freeze_hi_ = ge;
        std::vector<Range> todo{{gs, ge}};
        while (!todo.empty()) {
            const uint64_t s = todo.back().s, e = todo.back().e;
            todo.pop_back();
            if (e - s <= W_) { sort_window(s, e, false); continue; }
            const KeySrc<T> k = ks();
            uint64_t mm[2] = {~0ULL, 0};
            CUDA_CHECK(cudaMemcpyAsync(small_.p, mm, 16, cudaMemcpyHostToDevice, s_));
            for (uint64_t a = s; a < e; a += W_) {
                const uint64_t c = std::min(W_, e - a);
                load(w_sa_.p, a, c);
                minmax_kernel<T><<<G(c), kBT, 0, s_>>>(w_sa_.p, c, k, (unsigned long long*)small_.p);
                check_launch();
            }
            CUDA_CHECK(cudaMemcpyAsync(mm, small_.p, 16, cudaMemcpyDeviceToHost, s_));
            sync();
            const uint64_t mn = mm[0], mx = mm[1];
            if (mn == mx) {                                // one key: a new group as a whole
                ++st_.single_key_buckets;
                if (s != gs) set_label(s, e);
                emit(s, e);
                if (round0_) { cstart_.push_back(s); alpha_.push_back(mn); }
                continue;
            }
            const uint64_t span = mx - mn + 1, w = (span + kBins - 1) / kBins;
            const uint32_t nb = (uint32_t)((mx - mn) / w + 1);
            CUDA_CHECK(cudaMemsetAsync(hist_.p, 0, (nb + 2) * 8, s_));
            for (uint64_t a = s; a < e; a += W_) {
                const uint64_t c = std::min(W_, e - a);
                load(w_sa_.p, a, c);
                hist_kernel<T><<<G(c), kBT, 0, s_>>>(w_sa_.p, c, k, mn, mx, w, nb, (unsigned long long*)hist_.p);
                check_launch();
            }
            std::vector<uint64_t> hist(nb + 2);
            CUDA_CHECK(cudaMemcpyAsync(hist.data(), hist_.p, (nb + 2) * 8, cudaMemcpyDeviceToHost, s_));
            sync();
            // splitter t, c rows below it: peel the dominant extreme key off if it holds half the rows, else the bin
            // boundary closest to the median (bin 0 holds mn and a later bin mx, so both sides are non-empty)
            const uint64_t size = e - s;
            uint64_t t = 0, c = 0;
            if (2 * hist[nb + 1] >= size) { t = mx; c = size - hist[nb + 1]; }
            else if (2 * hist[nb] >= size) { t = mn + 1; c = hist[nb]; }
            else {
                uint64_t cum = 0, best = ~0ULL;
                for (uint32_t b = 1; b < nb; ++b) {
                    cum += hist[b - 1];
                    if (cum == 0 || cum == size) continue;
                    const uint64_t d = cum > size / 2 ? cum - size / 2 : size / 2 - cum;
                    if (d < best) { best = d; t = mn + (uint64_t)b * w; c = cum; }
                }
            }
            if (c == 0 || c >= size) throw ApiError(SEALFM_ECUDA, "key-range split found no splitter");
            partition(s, e, t, c);
            todo.push_back({s + c, e});
            todo.push_back({s, s + c});
        }
        freeze_lo_ = freeze_hi_ = 0;
    }

    // in place: rows [s, e) with key < t move to [s, s + c), the others to [s + c, e); no order within a side
    void partition(uint64_t s, uint64_t e, uint64_t t, uint64_t c) {
        ++st_.key_partitions;
        const KeySrc<T> k = ks();
        uint64_t r = s + c;                                // right-side cursor: rows before it hold no misplaced row
        for (uint64_t l = s; l < s + c; l += W_) {
            const uint64_t ln = std::min(W_, s + c - l);
            load(w_sa_.p, l, ln);
            below_kernel<T><<<G(ln), kBT, 0, s_>>>(w_sa_.p, ln, k, t, 0, w_flag_.p);
            check_launch();
            const uint64_t f = select_positions(w_flag_.p, l, ln, w_aux2_.p);
            if (!f) continue;
            uint64_t have = 0;
            while (have < f) {
                if (r >= e) throw ApiError(SEALFM_ECUDA, "key-range partition ran out of rows");
                const uint64_t rn = std::min(W_, e - r);
                load(w_sa2_.p, r, rn);
                below_kernel<T><<<G(rn), kBT, 0, s_>>>(w_sa2_.p, rn, k, t, 1, w_flag2_.p);
                check_launch();
                const uint64_t got = select_positions(w_flag2_.p, r, rn, w_key2_.p);
                const uint64_t take = std::min(got, f - have);
                if (take) CUDA_CHECK(cudaMemcpyAsync(w_aux_.p + have, w_key2_.p, take * 8, cudaMemcpyDeviceToDevice, s_));
                r = take < got ? fetch(w_key2_.p + take) : r + rn;
                have += take;
            }
            swap_kernel<T><<<G(f), kBT, 0, s_>>>(w_sa_.p, w_aux2_.p, l, w_aux_.p, sa_dev_, f);
            check_launch();
            store(w_sa_.p, l, ln);
            sync();
        }
    }

    // ---- one unsorted range [s, e): windows of whole groups
    void sort_range(uint64_t s, uint64_t e) {
        uint64_t a = s;
        while (a < e) {
            uint64_t b = std::min(a + W_, e);
            if (b < e) {
                const uint64_t g = label_at(b - 1);
                if (label_at(b) == g) {                    // the group of row b - 1 continues past the window
                    if (g > a) { b = g; ++st_.spanning_groups; }
                    else {                                 // it starts at a: larger than the window
                        uint64_t lo = b + 1, hi = e;       // first row past it: labels do not decrease along the range
                        while (lo < hi) { const uint64_t mid = lo + (hi - lo) / 2; if (label_at(mid) == g) lo = mid + 1; else hi = mid; }
                        ++st_.giant_groups;
                        split_group(a, lo);
                        a = lo;
                        continue;
                    }
                }
            }
            sort_window(a, b, true);
            a = b;
        }
    }

    void build(HostIndex& o) {
        CUDA_CHECK(cudaSetDevice(device_));
        const uint32_t L = hi_bit64(std::max<uint64_t>(max_sym_, 1)) + 1;       // sdsl/wt_int.hpp:182-193
        plan(L);                                                                 // ENOMEM before anything large
        st_.chunk_elems = W_;
        st_.wide = sizeof(T) == 8;
        st_.text_bytes = text16_ ? 2 : 4;
        {
            const uint64_t hb = m_ * sizeof(T);
            cudaError_t err = cudaHostAlloc(&host_.p, hb, cudaHostAllocMapped | cudaHostAllocPortable);
            if (err != cudaSuccess) {
                cudaGetLastError(); host_.p = nullptr;
                throw ApiError(SEALFM_ENOMEM, "pinned host allocation of " + std::to_string(hb) + " bytes for the suffix array failed");
            }
            st_.host_pinned_bytes = hb;
            sa_ = static_cast<T*>(host_.p);
            void* d = nullptr;
            CUDA_CHECK(cudaHostGetDevicePointer(&d, host_.p, 0));
            sa_dev_ = static_cast<T*>(d);
        }
        isa_.alloc(dt_, m_);
        w_sa_.alloc(dt_, W_); w_sa2_.alloc(dt_, W_);
        w_key_.alloc(dt_, W_); w_key2_.alloc(dt_, W_);
        w_aux_.alloc(dt_, W_ + 1); w_aux2_.alloc(dt_, W_ + 1);
        w_flag_.alloc(dt_, W_ + 1); w_flag2_.alloc(dt_, W_ + 1);
        small_.alloc(dt_, 8); hist_.alloc(dt_, kBins + 2);
        tmp_.alloc(dt_, cub_bytes(W_));

        // ---- round 0: SA = identity, one group labelled 0, keys = symbols
        auto t0 = Clock::now();
        upload_text();
        CUDA_CHECK(cudaMemsetAsync(isa_.p, 0, m_ * sizeof(T), s_));
        for (uint64_t a = 0; a < m_; a += W_) {
            const uint64_t c = std::min(W_, m_ - a);
            iota_window_kernel<T><<<G(c), kBT, 0, s_>>>(w_sa_.p, a, c);
            check_launch();
            store(w_sa_.p, a, c);
            sync();
        }
        std::vector<Range> ranges{{0, m_}};
        uint32_t round = 0;
        while (!ranges.empty()) {
            if (round >= kMaxRounds) throw ApiError(SEALFM_ECUDA, "suffix sort did not converge");
            auto tr = Clock::now();
            uint64_t rows = 0;
            for (const Range& r : ranges) rows += r.e - r.s;
            st_.round_unsorted[round] = rows;
            next_.clear();
            windows_round_ = 0;
            // neighbouring ranges share a window when they fit one and the sorted rows between them (re-sorted
            // unchanged) are no more than the unsorted rows already in it: one window instead of one per range
            std::vector<Range> work;
            uint64_t work_rows = 0;
            for (const Range& r : ranges) {
                if (!work.empty() && r.e - work.back().s <= W_ && r.s - work.back().e <= work_rows) {
                    work.back().e = r.e; work_rows += r.e - r.s;
                } else {
                    work.push_back(r); work_rows = r.e - r.s;
                }
            }
            for (const Range& r : work) sort_range(r.s, r.e);
            sync();
            st_.max_windows_per_round = std::max(st_.max_windows_per_round, windows_round_);
            st_.round_s[round] = secs(tr);
            if (round0_) {
                round0_ = false;
                text_.release();                           // not needed again until the BWT
                o.size = m_;
                o.sigma = alpha_.size();
                o.alphabet = std::move(alpha_);
                o.C = std::move(cstart_);
                o.C.push_back(m_);
                o.max_level = L;
                st_.phase_s[0] = secs(t0);
                t0 = Clock::now();
            }
            h_ = h_ ? 2 * h_ : 1;
            ranges.swap(next_);
            ++round;
        }
        st_.rounds = round;
        st_.phase_s[1] = secs(t0);

        // ---- ISA samples, then BWT + SA samples from one pass over the host SA
        t0 = Clock::now();
        const uint64_t n_sa = (m_ + 31) / 32, n_isa = (m_ - 1) / 64 + 1;
        {
            Buf<uint64_t> d_isas; d_isas.alloc(dt_, n_isa);
            isa_samples_kernel<T><<<G(n_isa), kBT, 0, s_>>>(isa_.p, d_isas.p, n_isa);
            check_launch();
            o.isa_samples.resize(n_isa);
            CUDA_CHECK(cudaMemcpyAsync(o.isa_samples.data(), d_isas.p, n_isa * 8, cudaMemcpyDeviceToHost, s_));
            sync();
        }
        isa_.release();
        upload_text();
        Buf<uint32_t> bwt; bwt.alloc(dt_, m_);
        {
            Buf<uint64_t> d_sas; d_sas.alloc(dt_, n_sa);
            for (uint64_t a = 0; a < m_; a += W_) {
                const uint64_t c = std::min(W_, m_ - a);
                load(w_sa_.p, a, c);
                if (text16_) bwt_window_kernel<T, uint16_t><<<G(c), kBT, 0, s_>>>(w_sa_.p, a, c, (const uint16_t*)text_.p, bwt.p, d_sas.p);
                else bwt_window_kernel<T, uint32_t><<<G(c), kBT, 0, s_>>>(w_sa_.p, a, c, (const uint32_t*)text_.p, bwt.p, d_sas.p);
                check_launch();
            }
            o.sa_samples.resize(n_sa);
            CUDA_CHECK(cudaMemcpyAsync(o.sa_samples.data(), d_sas.p, n_sa * 8, cudaMemcpyDeviceToHost, s_));
            sync();
        }
        text_.release();
        w_sa_.release(); w_sa2_.release(); w_key_.release(); w_key2_.release(); w_aux_.release(); w_aux2_.release();
        w_flag_.release(); w_flag2_.release(); tmp_.release();
        st_.phase_s[2] = secs(t0);

        // ---- wavelet tree, level by level (as fm_build.cu): level k's order = the BWT stably sorted by k leading bits
        t0 = Clock::now();
        const uint64_t words = (m_ * L + 63) >> 6;
        Buf<uint64_t> tree; tree.alloc(dt_, words);
        CUDA_CHECK(cudaMemsetAsync(tree.p, 0, words * 8, s_));
        Buf<uint32_t> sorted; sorted.alloc(dt_, L > 1 ? m_ : 0);
        Buf<uint8_t> ttmp; ttmp.alloc(dt_, L > 1 ? tree_cub_bytes() : 0);
        const int PG = pack_blocks_for(m_);
        for (uint32_t k = 0; k < L; ++k) {
            if (k > 0) {
                size_t tb = ttmp.n;
                CUDA_CHECK(cub::DeviceRadixSort::SortKeys(ttmp.p, tb, bwt.p, sorted.p, (int64_t)m_, (int)(L - k), (int)L, s_));
                pack_level_kernel<<<PG, kBT, 0, s_>>>(sorted.p, reinterpret_cast<uint32_t*>(tree.p), m_, k, L);
            } else {
                pack_level_kernel<<<PG, kBT, 0, s_>>>(bwt.p, reinterpret_cast<uint32_t*>(tree.p), m_, k, L);
            }
            check_launch();
        }
        o.tree.resize(words);
        CUDA_CHECK(cudaMemcpyAsync(o.tree.data(), tree.p, words * 8, cudaMemcpyDeviceToHost, s_));
        sync();
        st_.phase_s[3] = secs(t0);
        st_.device_peak_bytes = dt_.peak;
    }
};

// symbol checks and the largest symbol, on all host cores
template <typename S>
uint32_t scan_symbols(const S* sym, uint64_t n) {
    const unsigned nt = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
    std::vector<uint64_t> mx(nt, 0);
    std::vector<int> bad(nt, 0);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; ++t)
        th.emplace_back([&, t] {
            const uint64_t a = n * t / nt, b = n * (t + 1) / nt;
            uint64_t hi = 0; int z = 0;
            for (uint64_t i = a; i < b; ++i) { const uint64_t v = sym[i]; hi = v > hi ? v : hi; z |= v == 0; }
            mx[t] = hi; bad[t] = z;
        });
    for (auto& t : th) t.join();
    uint64_t hi = 0;
    for (unsigned t = 0; t < nt; ++t) {
        if (bad[t]) throw ApiError(SEALFM_EINVAL, "symbol 0 is reserved for the sentinel");
        hi = std::max(hi, mx[t]);
    }
    if (hi >= (1ULL << 32)) throw ApiError(SEALFM_EINVAL, "symbols must be < 2^32");
    return (uint32_t)hi;
}

}  // namespace

void build_index_gpu_large(const void* symbols, uint64_t n, int width_bytes, int device, const sealfm_build_opts_t* opts,
                           HostIndex& o) {
    o = HostIndex();
    sealfm_build_opts_t op{};
    if (opts) op = *opts;
    for (int r : op.reserved) if (r) throw ApiError(SEALFM_EINVAL, "reserved option fields must be 0");
    if (width_bytes != 4 && width_bytes != 8) throw ApiError(SEALFM_EINVAL, "width must be 4 or 8 bytes");
    if (n + 1 >= kMaxM) throw ApiError(SEALFM_EINVAL, "GPU index construction handles texts below 2^40 - 1 symbols");
    const uint32_t max_sym = width_bytes == 8 ? scan_symbols(static_cast<const uint64_t*>(symbols), n)
                                              : scan_symbols(static_cast<const uint32_t*>(symbols), n);
    CUDA_CHECK(cudaSetDevice(device));
    uint64_t budget = op.device_budget_bytes;
    if (!budget) {
        size_t free_b = 0, total_b = 0;
        CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
        budget = free_b > (1ULL << 30) ? free_b - (1ULL << 30) : 0;
    }
    sealfm_build_stats_t st{};
    if (n + 1 < (1ULL << 32) && !op.force_wide)
        LargeBuilder<uint32_t>(symbols, n, width_bytes, max_sym, device, budget, op.chunk_elems, st).run(o);
    else
        LargeBuilder<uint64_t>(symbols, n, width_bytes, max_sym, device, budget, op.chunk_elems, st).run(o);
    g_last_stats = st;
}

const sealfm_build_stats_t& build_gpu_large_last_stats() { return g_last_stats; }

}  // namespace sealb200
