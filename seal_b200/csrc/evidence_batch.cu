// Batched evidence aggregation on the GPU (include/sealev_batch.h): sealev_first_stage and sealev_score_docs
// (evidence_host.cpp) for every query of a batch at once, with the same results bit for bit.
//
// First stage (seal/keys.py:316-368).  The host walks the located occurrences of the rare keys in sequence order j
// (key order, then SA-row order) and keeps a set of covered token positions.  That walk decomposes exactly:
//   - first touch of a document = the smallest j landing in it (the tie order of the final stable sort);
//   - best key of a document = the host's strict-improvement scan over its occurrences in j order;
//   - fresh occurrences = a greedy in j order over the intervals [end - len, end): fresh iff no earlier fresh
//     interval overlaps it.  Intervals that do not overlap transitively cannot influence each other, so the intervals
//     are sorted by start, cut into connected overlap components, and each component is resolved sequentially in j
//     order against a bitmap of its own positions;
//   - key k credits document d once iff some occurrence of k in d is fresh (any occurrence with allow_overlaps);
//   - damping runs over each document's credits in key order; documents are independent;
//   - rank = (1 - single_key) * (-sum) + single_key * (-best); sort by (rank, first touch) per query.
// Queries share launches: positions and documents are offset into disjoint per-query key spaces.
//
// Full scoring (seal/keys.py:378-491): one thread per shortlisted document walks its query's trie (a CSR of sorted
// children) from every start position to list all occurrences, sorts them by (key rank, start) -- key rank =
// position of the key in (-score, key tuple) order, so this is the host's queue order -- and then runs the host's
// placement loop, sum and unigram pass on per-document scratch.  The host's best-key scan visits keys in the order
// its open-match list discovers them: by end position, and at one end position odd lengths ascending, then even
// lengths descending (the list is rebuilt reversed at every token); the kernel reproduces that order arithmetically.
//
// Every double operation rounds as on the host: this unit is compiled with -fmad=false (Makefile), so no multiply-add
// is contracted into an FMA.
#include "../../include/sealev_batch.h"
#include "../../include/sealfm.h"
#include "common.cuh"
#include "fm_device.cuh"
#include "fm_handle.hpp"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <map>
#include <numeric>
#include <string>
#include <vector>

using namespace sealb200;

namespace sealb200 { void sealev_set_error(const std::string& msg); }   // evidence_host.cpp

namespace {

uint64_t g_budget = 0;                       // sealev_set_device_budget
thread_local double g_phase_us[4];

template <typename Fn>
int ev_guarded(Fn&& fn) {
    const int rc = guarded(fn);
    if (rc) sealev_set_error(last_error());
    return rc;
}

int grid_for(uint64_t n, int per_block) {
    const uint64_t cap = (uint64_t)sm_count() * 16;
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + per_block - 1) / per_block, cap));
}

inline int bits_for(uint64_t x) { int b = 0; while (b < 64 && (x >> b)) ++b; return std::max(b, 1); }

// Stream-ordered device allocations of one chunk, freed when the chunk ends.
struct Arena {
    cudaStream_t s;
    std::vector<void*> ptrs;
    explicit Arena(cudaStream_t st) : s(st) {}
    ~Arena() { for (void* p : ptrs) cudaFreeAsync(p, s); }
    template <typename T> T* alloc(size_t n) {
        void* p = nullptr;
        CUDA_CHECK(cudaMallocAsync(&p, std::max<size_t>(n, 1) * sizeof(T), s));
        ptrs.push_back(p);
        return static_cast<T*>(p);
    }
    template <typename T> T* put(const T* src, size_t n) {
        T* d = alloc<T>(n);
        if (n) CUDA_CHECK(cudaMemcpyAsync(d, src, n * sizeof(T), cudaMemcpyHostToDevice, s));
        return d;
    }
    template <typename T> T* put(const std::vector<T>& v) { return put(v.data(), v.size()); }
    template <typename T> void get(T* dst, const T* d, size_t n) {
        if (n) CUDA_CHECK(cudaMemcpyAsync(dst, d, n * sizeof(T), cudaMemcpyDeviceToHost, s));
    }
    void sync() { CUDA_CHECK(cudaStreamSynchronize(s)); }
    void* scratch(size_t bytes) { return alloc<char>(bytes); }
};

struct Timer {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    double lap() {
        const auto t = std::chrono::steady_clock::now();
        const double us = std::chrono::duration<double, std::micro>(t - t0).count();
        t0 = t;
        return us;
    }
};

// ------------------------------------------------------------------------------------------------
// device helpers shared by both stages
// ------------------------------------------------------------------------------------------------

// Coverage::damp of evidence_host.cpp: the score damped by the share of the key's token types already seen.
// `seen(t)` answers membership; `any_seen` = the set is not empty.
template <typename Seen>
__device__ double damp(const int64_t* tok, int len, double score, double beta, bool any_seen, Seen seen) {
    if (!any_seen) return score;
    int types = 0, fresh = 0;
    for (int i = 0; i < len; ++i) {
        bool dup = false;
        for (int j = 0; j < i && !dup; ++j) dup = tok[j] == tok[i];
        if (dup) continue;
        ++types;
        fresh += seen(tok[i]) ? 0 : 1;
    }
    return (1.0 - beta + (beta * (double)fresh / (double)types)) * score;
}

// open-addressing set of int64 in a power-of-two table (kEmpty marks a free slot)
constexpr int64_t kEmpty = INT64_MIN;
__device__ __forceinline__ uint64_t hslot(int64_t t, uint64_t mask) { return ((uint64_t)t * 0x9E3779B97F4A7C15ULL >> 17) & mask; }
__device__ bool hset_has(const int64_t* tab, uint64_t mask, int64_t t) {
    for (uint64_t i = hslot(t, mask);; i = (i + 1) & mask) {
        if (tab[i] == t) return true;
        if (tab[i] == kEmpty) return false;
    }
}
// true if t was not in the set
__device__ bool hset_add(int64_t* tab, uint64_t mask, int64_t t) {
    for (uint64_t i = hslot(t, mask);; i = (i + 1) & mask) {
        if (tab[i] == t) return false;
        if (tab[i] == kEmpty) { tab[i] = t; return true; }
    }
}

__global__ void iota_kernel(uint32_t* out, uint64_t n) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) out[i] = (uint32_t)i;
}

// ------------------------------------------------------------------------------------------------
// first stage kernels
// ------------------------------------------------------------------------------------------------

// Occurrence j of the chunk: key k (occ_off[k] <= j < occ_off[k+1]), located, mapped to its document.  Its interval
// [pos - len, pos) goes into query q's key space: S = q*M + pos - len + B, E = q*M + pos + B (B > every key length,
// M = text size + B), so intervals of different queries never meet and every key is positive.
__global__ void fs_locate_kernel(FmView v, uint64_t N, int64_t K, const int64_t* __restrict__ occ_off,
                                 const uint64_t* __restrict__ key_lo, const int32_t* __restrict__ key_len,
                                 const int32_t* __restrict__ key_q, uint64_t M, uint64_t B, uint64_t nd1,
                                 uint64_t* __restrict__ S, uint64_t* __restrict__ E, uint64_t* __restrict__ gkey,
                                 int32_t* __restrict__ okey) {
    for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < N; j += (uint64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = K;                                   // last k with occ_off[k] <= j
        while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if ((uint64_t)occ_off[mid] <= j) lo = mid; else hi = mid; }
        const int64_t k = lo;
        const uint64_t pos = locate_row(v, key_lo[k] + (j - (uint64_t)occ_off[k]));
        const uint64_t doc = doc_of_pos(v, pos);
        const uint64_t base = (uint64_t)key_q[k] * M;
        S[j] = base + pos - (uint64_t)key_len[k] + B;
        E[j] = base + pos + B;
        gkey[j] = (uint64_t)key_q[k] * nd1 + doc;                 // (query, document) group
        okey[j] = (int32_t)k;
    }
}

__global__ void gather_u64_kernel(uint64_t n, const uint32_t* __restrict__ perm, const uint64_t* __restrict__ src, uint64_t* __restrict__ dst) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) dst[i] = src[perm[i]];
}

// heads of the overlap components in start order: an interval starts a component iff it starts at or after the
// largest end before it
__global__ void comp_head_kernel(uint64_t n, const uint64_t* __restrict__ Ss, const uint64_t* __restrict__ pm, uint32_t* __restrict__ head) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) head[i] = Ss[i] >= pm[i] ? 1u : 0u;
}

// component c: members [cbeg[c], cbeg[c+1]) of the start order, positions [cstart[c], cend[c]); key2 = (c, j) for the
// sort into j order within components
__global__ void comp_bounds_kernel(uint64_t n, const uint64_t* __restrict__ Ss, const uint64_t* __restrict__ Es,
                                   const uint64_t* __restrict__ pm, const uint32_t* __restrict__ cid,
                                   const uint32_t* __restrict__ perm, uint64_t* __restrict__ key2,
                                   uint64_t* __restrict__ cbeg, uint64_t* __restrict__ cstart, uint64_t* __restrict__ cend) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = cid[i] - 1;
        key2[i] = ((uint64_t)c << 32) | perm[i];
        const bool h = i == 0 || cid[i - 1] != cid[i];
        if (h) { cbeg[c] = i; cstart[c] = Ss[i]; if (c) cend[c - 1] = pm[i]; }
        if (i == n - 1) { cbeg[c + 1] = n; cend[c] = max(pm[i], Es[i]); }
    }
}

__global__ void comp_words_kernel(uint64_t nc, const uint64_t* __restrict__ cstart, const uint64_t* __restrict__ cend, uint64_t* __restrict__ words) {
    for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < nc; c += (uint64_t)gridDim.x * blockDim.x)
        words[c] = (cend[c] - cstart[c] + 31) / 32;
}

// one thread per component: the host's greedy over its members in j order
__global__ void comp_fresh_kernel(uint64_t nc, const uint64_t* __restrict__ cbeg, const uint64_t* __restrict__ cstart,
                                  const uint64_t* __restrict__ woff, const uint64_t* __restrict__ key2s,
                                  const uint64_t* __restrict__ S, const uint64_t* __restrict__ E, uint32_t* __restrict__ bits,
                                  uint8_t* __restrict__ fresh) {
    for (uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; c < nc; c += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t* b = bits + woff[c];
        const uint64_t base = cstart[c];
        for (uint64_t i = cbeg[c]; i < cbeg[c + 1]; ++i) {
            const uint32_t j = (uint32_t)(key2s[i] & 0xffffffffu);
            const uint64_t s = S[j] - base, e = E[j] - base;
            bool ok = true;
            for (uint64_t t = s; t < e && ok; ++t) ok = !((b[t >> 5] >> (t & 31)) & 1u);
            if (ok) for (uint64_t t = s; t < e; ++t) b[t >> 5] |= 1u << (t & 31);
            fresh[j] = ok;
        }
    }
}

__global__ void group_head_kernel(uint64_t n, const uint64_t* __restrict__ gs, uint8_t* __restrict__ head, uint64_t* __restrict__ mlen,
                                  const uint32_t* __restrict__ perm3, const int32_t* __restrict__ okey, const int32_t* __restrict__ key_len) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        head[i] = i == 0 || gs[i] != gs[i - 1];
        mlen[i] = (uint64_t)key_len[okey[perm3[i]]];
    }
}

struct FsKeys {
    const int64_t* tok; const int64_t* off; const double* score; const int64_t* count; const int32_t* len; const int32_t* q;
};

// one thread per (query, document): best key, credits, damping, rank (evidence_host.cpp sealev_first_stage)
__global__ void group_score_kernel(uint64_t ng, uint64_t n, const uint64_t* __restrict__ gbeg, const uint32_t* __restrict__ perm3,
                                   const int32_t* __restrict__ okey, const uint8_t* __restrict__ fresh,
                                   const uint64_t* __restrict__ lenoff, FsKeys K, const int64_t* __restrict__ empty_count,
                                   int sort_mode, int allow_overlaps, double beta, double single_key,
                                   int64_t* __restrict__ seen_buf, uint64_t* __restrict__ out_rankkey,
                                   uint32_t* __restrict__ out_ft, uint32_t* __restrict__ out_q, uint32_t* __restrict__ out_g,
                                   const uint64_t* __restrict__ gs, uint64_t nd1, int64_t* __restrict__ out_doc) {
    for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < ng; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = gbeg[g], e = g + 1 < ng ? gbeg[g + 1] : n;
        const uint32_t ft = perm3[b];
        const int32_t q = K.q[okey[ft]];
        const int64_t ec = empty_count[q];
        int64_t best = -1; double best_score = 0.0;
        int64_t* seen = seen_buf + lenoff[b];
        int n_seen = 0;
        double total = 0.0;
        for (uint64_t i = b; i < e;) {
            const int32_t k = okey[perm3[i]];
            const int64_t n_k = K.len[k];
            const double sc = K.score[k];
            bool credit = allow_overlaps != 0;
            for (; i < e && okey[perm3[i]] == k; ++i) {           // the occurrences of key k in this document
                const int64_t lb = best < 0 ? 0 : K.len[best];
                const int64_t cb = best < 0 ? ec : K.count[best];
                bool better;
                if (sort_mode == 1) better = n_k != lb ? n_k > lb : sc > best_score;
                else if (sort_mode == 2) better = K.count[k] != cb ? -K.count[k] > -cb : sc > best_score;
                else better = sc > best_score;
                if (better) { best = k; best_score = sc; }
                credit = credit || fresh[perm3[i]];
            }
            if (!credit) continue;
            const int64_t* t = K.tok + K.off[k];
            total += damp(t, (int)n_k, sc, beta, n_seen > 0, [&](int64_t x) {
                for (int s = 0; s < n_seen; ++s) if (seen[s] == x) return true;
                return false;
            });
            for (int64_t u = 0; u < n_k; ++u) {
                bool have = false;
                for (int s = 0; s < n_seen && !have; ++s) have = seen[s] == t[u];
                if (!have) seen[n_seen++] = t[u];
            }
        }
        double rank = (1.0 - single_key) * (-total) + single_key * (-best_score);
        if (rank == 0.0) rank = 0.0;                              // std::stable_sort sees -0.0 == 0.0
        const uint64_t u = (uint64_t)__double_as_longlong(rank);
        out_rankkey[g] = (u >> 63) ? ~u : (u | (1ULL << 63));     // ascending bit order = ascending value
        out_ft[g] = ft; out_q[g] = (uint32_t)q; out_g[g] = (uint32_t)g;
        out_doc[g] = (int64_t)(gs[b] - (uint64_t)q * nd1);
    }
}

// ------------------------------------------------------------------------------------------------
// scoring kernels
// ------------------------------------------------------------------------------------------------

struct Trie {                                 // all queries' tries; node ids are global, query q's root = root[q]
    const int32_t* root; const int32_t* child_off; const int64_t* child_tok; const int32_t* child_node; const int32_t* node_key;
};

__device__ __forceinline__ int32_t trie_next(const Trie& T, int32_t node, int64_t t) {
    int32_t lo = T.child_off[node], hi = T.child_off[node + 1];
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        const int64_t c = T.child_tok[mid];
        if (c == t) return T.child_node[mid];
        if (c < t) lo = mid + 1; else hi = mid;
    }
    return -1;
}

// doc token array of the reference: [2] + doc[:-1]
__global__ void doc_tokens_kernel(uint64_t nd, const uint64_t* __restrict__ raw_off, const uint64_t* __restrict__ raw,
                                  const int64_t* __restrict__ tok_off, int64_t shift, int64_t* __restrict__ tok) {
    for (uint64_t d = blockIdx.x; d < nd; d += gridDim.x) {
        const int64_t L = tok_off[d + 1] - tok_off[d];
        for (int64_t i = threadIdx.x; i < L; i += blockDim.x)
            tok[tok_off[d] + i] = i == 0 ? 2 : (int64_t)raw[raw_off[d] + i - 1] - shift;
    }
}

__global__ void __launch_bounds__(64) extract_docs_kernel(FmView v, uint64_t n, const uint64_t* __restrict__ b,
                                                          const uint64_t* __restrict__ e, const uint64_t* __restrict__ off,
                                                          uint64_t* __restrict__ out) {
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x)
        extract_text(v, b[t], e[t], out + off[t]);
}

__global__ void count_places_kernel(uint64_t nd, const int64_t* __restrict__ tok_off, const int64_t* __restrict__ tok,
                                    const int32_t* __restrict__ doc_q, Trie T, uint64_t* __restrict__ n_places) {
    for (uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; d < nd; d += (uint64_t)gridDim.x * blockDim.x) {
        const int64_t* x = tok + tok_off[d];
        const int32_t L = (int32_t)(tok_off[d + 1] - tok_off[d]);
        const int32_t root = T.root[doc_q[d]];
        uint64_t c = 0;
        for (int32_t a = 0; a < L; ++a)
            for (int32_t node = root, i = a; i < L && (node = trie_next(T, node, x[i])) >= 0; ++i) c += T.node_key[node] >= 0;
        n_places[d] = c;
    }
}

struct ScoreKeys {
    const int64_t* tok; const int64_t* off; const double* score; const int64_t* count; const int32_t* rank2key;
    const int64_t* qkey_off;    // query q's keys: [qkey_off[q], qkey_off[q+1]) of the chunk's key arrays
};
struct ScoreScratch {
    uint64_t* places; const uint64_t* place_off;     // per document: (key rank << 32 | start), sorted in place
    int64_t* pick_key; double* pick_score; const uint64_t* pick_soff;   // places + tokens per document
    uint8_t* free_; int64_t* sets; const int64_t* set_off;              // 2 hash tables of set_cap(L) per document
};
struct UniTab { const int64_t* off; const int64_t* tok; const double* val; const int64_t* size; };

__device__ void heap_sift(uint64_t* a, int64_t i, int64_t n) {
    const uint64_t x = a[i];
    for (;;) {
        int64_t c = 2 * i + 1;
        if (c >= n) break;
        if (c + 1 < n && a[c + 1] > a[c]) ++c;
        if (a[c] <= x) break;
        a[i] = a[c]; i = c;
    }
    a[i] = x;
}

__global__ void score_docs_kernel(uint64_t nd, const int64_t* __restrict__ tok_off, const int64_t* __restrict__ tok,
                                  const int32_t* __restrict__ doc_q, Trie T, ScoreKeys K, const int64_t* __restrict__ empty_count,
                                  UniTab U, ScoreScratch W, int sort_mode, int allow_overlaps, int ignore_free_places,
                                  int single_key_add_unigrams, int compensated, double beta, double single_key,
                                  double* __restrict__ out_score, int64_t* __restrict__ out_best, double* __restrict__ out_best_score,
                                  uint64_t* __restrict__ n_pick_out, int* __restrict__ err) {
    for (uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; d < nd; d += (uint64_t)gridDim.x * blockDim.x) {
        const int64_t* x = tok + tok_off[d];
        const int32_t L = (int32_t)(tok_off[d + 1] - tok_off[d]);
        const int32_t q = doc_q[d];
        const int32_t root = T.root[q];
        const int64_t k0 = K.qkey_off[q];
        auto klen = [&](int64_t k) { return k < 0 ? (int64_t)0 : K.off[k0 + k + 1] - K.off[k0 + k]; };
        auto kcount = [&](int64_t k) { return k < 0 ? empty_count[q] : K.count[k0 + k]; };
        // ---- every occurrence, as (key rank, start) ----
        uint64_t* P = W.places + W.place_off[d];
        int64_t np = 0;
        for (int32_t a = 0; a < L; ++a)
            for (int32_t node = root, i = a; i < L && (node = trie_next(T, node, x[i])) >= 0; ++i) {
                const int32_t k = T.node_key[node];
                if (k >= 0) P[np++] = ((uint64_t)(uint32_t)k << 32) | (uint32_t)a;   // node_key = the key's rank
            }
        // heap sort into (rank, start) = the host's queue order
        for (int64_t i = np / 2 - 1; i >= 0; --i) heap_sift(P, i, np);
        for (int64_t m = np - 1; m > 0; --m) { const uint64_t t = P[0]; P[0] = P[m]; P[m] = t; heap_sift(P, 0, m); }
        // ---- best single key in the host's discovery order (see the file comment) ----
        int64_t best = -1; double best_score = 0.0; uint64_t best_hit = 0; bool have = false;
        for (int64_t i = 0; i < np; ++i) {
            const uint32_t r = (uint32_t)(P[i] >> 32);
            if (i && (uint32_t)(P[i - 1] >> 32) == r) continue;   // first (smallest-start) occurrence of each key
            const int64_t k = K.rank2key[k0 + r];
            const int64_t len = klen(k);
            const uint64_t endp = (uint64_t)(uint32_t)P[i] + (uint64_t)len;
            const uint64_t hit = (endp << 32) | (len & 1 ? (uint64_t)len : ((1ULL << 31) - (uint64_t)len));
            const double s = K.score[k0 + k];
            auto ahead = [&](int64_t xk, double xs, int64_t yk, double ys) {   // strictly smaller (-len,-s) | (count,-s) | -s
                if (sort_mode == 1) return klen(xk) != klen(yk) ? -klen(xk) < -klen(yk) : -xs < -ys;
                if (sort_mode == 2) return kcount(xk) != kcount(yk) ? kcount(xk) < kcount(yk) : -xs < -ys;
                return -xs < -ys;
            };
            if (ahead(k, s, best, best_score) || (have && !ahead(best, best_score, k, s) && hit < best_hit)) {
                best = k; best_score = s; best_hit = hit; have = true;
            }
        }
        // ---- the greedy placement (:434-470) ----
        const uint64_t cap = (uint64_t)W.set_off[d + 1] - (uint64_t)W.set_off[d];
        int64_t* seen = W.sets + W.set_off[d];
        int64_t* done = seen + cap / 2;
        const uint64_t mask = cap / 2 - 1;
        for (uint64_t i = 0; i < cap; ++i) seen[i] = kEmpty;
        bool any_seen = false;
        uint8_t* fr = W.free_ + tok_off[d];
        for (int32_t i = 0; i < L; ++i) fr[i] = 1;
        int64_t* pk = W.pick_key + W.pick_soff[d];
        double* ps = W.pick_score + W.pick_soff[d];
        int64_t n_pick = 0;
        int64_t prev = -1; double prev_adj = 0.0;
        auto in_seen = [&](int64_t t) { return hset_has(seen, mask, t); };
        for (int64_t i = 0; i < np; ++i) {
            const int64_t k = K.rank2key[k0 + (uint32_t)(P[i] >> 32)];
            const int32_t a = (int32_t)(uint32_t)P[i];
            const int64_t len = klen(k);
            const int32_t bnd = a + (int32_t)len;
            const int64_t* kt = K.tok + K.off[k0 + k];
            const bool same = prev >= 0 && prev == k;              // keys of one query are distinct tuples
            const double adj = same ? prev_adj : damp(kt, (int)len, K.score[k0 + k], beta, any_seen, in_seen);
            if (adj <= 0.0) continue;
            if (!allow_overlaps) { bool ok = true; for (int32_t t = a; t < bnd && ok; ++t) ok = fr[t]; if (!ok) continue; }
            if (!same) {
                prev = k; prev_adj = adj;
                for (int64_t u = 0; u < len; ++u) hset_add(seen, mask, kt[u]);
                any_seen = any_seen || len > 0;
                pk[n_pick] = k; ps[n_pick] = adj; ++n_pick;
            }
            for (int32_t t = a; t < bnd; ++t) fr[t] = 0;
        }
        if (ignore_free_places) for (int32_t i = 0; i < L; ++i) fr[i] = 1;
        double total = 0.0;                                        // Python's sum() (sealev_set_sum_mode)
        if (!compensated) {
            for (int64_t i = 0; i < n_pick; ++i) total += ps[i];
        } else if (n_pick > 0) {
            total = ps[0];
            double comp = 0.0;
            for (int64_t i = 1; i < n_pick; ++i) {
                const double v = ps[i], t = total + v;
                if (fabs(total) >= fabs(v)) comp += (total - t) + v; else comp += (v - t) + total;
                total = t;
            }
            if (comp != 0.0 && isfinite(comp)) total += comp;
        }
        double uni = 0.0;
        const int64_t V = U.size[q];
        if (V >= 0) {                                              // :479-486
            for (uint64_t i = 0; i < cap / 2; ++i) done[i] = kEmpty;
            const int64_t u0 = U.off[q], u1 = U.off[q + 1];
            for (int32_t i = 0; i < L; ++i) {
                if (!fr[i] || !hset_add(done, mask, x[i])) continue;
                const int64_t t = x[i];
                if (t < 0 || t >= V) { atomicExch(err, 1); break; }
                int64_t lo = u0, hi = u1;                          // sorted sparse table
                while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (U.tok[mid] < t) lo = mid + 1; else hi = mid; }
                double s = lo < u1 && U.tok[lo] == t ? U.val[lo] : 0.0;
                if (s > 0.0) {
                    s = damp(&t, 1, s, beta, any_seen, in_seen);
                    if (s != 0.0) { uni += s; pk[n_pick] = -1 - t; ps[n_pick] = s; ++n_pick; }
                }
            }
        }
        const double lone = best_score + (single_key_add_unigrams ? uni : 0.0);
        total += uni;
        out_score[d] = (1.0 - single_key) * total + single_key * lone;
        out_best[d] = best; out_best_score[d] = best_score;
        n_pick_out[d] = (uint64_t)n_pick;
    }
}

__global__ void compact_picks_kernel(uint64_t nd, const uint64_t* __restrict__ n_pick, const uint64_t* __restrict__ poff,
                                     const uint64_t* __restrict__ soff, const int64_t* __restrict__ sk, const double* __restrict__ ss,
                                     int64_t* __restrict__ ok, double* __restrict__ os) {
    for (uint64_t d = blockIdx.x; d < nd; d += gridDim.x)
        for (uint64_t i = threadIdx.x; i < n_pick[d]; i += blockDim.x) { ok[poff[d] + i] = sk[soff[d] + i]; os[poff[d] + i] = ss[soff[d] + i]; }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

uint64_t budget_bytes() { return g_budget ? g_budget : (2ULL << 30); }

template <typename T>
void exclusive_sum(Arena& A, const T* in, T* out, uint64_t n) {
    size_t tb = 0;
    CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, (int64_t)n, A.s));
    void* t = A.scratch(tb);
    CUDA_CHECK(cub::DeviceScan::ExclusiveSum(t, tb, in, out, (int64_t)n, A.s));
}

template <typename K, typename V>
void sort_pairs(Arena& A, const K* ki, K* ko, const V* vi, V* vo, uint64_t n, int end_bit) {
    size_t tb = 0;
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tb, ki, ko, vi, vo, (int64_t)n, 0, end_bit, A.s));
    void* t = A.scratch(tb);
    CUDA_CHECK(cub::DeviceRadixSort::SortPairs(t, tb, ki, ko, vi, vo, (int64_t)n, 0, end_bit, A.s));
}

struct MaxOp { __device__ uint64_t operator()(uint64_t a, uint64_t b) const { return a > b ? a : b; } };

// First stage of queries [q0, q1): shortlists appended to out (per query, in order)
void first_stage_chunk(const sealfm_t* h, cudaStream_t s, int64_t q0, int64_t q1, const int64_t* qko, const int64_t* key_tok,
                       const int64_t* key_off, const double* key_score, const int64_t* key_count, const uint64_t* key_lo,
                       const int64_t* key_rows, const int64_t* empty_count, int sort_mode, int allow_overlaps, double beta,
                       double single_key, int64_t max_docs, std::vector<std::vector<int64_t>>& out) {
    const FmView v = sealfm_view(h);
    Timer tm;
    const int64_t k0 = qko[q0], K = qko[q1] - k0;
    std::vector<int64_t> occ_off(K + 1, 0);
    std::vector<int32_t> klen(K), kq(K);
    int64_t maxlen = 0;
    for (int64_t q = q0; q < q1; ++q)
        for (int64_t k = qko[q]; k < qko[q + 1]; ++k) {
            const int64_t i = k - k0;
            klen[i] = (int32_t)(key_off[k + 1] - key_off[k]); kq[i] = (int32_t)(q - q0);
            maxlen = std::max<int64_t>(maxlen, klen[i]);
            occ_off[i + 1] = occ_off[i] + std::max<int64_t>(key_rows[k], 0);
        }
    const uint64_t N = (uint64_t)occ_off[K];
    if (N == 0) return;
    if (N >= (1ULL << 32)) throw ApiError(SEALFM_EINVAL, "more than 2^32 located rows in one query");
    Arena A(s);
    const uint64_t B = (uint64_t)maxlen + 1, M = v.m + B, nq = (uint64_t)(q1 - q0);
    const uint64_t nd1 = v.n_beginnings + 1;
    std::vector<int64_t> ktok_local(key_tok + key_off[k0], key_tok + key_off[k0 + K]);
    std::vector<int64_t> koff_local(K + 1);
    for (int64_t i = 0; i <= K; ++i) koff_local[i] = key_off[k0 + i] - key_off[k0];
    int64_t* d_occ = A.put(occ_off);
    uint64_t* d_lo = A.put(key_lo + k0, K);
    int32_t* d_len = A.put(klen); int32_t* d_q = A.put(kq);
    FsKeys KD{A.put(ktok_local), A.put(koff_local), A.put(key_score + k0, K), A.put(key_count + k0, K), d_len, d_q};
    int64_t* d_ec = A.put(empty_count + q0, nq);
    uint64_t* S = A.alloc<uint64_t>(N); uint64_t* E = A.alloc<uint64_t>(N); uint64_t* gk = A.alloc<uint64_t>(N);
    int32_t* okey = A.alloc<int32_t>(N);
    fs_locate_kernel<<<grid_for(N, 128), 128, 0, s>>>(v, N, K, d_occ, d_lo, d_len, d_q, M, B, nd1, S, E, gk, okey);
    CUDA_CHECK(cudaGetLastError());
    A.sync();
    g_phase_us[0] += tm.lap();
    // ---- fresh occurrences: components in start order, each resolved in j order ----
    uint32_t* iota = A.alloc<uint32_t>(N);
    iota_kernel<<<grid_for(N, 256), 256, 0, s>>>(iota, N);
    uint64_t* Ss = A.alloc<uint64_t>(N); uint32_t* perm = A.alloc<uint32_t>(N);
    sort_pairs(A, S, Ss, iota, perm, N, bits_for(nq * M));
    uint64_t* Es = A.alloc<uint64_t>(N); uint64_t* pm = A.alloc<uint64_t>(N);
    gather_u64_kernel<<<grid_for(N, 256), 256, 0, s>>>(N, perm, E, Es);
    {
        size_t tb = 0;
        CUDA_CHECK(cub::DeviceScan::ExclusiveScan(nullptr, tb, Es, pm, MaxOp(), (uint64_t)0, (int64_t)N, s));
        void* t = A.scratch(tb);
        CUDA_CHECK(cub::DeviceScan::ExclusiveScan(t, tb, Es, pm, MaxOp(), (uint64_t)0, (int64_t)N, s));
    }
    uint32_t* head = A.alloc<uint32_t>(N); uint32_t* cid = A.alloc<uint32_t>(N);
    comp_head_kernel<<<grid_for(N, 256), 256, 0, s>>>(N, Ss, pm, head);
    {
        size_t tb = 0;
        CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, tb, head, cid, (int64_t)N, s));
        void* t = A.scratch(tb);
        CUDA_CHECK(cub::DeviceScan::InclusiveSum(t, tb, head, cid, (int64_t)N, s));
    }
    uint32_t nc = 0;
    A.get(&nc, cid + N - 1, 1);
    A.sync();
    uint64_t* key2 = A.alloc<uint64_t>(N); uint64_t* key2s = A.alloc<uint64_t>(N);
    uint64_t* cbeg = A.alloc<uint64_t>(nc + 1); uint64_t* cstart = A.alloc<uint64_t>(nc); uint64_t* cend = A.alloc<uint64_t>(nc);
    comp_bounds_kernel<<<grid_for(N, 256), 256, 0, s>>>(N, Ss, Es, pm, cid, perm, key2, cbeg, cstart, cend);
    uint64_t* words = A.alloc<uint64_t>(nc); uint64_t* woff = A.alloc<uint64_t>(nc);
    comp_words_kernel<<<grid_for(nc, 256), 256, 0, s>>>(nc, cstart, cend, words);
    exclusive_sum(A, words, woff, nc);
    // a component spans at most the sum of its members' lengths: N * maxlen bits over all components, + 1 word each
    const uint64_t max_words = (N * (uint64_t)maxlen + 31) / 32 + nc;
    uint32_t* bits = A.alloc<uint32_t>(max_words);
    CUDA_CHECK(cudaMemsetAsync(bits, 0, max_words * 4, s));
    {
        size_t tb = 0;
        CUDA_CHECK(cub::DeviceRadixSort::SortKeys(nullptr, tb, key2, key2s, (int64_t)N, 0, 32 + bits_for(nc), s));
        void* t = A.scratch(tb);
        CUDA_CHECK(cub::DeviceRadixSort::SortKeys(t, tb, key2, key2s, (int64_t)N, 0, 32 + bits_for(nc), s));
    }
    uint8_t* fresh = A.alloc<uint8_t>(N);
    comp_fresh_kernel<<<grid_for(nc, 128), 128, 0, s>>>(nc, cbeg, cstart, woff, key2s, S, E, bits, fresh);
    CUDA_CHECK(cudaGetLastError());
    // ---- (query, document) groups in j order ----
    uint64_t* gs = A.alloc<uint64_t>(N); uint32_t* perm3 = A.alloc<uint32_t>(N);
    sort_pairs(A, gk, gs, iota, perm3, N, bits_for(nq * nd1));
    uint8_t* ghead = A.alloc<uint8_t>(N); uint64_t* mlen = A.alloc<uint64_t>(N);
    group_head_kernel<<<grid_for(N, 256), 256, 0, s>>>(N, gs, ghead, mlen, perm3, okey, d_len);
    uint64_t* gbeg = A.alloc<uint64_t>(N); uint64_t* d_ng = A.alloc<uint64_t>(1);
    {
        size_t tb = 0;
        thrust::counting_iterator<uint64_t> it(0);
        CUDA_CHECK(cub::DeviceSelect::Flagged(nullptr, tb, it, ghead, gbeg, d_ng, (int64_t)N, s));
        void* t = A.scratch(tb);
        CUDA_CHECK(cub::DeviceSelect::Flagged(t, tb, it, ghead, gbeg, d_ng, (int64_t)N, s));
    }
    uint64_t* lenoff = A.alloc<uint64_t>(N);              // seen-token scratch of each group: its members' lengths
    exclusive_sum(A, mlen, lenoff, N);
    int64_t* seen_buf = A.alloc<int64_t>(N * (uint64_t)std::max<int64_t>(maxlen, 1));
    uint64_t ng = 0;
    A.get(&ng, d_ng, 1);
    A.sync();
    uint64_t* rk = A.alloc<uint64_t>(ng); uint32_t* ft = A.alloc<uint32_t>(ng); uint32_t* gq = A.alloc<uint32_t>(ng);
    uint32_t* gid = A.alloc<uint32_t>(ng); int64_t* gdoc = A.alloc<int64_t>(ng);
    group_score_kernel<<<grid_for(ng, 128), 128, 0, s>>>(ng, N, gbeg, perm3, okey, fresh, lenoff, KD, d_ec, sort_mode,
                                                         allow_overlaps, beta, single_key, seen_buf, rk, ft, gq, gid,
                                                         gs, nd1, gdoc);
    CUDA_CHECK(cudaGetLastError());
    // ---- per query: stable sort by (rank, first touch): LSD passes first touch, rank, query ----
    uint32_t* ft_s = A.alloc<uint32_t>(ng); uint32_t* o1 = A.alloc<uint32_t>(ng);
    sort_pairs(A, ft, ft_s, gid, o1, ng, 32);
    uint64_t* rk1 = A.alloc<uint64_t>(ng);
    gather_u64_kernel<<<grid_for(ng, 256), 256, 0, s>>>(ng, o1, rk, rk1);
    uint64_t* rk_s = A.alloc<uint64_t>(ng); uint32_t* o2 = A.alloc<uint32_t>(ng);
    sort_pairs(A, rk1, rk_s, o1, o2, ng, 64);
    std::vector<uint32_t> order(ng), gq_h(ng);
    std::vector<int64_t> gdoc_h(ng);
    A.get(order.data(), o2, ng); A.get(gq_h.data(), gq, ng); A.get(gdoc_h.data(), gdoc, ng);
    A.sync();
    // the query pass of the LSD sort is a stable bucket pass on the host (the shortlists are cut there anyway)
    std::vector<std::vector<int64_t>> per(nq);
    for (uint64_t i = 0; i < ng; ++i) {
        const uint32_t g = order[i], q = gq_h[g];
        if ((int64_t)per[q].size() < max_docs) per[q].push_back(gdoc_h[g]);
    }
    for (uint64_t q = 0; q < nq; ++q) out[q0 + q] = std::move(per[q]);
    g_phase_us[1] += tm.lap();
}

// per-query trie CSR over the chunk's keys; node_key = the key's rank in (-score, key tuple) order
struct HostTrie {
    std::vector<int32_t> root, child_off{0}, child_node, node_key, rank2key;
    std::vector<int64_t> child_tok;
};

void build_tries(int64_t q0, int64_t q1, const int64_t* qko, const int64_t* key_tok, const int64_t* key_off,
                 const double* key_score, HostTrie& T) {
    for (int64_t q = q0; q < q1; ++q) {
        const int64_t a = qko[q], n = qko[q + 1] - qko[q];
        std::vector<int32_t> order(n);
        std::iota(order.begin(), order.end(), 0);
        auto tup_less = [&](int64_t x, int64_t y) {
            const int64_t *tx = key_tok + key_off[a + x], *ty = key_tok + key_off[a + y];
            const int64_t lx = key_off[a + x + 1] - key_off[a + x], ly = key_off[a + y + 1] - key_off[a + y];
            return std::lexicographical_compare(tx, tx + lx, ty, ty + ly);
        };
        std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) {
            const double sx = key_score[a + x], sy = key_score[a + y];
            if (-sx != -sy) return -sx < -sy;
            return tup_less(x, y);
        });
        std::vector<int32_t> rank(n);
        for (int64_t r = 0; r < n; ++r) { rank[order[r]] = (int32_t)r; T.rank2key.push_back(order[r]); }
        // trie with std::map children (sorted), flattened breadth-agnostic: node ids in creation order
        std::vector<std::map<int64_t, int32_t>> kids(1);
        std::vector<int32_t> nkey(1, -1);
        for (int64_t k = 0; k < n; ++k) {
            int32_t cur = 0;
            for (int64_t i = key_off[a + k]; i < key_off[a + k + 1]; ++i) {
                auto it = kids[cur].find(key_tok[i]);
                if (it == kids[cur].end()) {
                    const int32_t nn = (int32_t)kids.size();
                    kids[cur].emplace(key_tok[i], nn); kids.emplace_back(); nkey.push_back(-1); cur = nn;
                } else cur = it->second;
            }
            nkey[cur] = rank[k];
        }
        const int32_t base = (int32_t)T.node_key.size();
        T.root.push_back(base);
        for (size_t nd = 0; nd < kids.size(); ++nd) {
            for (auto& c : kids[nd]) { T.child_tok.push_back(c.first); T.child_node.push_back(base + c.second); }
            T.child_off.push_back((int32_t)T.child_tok.size());
            T.node_key.push_back(nkey[nd]);
        }
    }
}

inline uint64_t set_cap(int64_t L) {          // two power-of-two tables of at least 2L + 2 slots
    uint64_t c = 4;
    while (c < (uint64_t)(2 * L + 2)) c <<= 1;
    return 2 * c;
}

}  // namespace

namespace sealb200 { bool sealev_compensated_sum(); }   // evidence_host.cpp

extern "C" {

void sealev_set_device_budget(uint64_t bytes) { g_budget = bytes; }

void sealev_batch_phase_us(double* out4) { if (out4) std::memcpy(out4, g_phase_us, sizeof(g_phase_us)); }

int sealev_batch_first_stage(const sealfm_t* h, int64_t n_queries, const int64_t* query_key_off, const int64_t* key_tok,
                             const int64_t* key_off, const double* key_score, const int64_t* key_count,
                             const uint64_t* key_lo, const int64_t* key_rows, const int64_t* empty_count,
                             int32_t sort_mode, int32_t allow_overlaps, double beta, double single_key, int64_t max_docs,
                             int64_t* out_off, int64_t* out_docs, int64_t out_cap) {
    return ev_guarded([&] {
        std::memset(g_phase_us, 0, sizeof(g_phase_us));
        if (n_queries < 0 || !out_off || (n_queries && (!query_key_off || !key_off || !empty_count)))
            throw ApiError(SEALFM_EINVAL, "null argument");
        out_off[0] = 0;
        if (!n_queries) return;
        if (sealfm_beginnings(h).empty()) throw ApiError(SEALFM_EINVAL, "sealfm_set_beginnings not called");
        cudaStream_t s = sealfm_stream(h);
        std::vector<std::vector<int64_t>> out(n_queries);
        const uint64_t row_budget = std::max<uint64_t>(1, budget_bytes() / 160);    // ~160 device bytes per located row
        // queries of one chunk share 64-bit key spaces of (text size + longest key + 1) positions, (documents + 1) groups
        int64_t maxlen = 0;
        for (int64_t k = 0; k < query_key_off[n_queries]; ++k) maxlen = std::max<int64_t>(maxlen, key_off[k + 1] - key_off[k]);
        const FmView v = sealfm_view(h);
        const uint64_t max_q = std::max<uint64_t>(1, ((uint64_t)1 << 62) / (v.m + (uint64_t)maxlen + 1 + v.n_beginnings + 1));
        for (int64_t q0 = 0; q0 < n_queries;) {
            int64_t q1 = q0;
            uint64_t rows = 0;
            while (q1 < n_queries && (uint64_t)(q1 - q0) < max_q) {
                uint64_t r = 0;
                for (int64_t k = query_key_off[q1]; k < query_key_off[q1 + 1]; ++k) r += (uint64_t)std::max<int64_t>(key_rows[k], 0);
                if (q1 > q0 && rows + r > row_budget) break;
                rows += r; ++q1;
            }
            first_stage_chunk(h, s, q0, q1, query_key_off, key_tok, key_off, key_score, key_count, key_lo, key_rows,
                              empty_count, sort_mode, allow_overlaps, beta, single_key, max_docs < 0 ? 0 : max_docs, out);
            q0 = q1;
        }
        for (int64_t q = 0; q < n_queries; ++q) {
            out_off[q + 1] = out_off[q] + (int64_t)out[q].size();
            if (out_off[q + 1] > out_cap) throw ApiError(SEALFM_ECAPACITY, "output buffer too small");
            std::copy(out[q].begin(), out[q].end(), out_docs + out_off[q]);
        }
    });
}

int sealev_batch_score_docs(const sealfm_t* h, int64_t n_queries, const int64_t* query_key_off, const int64_t* key_tok,
                            const int64_t* key_off, const double* key_score, const int64_t* key_count,
                            const int64_t* empty_count, const int64_t* query_doc_off, const int64_t* docs,
                            const int64_t* query_uni_off, const int64_t* uni_tok, const double* uni_val,
                            const int64_t* uni_size, int64_t shift, int32_t sort_mode, int32_t allow_overlaps,
                            int32_t ignore_free_places, int32_t single_key_add_unigrams, double beta, double single_key,
                            int64_t* doc_tok_off, int64_t* doc_tok, int64_t tok_cap, double* out_score, int64_t* out_best,
                            double* out_best_score, int64_t* pick_off, int64_t* pick_key, double* pick_score,
                            int64_t pick_cap, int64_t* pick_needed) {
    return ev_guarded([&] {
        for (int i = 2; i < 4; ++i) g_phase_us[i] = 0.0;
        if (n_queries < 0 || !doc_tok_off || !pick_off || !pick_needed ||
            (n_queries && (!query_key_off || !key_off || !empty_count || !query_doc_off || !query_uni_off || !uni_size)))
            throw ApiError(SEALFM_EINVAL, "null argument");
        const std::vector<uint64_t>& beg = sealfm_beginnings(h);
        const int64_t nd_all = n_queries ? query_doc_off[n_queries] : 0;
        doc_tok_off[0] = 0; pick_off[0] = 0; *pick_needed = 0;
        for (int64_t d = 0; d < nd_all; ++d) {
            if (docs[d] < 0 || (uint64_t)docs[d] + 1 >= beg.size()) throw ApiError(SEALFM_EINVAL, "document id out of range");
            doc_tok_off[d + 1] = doc_tok_off[d] + std::max<int64_t>((int64_t)(beg[docs[d] + 1] - beg[docs[d]]), 1);
        }
        if (doc_tok_off[nd_all] > tok_cap) throw ApiError(SEALFM_ECAPACITY, "token buffer too small");
        if (!nd_all) return;
        const FmView v = sealfm_view(h);
        cudaStream_t s = sealfm_stream(h);
        const int compensated = sealev_compensated_sum() ? 1 : 0;
        const uint64_t tok_budget = std::max<uint64_t>(1, budget_bytes() / 96);     // tokens, with places and scratch
        std::vector<uint64_t> npick_all(nd_all);
        std::vector<std::vector<int64_t>> pk_chunks; std::vector<std::vector<double>> ps_chunks;
        int64_t total_picks = 0;
        for (int64_t q0 = 0; q0 < n_queries;) {
            int64_t q1 = q0;
            uint64_t toks = 0;
            while (q1 < n_queries) {
                const uint64_t t = (uint64_t)(doc_tok_off[query_doc_off[q1 + 1]] - doc_tok_off[query_doc_off[q1]]);
                if (q1 > q0 && toks + t > tok_budget) break;
                toks += t; ++q1;
            }
            const int64_t d0 = query_doc_off[q0], nd = query_doc_off[q1] - d0;
            if (nd == 0) { q0 = q1; continue; }
            Timer tm;
            Arena A(s);
            // ---- extraction: one launch for the chunk's documents ----
            std::vector<uint64_t> b(nd), e(nd), raw_off(nd + 1, 0);
            std::vector<int64_t> toff(nd + 1);
            std::vector<int32_t> dq(nd);
            for (int64_t q = q0; q < q1; ++q)
                for (int64_t d = query_doc_off[q]; d < query_doc_off[q + 1]; ++d) dq[d - d0] = (int32_t)(q - q0);
            for (int64_t i = 0; i < nd; ++i) {
                b[i] = beg[docs[d0 + i]]; e[i] = beg[docs[d0 + i] + 1];
                raw_off[i + 1] = raw_off[i] + (e[i] - b[i]);
                toff[i] = doc_tok_off[d0 + i] - doc_tok_off[d0];
            }
            toff[nd] = doc_tok_off[d0 + nd] - doc_tok_off[d0];
            const uint64_t T = (uint64_t)toff[nd];
            uint64_t* d_raw = A.alloc<uint64_t>(raw_off[nd]);
            uint64_t* d_b = A.put(b); uint64_t* d_e = A.put(e); uint64_t* d_roff = A.put(raw_off);
            int64_t* d_toff = A.put(toff);
            int64_t* d_tok = A.alloc<int64_t>(T);
            extract_docs_kernel<<<grid_for(nd, 64), 64, 0, s>>>(v, (uint64_t)nd, d_b, d_e, d_roff, d_raw);
            doc_tokens_kernel<<<grid_for(nd * 32, 32), 32, 0, s>>>(nd, d_roff, d_raw, d_toff, shift, d_tok);
            CUDA_CHECK(cudaGetLastError());
            A.get(doc_tok + doc_tok_off[d0], d_tok, T);
            A.sync();
            g_phase_us[2] += tm.lap();
            // ---- tries, key arrays, unigram tables of the chunk's queries ----
            HostTrie HT;
            build_tries(q0, q1, query_key_off, key_tok, key_off, key_score, HT);
            const int64_t k0 = query_key_off[q0], nk = query_key_off[q1] - k0;
            std::vector<int64_t> qko(q1 - q0 + 1), koff(nk + 1);
            for (int64_t q = q0; q <= q1; ++q) qko[q - q0] = query_key_off[q] - k0;
            for (int64_t k = 0; k <= nk; ++k) koff[k] = key_off[k0 + k] - key_off[k0];
            std::vector<int64_t> ktok(key_tok + key_off[k0], key_tok + key_off[k0 + nk]);
            const int64_t u0 = query_uni_off[q0], nu = query_uni_off[q1] - u0;
            std::vector<int64_t> uoff(q1 - q0 + 1), utok(nu);
            std::vector<double> uval(nu);
            for (int64_t q = q0; q < q1; ++q) {                  // sort each table by token for the kernel's bisection
                const int64_t a = query_uni_off[q], z = query_uni_off[q + 1];
                std::vector<int64_t> idx(z - a);
                std::iota(idx.begin(), idx.end(), a);
                std::sort(idx.begin(), idx.end(), [&](int64_t x, int64_t y) { return uni_tok[x] < uni_tok[y]; });
                for (int64_t i = 0; i < z - a; ++i) { utok[a - u0 + i] = uni_tok[idx[i]]; uval[a - u0 + i] = uni_val[idx[i]]; }
                uoff[q - q0] = a - u0;
            }
            uoff[q1 - q0] = nu;
            const Trie TD{A.put(HT.root), A.put(HT.child_off), A.put(HT.child_tok), A.put(HT.child_node), A.put(HT.node_key)};
            const ScoreKeys KD{A.put(ktok), A.put(koff), A.put(key_score + k0, nk), A.put(key_count + k0, nk), A.put(HT.rank2key), A.put(qko)};
            const UniTab UD{A.put(uoff), A.put(utok), A.put(uval), A.put(uni_size + q0, q1 - q0)};
            int64_t* d_ec = A.put(empty_count + q0, q1 - q0);
            int32_t* d_dq = A.put(dq);
            // ---- counting pass, then scratch ----
            uint64_t* np = A.alloc<uint64_t>(nd);
            count_places_kernel<<<grid_for(nd, 64), 64, 0, s>>>(nd, d_toff, d_tok, d_dq, TD, np);
            CUDA_CHECK(cudaGetLastError());
            std::vector<uint64_t> np_h(nd);
            A.get(np_h.data(), np, nd);
            A.sync();
            std::vector<uint64_t> place_off(nd + 1, 0), pick_soff(nd + 1, 0);
            std::vector<int64_t> set_off(nd + 1, 0);
            for (int64_t i = 0; i < nd; ++i) {
                const int64_t L = toff[i + 1] - toff[i];
                place_off[i + 1] = place_off[i] + np_h[i];
                pick_soff[i + 1] = pick_soff[i] + np_h[i] + (uint64_t)L;   // key picks <= places, unigram picks <= tokens
                set_off[i + 1] = set_off[i] + (int64_t)set_cap(L);
            }
            ScoreScratch W{A.alloc<uint64_t>(place_off[nd]), A.put(place_off), A.alloc<int64_t>(pick_soff[nd]),
                           A.alloc<double>(pick_soff[nd]), A.put(pick_soff), A.alloc<uint8_t>(T), A.alloc<int64_t>(set_off[nd]),
                           A.put(set_off)};
            double* d_score = A.alloc<double>(nd); int64_t* d_best = A.alloc<int64_t>(nd); double* d_bs = A.alloc<double>(nd);
            uint64_t* d_npick = A.alloc<uint64_t>(nd);
            int* d_err = A.alloc<int>(1);
            CUDA_CHECK(cudaMemsetAsync(d_err, 0, sizeof(int), s));
            score_docs_kernel<<<grid_for(nd, 64), 64, 0, s>>>(nd, d_toff, d_tok, d_dq, TD, KD, d_ec, UD, W, sort_mode, allow_overlaps,
                                                             ignore_free_places, single_key_add_unigrams, compensated, beta,
                                                             single_key, d_score, d_best, d_bs, d_npick, d_err);
            CUDA_CHECK(cudaGetLastError());
            int err = 0;
            A.get(&err, d_err, 1);
            A.get(out_score + d0, d_score, nd); A.get(out_best + d0, d_best, nd); A.get(out_best_score + d0, d_bs, nd);
            A.get(npick_all.data() + d0, d_npick, nd);
            A.sync();
            if (err) throw ApiError(SEALFM_EINVAL, "token id outside the unigram table");
            std::vector<uint64_t> cpo(nd + 1, 0);
            for (int64_t i = 0; i < nd; ++i) cpo[i + 1] = cpo[i] + npick_all[d0 + i];
            uint64_t* d_cpo = A.put(cpo);
            int64_t* d_pk = A.alloc<int64_t>(cpo[nd]); double* d_ps = A.alloc<double>(cpo[nd]);
            compact_picks_kernel<<<grid_for(nd * 32, 32), 32, 0, s>>>(nd, d_npick, d_cpo, W.pick_soff, W.pick_key, W.pick_score, d_pk, d_ps);
            CUDA_CHECK(cudaGetLastError());
            pk_chunks.emplace_back(cpo[nd]); ps_chunks.emplace_back(cpo[nd]);
            A.get(pk_chunks.back().data(), d_pk, cpo[nd]); A.get(ps_chunks.back().data(), d_ps, cpo[nd]);
            A.sync();
            total_picks += (int64_t)cpo[nd];
            g_phase_us[3] += tm.lap();
            q0 = q1;
        }
        for (int64_t d = 0; d < nd_all; ++d) pick_off[d + 1] = pick_off[d] + (int64_t)npick_all[d];
        *pick_needed = total_picks;
        if (total_picks > pick_cap) throw ApiError(SEALFM_ECAPACITY, "pick buffer too small");
        int64_t w = 0;
        for (size_t c = 0; c < pk_chunks.size(); ++c) {
            std::copy(pk_chunks[c].begin(), pk_chunks[c].end(), pick_key + w);
            std::copy(ps_chunks[c].begin(), ps_chunks[c].end(), pick_score + w);
            w += (int64_t)pk_chunks[c].size();
        }
    });
}

}  // extern "C"
