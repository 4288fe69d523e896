// Warp-cooperative expansion of the distinct symbols of an SA range (wt_int::interval_symbols,
// sdsl/wt_int.hpp:489-509) — shared by the stand-alone expand kernels (fm_kernels.cu) and the fused
// decode step (decode_kernels.cuh).
#pragma once
#include "fm_device.cuh"

namespace sealb200 {

struct MaskSink {
    uint32_t* row;        // bitmask row
    uint32_t vocab, shift;
    __device__ void operator()(uint32_t symbol, uint64_t, uint64_t) const {
        // seal/index.py:141,153: the sentinel (0) is dropped, tokens are symbol - SHIFT
        if (symbol < shift || symbol == 0) return;
        const uint32_t tok = symbol - shift;
        if (tok < vocab) atomicOr(row + (tok >> 5), 1u << (tok & 31));
    }
};
// (symbol, count) pairs appended in discovery order to a per-range list + a presence bitmap over the symbol space;
// order_pairs_kernel (fm_kernels.cu) turns that into the ascending-symbol output of FMIndex::distinct_count
// (fm_index.cpp:91-109) without the reference's (and round 1's) dense sigma-wide scratch per range.
struct PairSink {
    uint64_t* list;           // this range's unordered pairs
    unsigned int* counter;    // pairs appended so far
    uint32_t* present;        // 2^L / 32 words, zeroed
    __device__ void operator()(uint32_t symbol, uint64_t ri, uint64_t rj) const {
        const unsigned int k = atomicAdd(counter, 1u);
        list[2ull * k] = symbol; list[2ull * k + 1] = rj - ri;
        atomicOr(present + (symbol >> 5), 1u << (symbol & 31));
    }
};

// Depth-first expansion below (level, prefix) WITHOUT a local-memory stack.  A thread only ever has to remember
// the right sibling of the nodes on its current root-to-node path where both children exist: at most one (i, j)
// pair per tree level.  Those live in shared memory ([level][slot], conflict-free), a 32-bit mask says which
// levels are pending, and the prefix of a popped sibling is rebuilt from the current prefix (the ancestor at that
// level is the left child).  The previous per-thread `Frame stk[36]` (48-byte frames in local memory) produced
// several times the algorithmic traffic in the wide regime.  The children's node-table
// entries share one 32-byte sector and are fetched together with the rank sectors, so a level costs ONE dependent
// memory round trip; a popped sibling re-reads its entry (once per branching node, top-of-tree entries are cache-hot).
// Symbols are delivered in ascending order per call, like wt_int::_interval_symbols (sdsl/wt_int.hpp:108-147).
template <typename Sink>
__device__ __forceinline__ void expand_dfs_smem(const FmView& v, uint32_t level, uint32_t prefix, uint64_t i, uint64_t j, Sink& sink,
                                                uint64_t* __restrict__ stk_i, uint64_t* __restrict__ stk_j, int stride, int slot) {
    const uint32_t L = v.L;
    uint32_t pending = 0;
    NodeEntry e{0, 0};
    if (level < L) e = load_node(v, (1u << level) + prefix);
    for (;;) {
        if (level == L) {
            sink(prefix, i, j);
        } else {
            NodeEntry c0{0, 0}, c1{0, 0};
            if (level + 1 < L) {
                const uint32_t h = (2u << level) + 2u * prefix;
                c0 = load_node(v, h); c1 = load_node(v, h + 1);
            }
            uint64_t a, b;
            if (j == i + 1) {                                  // single position: one sector, take the bit
                int bit;
                a = rank1(v, e.base + i, &bit) - e.ones;
                b = a + static_cast<uint64_t>(bit);
            } else {
                a = rank1(v, e.base + i) - e.ones;
                b = rank1(v, e.base + j) - e.ones;
            }
            const bool has1 = b != a, has0 = (j - i) != (b - a);
            if (has0) {
                if (has1) { stk_i[level * stride + slot] = a; stk_j[level * stride + slot] = b; pending |= 1u << level; }
                i -= a; j -= b; prefix <<= 1; e = c0; ++level;
                continue;
            }
            if (has1) { i = a; j = b; prefix = (prefix << 1) | 1u; e = c1; ++level; continue; }
        }
        if (!pending) break;
        const uint32_t l = 31u - static_cast<uint32_t>(__clz(pending));
        pending &= ~(1u << l);
        prefix = (prefix >> (level - (l + 1))) | 1u;           // ancestor at level l+1 is a left child: its right sibling
        level = l + 1;
        i = stk_i[l * stride + slot]; j = stk_j[l * stride + slot];
        e = NodeEntry{0, 0};
        if (level < L) e = load_node(v, (1u << level) + prefix);
    }
}

// One warp expands one SA range.  Phase 1: level-synchronous frontier expansion, one lane per
// frontier node, children compacted in order with a shuffle scan (frontier lives in shared memory).
// Phase 2: once the frontier is wider than a warp, every lane walks its own subtrees depth-first.
constexpr int kMaxLevels = 24;                 // wavelet-tree height bound (SEAL: 16)
struct WarpFrontier {
    uint64_t i[2][64];
    uint64_t j[2][64];
    uint32_t prefix[2][64];
};
// shared memory one warp needs for warp_expand on a tree of height L: the frontier + 2 x L x 32 u64 of DFS stack
__host__ __device__ inline size_t warp_expand_smem(uint32_t L) { return sizeof(WarpFrontier) + 2ull * L * 32 * 8; }

// stk: 2 x L x 32 u64 of shared memory owned by this warp (pending right siblings of the depth-first phase)
template <typename Sink>
__device__ void warp_expand(const FmView& v, uint64_t lo, uint64_t hi, Sink& sink, WarpFrontier& F, uint64_t* stk) {
    if (lo >= hi) return;                                  // fm_index.cpp:98 `if (low == high) return`
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t L = v.L;
    uint32_t n = 1, level = 0, cur = 0;
    if (lane == 0) { F.i[0][0] = lo; F.j[0][0] = hi; F.prefix[0][0] = 0; }
    __syncwarp();
    while (level < L && n <= 32) {
        uint32_t nc = 0;
        uint64_t a = 0, b = 0, ei = 0, ej = 0;
        uint32_t ep = 0;
        bool has0 = false, has1 = false;
        if (lane < n) {
            ei = F.i[cur][lane]; ej = F.j[cur][lane]; ep = F.prefix[cur][lane];
            const NodeEntry ne = load_node(v, (1u << level) + ep);
            const uint64_t base = ne.base, o1 = ne.ones;
            if (ej == ei + 1) {
                int bit;
                a = rank1(v, base + ei, &bit) - o1;
                b = a + static_cast<uint64_t>(bit);
            } else {
                a = rank1(v, base + ei) - o1;
                b = rank1(v, base + ej) - o1;
            }
            has1 = (b - a) != 0;
            has0 = ((ej - ei) - (b - a)) != 0;
            nc = (has0 ? 1u : 0u) + (has1 ? 1u : 0u);
        }
        uint32_t incl = nc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= (uint32_t)d) incl += t;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t w = incl - nc;
        const uint32_t nxt = cur ^ 1;
        if (has0) { F.i[nxt][w] = ei - a; F.j[nxt][w] = ej - b; F.prefix[nxt][w] = ep << 1; ++w; }
        if (has1) { F.i[nxt][w] = a; F.j[nxt][w] = b; F.prefix[nxt][w] = (ep << 1) | 1u; }
        __syncwarp();
        cur = nxt; n = total; ++level;
    }
    for (uint32_t e = lane; e < n; e += 32)
        expand_dfs_smem(v, level, F.prefix[cur][e], F.i[cur][e], F.j[cur][e], sink, stk, stk + (size_t)L * 32, 32, (int)lane);
}



// Shared-memory frontier of the block-cooperative expansion of WIDE ranges (block_expand_bfs below).
template <int CAP>
struct BlockFrontierT {
    static constexpr int kCap = CAP;
    uint64_t i[2][CAP];
    uint64_t j[2][CAP];
    uint32_t prefix[2][CAP];
    int count[2];
};
using BlockFrontier = BlockFrontierT<1024>;   // 40 KB: five 256-thread CTAs per SM
constexpr uint64_t kWideRange = 2048;       // ranges at least this wide go to the block path


// Level-synchronous expansion of one WIDE range by a whole CTA -- no depth-first phase, no per-thread stack: the
// frontier of level l (at most 2^l nodes, (i, j, prefix) each) lives in shared memory while it fits and in this CTA's
// global scratch (two buffers of 2^(L-1) entries; L2-resident) beyond that; every thread takes frontier entries in a
// strided loop, so a range with thousands of distinct successors keeps all 256 threads on independent rank queries
// at every level (the depth-first hand-out left threads walking sub-trees of very different sizes, and its stacks
// capped the occupancy at 512 threads per SM).  Children of the last level go straight to the sink.
// Visits exactly the nodes wt_int::_interval_symbols visits (sdsl/wt_int.hpp:108-147); order-independent sinks only.
struct GlobalFrontier {
    uint64_t* i; uint64_t* j; uint32_t* prefix;      // [2][cap] each
    uint32_t cap;                                    // entries per buffer (>= 2^(L-1))
};
__host__ __device__ inline size_t global_frontier_bytes(uint32_t L) { return (size_t)2 * ((size_t)1 << (L - 1)) * 20; }

template <typename Sink, typename Frontier>
__device__ void block_expand_bfs(const FmView& v, uint64_t lo, uint64_t hi, Sink& sink, Frontier& F, const GlobalFrontier& G) {
    if (lo >= hi) return;                                      // uniform
    const int tid = threadIdx.x, nt = blockDim.x;
    const uint32_t L = v.L;
    __syncthreads();
    if (tid == 0) { F.i[0][0] = lo; F.j[0][0] = hi; F.prefix[0][0] = 0; F.count[0] = 1; F.count[1] = 0; }
    __syncthreads();
    int cur = 0, n = 1;
    bool cur_global = false;
    for (uint32_t level = 0; level < L; ++level) {
        const int nxt = cur ^ 1;
        const bool last = level + 1 == L;
        const bool nxt_global = !last && 2 * n > Frontier::kCap;          // uniform: an upper bound on the children
        const uint64_t* ci = cur_global ? G.i + (size_t)cur * G.cap : F.i[cur];
        const uint64_t* cj = cur_global ? G.j + (size_t)cur * G.cap : F.j[cur];
        const uint32_t* cp = cur_global ? G.prefix + (size_t)cur * G.cap : F.prefix[cur];
        uint64_t* ni = nxt_global ? G.i + (size_t)nxt * G.cap : F.i[nxt];
        uint64_t* nj = nxt_global ? G.j + (size_t)nxt * G.cap : F.j[nxt];
        uint32_t* np = nxt_global ? G.prefix + (size_t)nxt * G.cap : F.prefix[nxt];
        for (int e = tid; e < n; e += nt) {
            const uint64_t ei = ci[e], ej = cj[e];
            const uint32_t ep = cp[e];
            const NodeEntry ne = load_node(v, (1u << level) + ep);
            uint64_t a, b;
            if (ej == ei + 1) {
                int bit;
                a = rank1(v, ne.base + ei, &bit) - ne.ones;
                b = a + static_cast<uint64_t>(bit);
            } else {
                a = rank1(v, ne.base + ei) - ne.ones;
                b = rank1(v, ne.base + ej) - ne.ones;
            }
            const bool has1 = b != a, has0 = (ej - ei) != (b - a);
            if (last) {
                if (has0) sink(ep << 1, ei - a, ej - b);
                if (has1) sink((ep << 1) | 1u, a, b);
            } else {
                const int nc = (has0 ? 1 : 0) + (has1 ? 1 : 0);
                int w = atomicAdd(&F.count[nxt], nc);
                if (has0) { ni[w] = ei - a; nj[w] = ej - b; np[w] = ep << 1; ++w; }
                if (has1) { ni[w] = a; nj[w] = b; np[w] = (ep << 1) | 1u; }
            }
        }
        __syncthreads();                                       // (global frontier writes are block-visible after the barrier)
        n = F.count[nxt];
        __syncthreads();
        if (tid == 0) F.count[cur] = 0;
        cur = nxt; cur_global = nxt_global;
        __syncthreads();
    }
}
}  // namespace sealb200
