// Hopper (sm_90a) GEMM for the BART encoder/decoder linears and the lm_head:
//   C[M,N] = A[M,K] * W[N,K]^T + bias[N]   (optional exact GELU or ReLU), fp32 in / fp32 out,
// computed on the tensor cores as an error-compensated 3-pass product
//   A*W ~= A_lo*W_hi + A_hi*W_lo + A_hi*W_hi,
// which keeps the fp32-level accuracy the 1e-4 beam-score parity needs (a single TF32/FP16 pass does not).
// Three operand splits (operand_split.cuh):
//   3xFP16 (gemm_mode 3 / 5): x = h1 + h2, h1 = rn_half(x), h2 = rn_half(x - h1).  fp16 products are exact in the
//     fp32 accumulator, so the accuracy class is that of 3xTF32 at half the operand bytes and twice the tensor rate --
//     for activations of magnitude at least 2^-3.  Activations are used unscaled (|x| must stay below 65504; the
//     producers saturate and raise a sticky flag otherwise).  |x - h1| <= 2^-11 |x|, so below about 2^-3 the low half
//     h2 is an fp16 subnormal (spacing 2^-24) and below 2^-14 h1 is too: each such activation carries an absolute
//     error of up to 2^-25 (relative 2^-19 at 2^-6, 2^-11 at 2^-14), and below 2^-25 it flushes to zero.  Element
//     (i, j) is then good to about
//     sum_k |w_jk| * max(2^-22 |a_ik|, 2^-25), not 2^-22 sum_k |a_ik w_jk| (tests/test_gemm_range_gpu.py); at the
//     BART activation scales that floor is far below the forward's rounding.  Each weight matrix is pre-multiplied by a power of two 2^s so that max|W| ~ 2^14 and the epilogue
//     multiplies the accumulator by 2^-s (exact).
//   3xTF32 (gemm_mode 2, fp32 range): hi = x with the 13 low mantissa bits cleared, lo = x - hi (exact).
//   3xBF16 (gemm_mode 6, bf16 weights): W is stored once in bf16 (exact for a bf16 checkpoint), A = b1 + b2 + b3 in
//     bf16 pieces (exact for 2^-100 <= |a| < (2 - 2^-8) 2^127) and A*W = b3*W + b2*W + b1*W.  Each
//     product has 8 x 8 significant bits, exact in the fp32 accumulator, so the only error is the accumulation's --
//     at any magnitude in fp32's range, with no absolute floor and no overflow flag.  The stage holds A b1, A b2, W and
//     A b3 in the four 16 KB slots the other modes use for A hi / lo and W hi / lo.
//
// Kernel: persistent, 128 x 128 output tile per CTA, three warpgroups.  Warpgroup 0 is the producer (one thread
// issues the TMA loads of A hi/lo and W hi/lo into 128B-swizzled K-major shared-memory stages, and warp 1 stages each
// tile's bias slice in shared memory for the epilogue); warpgroups 1 and 2
// each own 64 rows of the tile and issue wgmma.mma_async (m64n128, both operands from shared memory) into register
// accumulators.  Stage hand-off uses mbarriers (full: TMA transaction bytes; empty: one arrive per consumer warp).
// With CL = 2 (gemm_mode 5) two CTAs of a cluster compute vertically adjacent tiles that share the W tile: each CTA
// loads half of the W rows and multicasts them to both, which halves the W traffic out of L2.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>

#include "decode_types.cuh"
#include "launch.cuh"
#include "operand_split.cuh"

namespace sealb200 {

constexpr int GSTAGES = 3;
constexpr int GTHREADS = 384;                        // producer warpgroup + 2 consumer warpgroups
constexpr int G_AB = GM * 128;                       // one A tile (hi or lo): 128 rows x 128 B of K
constexpr int G_WB = GN * 128;                       // one W tile (hi or lo)
constexpr int G_STAGE = 2 * G_AB + 2 * G_WB;         // 64 KB
constexpr int G_BARS = 64;                           // mbarriers: full / empty per stage, bias full / empty
constexpr int G_BIAS = GN * 4;                       // the unit's 128-column bias slice, fp32
constexpr int G_SMEM = GSTAGES * G_STAGE + 1024 /*alignment slack*/ + G_BARS + G_BIAS;
static_assert(8 * (2 * GSTAGES + 2) <= G_BARS, "barrier area");
constexpr int UK16 = 64;                             // 3xFP16 k-block: 64 halves = one 128-byte swizzle row
constexpr int UK = 32;                               // 3xTF32 k-block: 32 floats

// Per operand type: K elements per k-block, K per wgmma, and k-blocks per register chunk.  The tensor core adds into
// its fp32 accumulator with truncation, so a long K loop drifts by ~N_adds * 2^-24 relative, in one direction --
// enough at K = 1024..4096 to push summed beam scores past the 1e-4 parity bound.  The K loop is therefore cut into
// chunks (48 tensor-core adds for 3xFP16, 24 for 3xTF32): each chunk accumulates from zero in the wgmma registers
// and is then added, with round-to-nearest, into a second set of fp32 registers.
template <typename T> struct GemmElem;
template <> struct GemmElem<__half> { static constexpr int KE = 64, KSTEP = 16, CHUNK = 4; };
template <> struct GemmElem<float> { static constexpr int KE = 32, KSTEP = 8, CHUNK = 2; };
template <> struct GemmElem<__nv_bfloat16> { static constexpr int KE = 64, KSTEP = 16, CHUNK = 4; };

// ---- PTX wrappers --------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded spin: a protocol bug must trap (error code back to the host), never hang the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (!done && spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t map_to_cta(uint32_t addr, uint32_t rank) {
    uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}
// Consumer release of a stage: one arrive on the empty barrier of each CTA whose producer refills the stage.  The
// stage was read only by wgmma (async proxy), which wgmma.wait_group has retired, so no generic-proxy writes need to
// be ordered before the producer's next TMA: the arrive takes the default .release.cta semantics.  A .release.cluster
// arrive puts a cluster-scope fence in every consumer warp at every k-block: at the benchmark's shapes it cost the
// one-CTA kernel 18-30 % of its time and the 2-CTA kernel 36 % (H100 SXM, 700 W; DESIGN.md section 4).
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
// the box lands at offset dst in every CTA of `mask`, completing bytes on the barrier at offset bar in each of them
__device__ __forceinline__ void tma_load_2d_multicast(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(mask) : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma): start >> 4 | LBO (unused for swizzled K-major,
// 1) << 16 | SBO = 1024 B between 8-row groups (>> 4) << 32 | layout SWIZZLE_128B (1) << 62.  Advancing K by 32 bytes
// inside the 128-byte row adds 2 to the address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define SEAL_WG_D64                                                                                              \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "  \
    "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
#define SEAL_WG_OPS(d)                                                                                           \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),      \
    "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),          \
    "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),         \
    "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),         \
    "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),         \
    "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),         \
    "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),         \
    "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// D[64 x 128] += A[64 x K] * B[128 x K]^T, both operands K-major in shared memory (scale-d = 1: D is zeroed per chunk)
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t a, uint64_t b, __half) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " SEAL_WG_D64 ", %64, %65, 1, 1, 1, 0, 0;"
                 : SEAL_WG_OPS(d) : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t a, uint64_t b, float) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " SEAL_WG_D64 ", %64, %65, 1, 1, 1;"
                 : SEAL_WG_OPS(d) : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_128(float (&d)[64], uint64_t a, uint64_t b, __nv_bfloat16) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " SEAL_WG_D64 ", %64, %65, 1, 1, 1, 0, 0;"
                 : SEAL_WG_OPS(d) : "l"(a), "l"(b));
}
#undef SEAL_WG_D64
#undef SEAL_WG_OPS

__device__ __forceinline__ float gelu_erf_u(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// Epilogue activation ACT (kActNone, kActGelu, kActRelu: decode_types.cuh)
template <int ACT> __device__ __forceinline__ float epi_act(float x) {
    return ACT == kActGelu ? gelu_erf_u(x) : ACT == kActRelu ? (x < 0.f ? 0.f : x) : x;
}

// x * scale -> format T's pieces p0, p1 (, p2), for weights (once) and for activations whose producer did not split;
// a value the fp16 split saturated raises *overflow
template <typename T>
__global__ void __launch_bounds__(256) split_kernel(int64_t n, const float* __restrict__ x, float scale, T* __restrict__ p0,
                                                    T* __restrict__ p1, T* __restrict__ p2, int* __restrict__ overflow) {
    T* const s[3] = {p0, p1, p2};
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int ov = 0;
        store_split<T, 1>(s, i, {x[i] * scale}, ov);
        if (ov) atomicExch(overflow, 1);
    }
}

__global__ void __launch_bounds__(256) absmax_kernel(int64_t n, const float* __restrict__ x, unsigned int* __restrict__ out) {
    float m = 0.f;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = fabsf(x[i]);
        if (v == v && v != INFINITY) m = fmaxf(m, v);
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));       // non-negative floats order like uints
}

// Optional in-kernel timeline of CTA 0 (debug ABI sealdec_debug_gemm_trace): SM cycle counter at 0 entry,
// 1 prologue done, 2 first operands landed, 3 last MMA of the first tile issued, 4 its last chunk complete,
// 5 tile stored, 6 exit; 7/8 = %globaltimer (ns) at entry / exit.
__device__ long long g_gemm_trace[20];
__device__ int g_gemm_trace_on;
__device__ __forceinline__ void gemm_trace(int i) {
    if (blockIdx.x == 0 && g_gemm_trace_on) {
        g_gemm_trace[i] = clock64();
        if (i == 0 || i == 6) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); g_gemm_trace[i == 0 ? 7 : 8] = (long long)t; }
    }
}
// Per-unit timeline of CTA 0 (consumer warpgroup 1, thread 0) under the same switch (debug ABI
// sealdec_debug_gemm_units), compiled in only with -DSEAL_GEMM_UNIT_TRACE (make GEMM_UNIT_TRACE=1): the stamps cost the
// lm_head 5 % even with tracing off (H100 SXM, 700 W), so the default build leaves them out: for its i-th work unit, i < kTraceUnits, SM cycles at 4i + 0 the unit's first k-block of
// MMAs committed, 1 its K loop done (last chunk promoted), 2 epilogue start, 3 epilogue end.  From these,
// tools/gemm_epilogue_probe.py reports the epilogue's share of the CTA's time and the tensor-idle gap between a unit's
// last and the next unit's first MMAs.
constexpr int kTraceUnits = 256;
__device__ long long g_gemm_units[4 * kTraceUnits];
__device__ __forceinline__ void unit_trace(bool on, int unit, int e) {
#ifdef SEAL_GEMM_UNIT_TRACE
    if (on && unit < kTraceUnits) g_gemm_units[4 * unit + e] = clock64();
#endif
}

// Epilogue store of two adjacent columns (n, n + 1) of one row: fp32 to C and/or format T's split of the next GEMM's
// operand to S (S[0] == nullptr: none).  kFull: the caller knows both columns are below N (a tile inside the matrix),
// so neither is checked.
template <bool kFull, typename T>
__device__ __forceinline__ void store_pair(float* C, T* const* S, int64_t off, int n, int N, float v0, float v1, int& ov) {
    if (kFull || n + 1 < N) {
        if (C) *reinterpret_cast<float2*>(C + off) = make_float2(v0, v1);
        if (S[0]) store_split<T, 2>(S, off, {v0, v1}, ov);
    } else if (n < N) {
        if (C) C[off] = v0;
        if (S[0]) store_split<T, 1>(S, off, {v0}, ov);
    }
}

// Tile group (mg, n_tile) of work index `tile`.  n_fastest: row-major over (m group, n tile).  Otherwise the m groups
// are walked in bands of `band` groups (0: one band of all of them), band after band; inside a band the walk is
// n-major with m fastest, so the concurrent CTAs share W tiles and the band's A rows are re-read from L2, not HBM.
// Producer and consumers of a CTA must agree on this mapping.
__device__ __forceinline__ void tile_coords(int tile, int n_fastest, int band, int m_groups, int n_tiles, int& mg, int& n_tile) {
    if (n_fastest) { mg = tile / n_tiles; n_tile = tile % n_tiles; return; }
    if (band <= 0 || band > m_groups) band = m_groups;
    const int b0 = tile / (band * n_tiles) * band;                       // first m group of the band
    const int rows = min(band, m_groups - b0);
    const int r = tile - b0 * n_tiles;
    n_tile = r / rows; mg = b0 + r % rows;
}

// T = __half (3xFP16), float (3xTF32) or __nv_bfloat16 (3xBF16: tmA_hi / tmA_lo / tmW_lo are A's pieces b1 / b2 / b3,
// tmW_hi is W; C_s1 / C_s2 / C_s3 the three output pieces); CL = CTAs per cluster sharing the W tile (1 or 2).
// Persistent: work unit u = blockIdx.x / CL walks units u, u + gridDim.x / CL, ...  A unit is (tile group, K slice);
// a tile group is CL vertically adjacent 128 x 128 tiles.  Tile order is chosen by the host (tile_coords): n fastest
// when the activations dominate (concurrent CTAs then share A tiles and all of W stays in L2), m fastest when the
// weights dominate (lm_head).  With m fastest each n column re-reads all of A, which streams from HBM once per column
// when A is larger than the L2 (lm_head at 15 000 rows: 61 MB of A halves, 393 columns); m_band > 0 then bounds the
// A rows in flight to a band that stays in L2, so A is read from HBM once and W once per band.
// Split-K (CL = 1 only; skinny M, where a handful of tiles would leave most SMs idle): slice s accumulates k-blocks
// [s*num_k, (s+1)*num_k) and stores its raw fp32 partial tile at C + s*slice_stride (the caller passes bias = nullptr,
// w_unscale = 1, no split outputs; gemm_splitk_finish_kernel or the consumer kernel sums the slices in a fixed order).
// Registers: the CTA launches at 128 per thread (49 152 of the SM's 65 536), then the producer warpgroup, whose one live
// thread only issues TMA, gives its share back (40) and the consumer warpgroups take 168 each (128 x 40 + 256 x 168 <=
// 384 x 128).  The 16 384 registers left over (and the ~33 KB of shared memory) let small memory-bound kernels of another
// stream -- add+LN, cross attention -- run beside a GEMM CTA on the same SM.
constexpr int G_REGS = 128, G_REGS_PRODUCER = 40, G_REGS_CONSUMER = 168;
static_assert(128 * G_REGS_PRODUCER + 256 * G_REGS_CONSUMER <= GTHREADS * G_REGS, "setmaxnreg budget");
template <typename T, int ACT, int CL, bool HEAD = false>
__global__ void __maxnreg__(G_REGS)                   // (excludes __launch_bounds__; launched with GTHREADS threads)
wgmma_gemm_x3_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                     const __grid_constant__ CUtensorMap tmW_hi, const __grid_constant__ CUtensorMap tmW_lo,
                     int M, int N, int K, const float* __restrict__ bias, float w_unscale, float* __restrict__ C,
                     T* __restrict__ C_s1, T* __restrict__ C_s2, int ldc, int n_fastest, int m_band, int* __restrict__ overflow,
                     int k_slices, int64_t slice_stride, HeadEpi he, T* __restrict__ C_s3) {
    using E = GemmElem<T>;
    constexpr bool kBf16 = std::is_same<T, __nv_bfloat16>::value;
    static_assert(!kBf16 || CL == 1, "3xBF16 runs one CTA per tile");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;          // SWIZZLE_128B wants 1024 B alignment
    const uint32_t full0 = base + GSTAGES * G_STAGE, empty0 = full0 + 8 * GSTAGES;
    const uint32_t bias_full = empty0 + 8 * GSTAGES, bias_empty = bias_full + 8;
    float* const bias_s = reinterpret_cast<float*>(smem_raw + (full0 + G_BARS - smem_u32(smem_raw)));
    const int wg = threadIdx.x >> 7;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0;
    if (threadIdx.x == 0) gemm_trace(0);

    const int m_tiles = (M + GM - 1) / GM, n_tiles = (N + GN - 1) / GN;
    const int m_groups = (m_tiles + CL - 1) / CL;
    const int total = m_groups * n_tiles * k_slices;
    const int num_k = (K / E::KE) / k_slices;
    const int num_chunks = (num_k + E::CHUNK - 1) / E::CHUNK;
    const int unit0 = blockIdx.x / CL, n_units = gridDim.x / CL;

    if (threadIdx.x == 0) {
        for (int s = 0; s < GSTAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8 * CL); }
        mbar_init(bias_full, 32); mbar_init(bias_empty, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();                                        // the peer's barriers exist before anything targets them
    if (threadIdx.x == 0) gemm_trace(1);

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(G_REGS_PRODUCER));
        if (threadIdx.x == 0) {
            uint32_t it = 0;                                               // k-blocks issued so far (all units)
            for (int u = unit0; u < total; u += n_units) {
                const int tile = u / k_slices, kb0 = (u % k_slices) * num_k;
                int mg, n_tile;
                tile_coords(tile, n_fastest, m_band, m_groups, n_tiles, mg, n_tile);
                const int row_a = (mg * CL + (int)rank) * GM;
                for (int kb = 0; kb < num_k; ++kb, ++it) {
                    const int s = it % GSTAGES;
                    mbar_wait(empty0 + 8 * s, ((it / GSTAGES) & 1) ^ 1);
                    const uint32_t st = base + s * G_STAGE, fb = full0 + 8 * s;
                    const int kx = (kb0 + kb) * E::KE;
                    mbar_expect_tx(fb, G_STAGE);
                    tma_load_2d(st, &tmA_hi, fb, kx, row_a);
                    tma_load_2d(st + G_AB, &tmA_lo, fb, kx, row_a);
                    if (kBf16) {
                        tma_load_2d(st + 2 * G_AB, &tmW_hi, fb, kx, n_tile * GN);
                        tma_load_2d(st + 2 * G_AB + G_WB, &tmW_lo, fb, kx, row_a);
                    } else if (CL == 1) {
                        tma_load_2d(st + 2 * G_AB, &tmW_hi, fb, kx, n_tile * GN);
                        tma_load_2d(st + 2 * G_AB + G_WB, &tmW_lo, fb, kx, n_tile * GN);
                    } else {                                               // this CTA's share of the W rows, to both CTAs
                        const uint32_t part = rank * (G_WB / CL);
                        const int row_w = n_tile * GN + (int)rank * (GN / CL);
                        tma_load_2d_multicast(st + 2 * G_AB + part, &tmW_hi, fb, kx, row_w, (uint16_t)((1u << CL) - 1));
                        tma_load_2d_multicast(st + 2 * G_AB + G_WB + part, &tmW_lo, fb, kx, row_w, (uint16_t)((1u << CL) - 1));
                    }
                }
            }
        } else if (threadIdx.x >> 5 == 1) {
            // Warp 1 stages each unit's bias slice (0 past N, or everywhere without a bias) in shared memory during the
            // unit's K loop, so that the epilogue reads no global memory: a global load issued there waits behind the
            // next unit's operand stages, which the producer has already put in flight (DESIGN.md section 10).  One
            // buffer: it is refilled after both consumer warpgroups have finished the previous unit's epilogue, a whole
            // K loop before it is read.
            const int lane = threadIdx.x & 31;
            for (int u = unit0, ui = 0; u < total; u += n_units, ++ui) {
                int mg, n_tile;
                tile_coords(u / k_slices, n_fastest, m_band, m_groups, n_tiles, mg, n_tile);
                mbar_wait(bias_empty, (ui & 1) ^ 1);
                for (int i = lane; i < GN; i += 32) {
                    const int n = n_tile * GN + i;
                    bias_s[i] = bias && n < N ? bias[n] : 0.f;
                }
                mbar_arrive(bias_full);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(G_REGS_CONSUMER));
        const int t = threadIdx.x - 128 * wg, warp = t >> 5, lane = t & 31;
        const uint32_t a_off = (uint32_t)(wg - 1) * 64 * 128;               // this warpgroup's 64 rows of the A tile
        uint32_t empty_peer[CL];
#pragma unroll
        for (int r = 0; r < CL; ++r) empty_peer[r] = CL > 1 ? map_to_cta(empty0, r) : empty0;
        auto release = [&](int stage) {
            if (CL == 1) mbar_arrive(empty0 + 8 * stage);
            else
#pragma unroll
                for (int r = 0; r < CL; ++r) mbar_arrive_cluster(empty_peer[r] + 8 * stage);
        };
        const bool tr = blockIdx.x == 0 && t == 0 && wg == 1 && g_gemm_trace_on;
        uint32_t it = 0;
        bool first = true;
        for (int u = unit0, ui = 0; u < total; u += n_units, ++ui) {
            const int tile = u / k_slices;
            float acc[64];
#pragma unroll
            for (int j = 0; j < 64; ++j) acc[j] = 0.f;
            int kb = 0;
            for (int c = 0; c < num_chunks; ++c) {
                float d[64];
#pragma unroll
                for (int j = 0; j < 64; ++j) d[j] = 0.f;
                int prev_s = -1;
                const int kend = (kb + E::CHUNK < num_k) ? kb + E::CHUNK : num_k;
                for (; kb < kend; ++kb, ++it) {
                    const int s = it % GSTAGES;
                    mbar_wait(full0 + 8 * s, (it / GSTAGES) & 1);
                    if (first && t == 0 && wg == 1) gemm_trace(2);
                    const uint32_t st = base + s * G_STAGE;
                    const uint64_t a_hi = gmma_desc_sw128(st + a_off), a_lo = gmma_desc_sw128(st + G_AB + a_off);
                    const uint64_t w_hi = gmma_desc_sw128(st + 2 * G_AB), w_lo = gmma_desc_sw128(st + 2 * G_AB + G_WB);
                    acc_fence(d);
                    wgmma_fence();
                    if constexpr (kBf16) {
                        const uint64_t a_b3 = gmma_desc_sw128(st + 2 * G_AB + G_WB + a_off);   // w_hi = W, a_hi / a_lo = b1 / b2
#pragma unroll
                        for (int k = 0; k < E::KE / E::KSTEP; ++k) {
                            wgmma_128(d, a_b3 + 2 * k, w_hi + 2 * k, T{});
                            wgmma_128(d, a_lo + 2 * k, w_hi + 2 * k, T{});
                            wgmma_128(d, a_hi + 2 * k, w_hi + 2 * k, T{});
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < E::KE / E::KSTEP; ++k) {       // KSTEP elements = 32 B -> +2 in the address field
                            wgmma_128(d, a_lo + 2 * k, w_hi + 2 * k, T{});
                            wgmma_128(d, a_hi + 2 * k, w_lo + 2 * k, T{});
                            wgmma_128(d, a_hi + 2 * k, w_hi + 2 * k, T{});
                        }
                    }
                    wgmma_commit();
                    if (kb == 0) unit_trace(tr, ui, 0);
                    wgmma_wait<1>();                                       // the previous k-block's MMAs have retired
                    acc_fence(d);
                    if (prev_s >= 0) {
                        __syncwarp();
                        if (lane == 0) release(prev_s);
                    }
                    prev_s = s;
                }
                wgmma_wait<0>();
                acc_fence(d);
                __syncwarp();
                if (lane == 0) release(prev_s);
#pragma unroll
                for (int j = 0; j < 64; ++j) acc[j] += d[j];              // round-to-nearest promotion
            }
            unit_trace(tr, ui, 1);
            if (first && t == 0 && wg == 1) gemm_trace(4);
            // accumulator layout of m64n128: warp w holds rows 16w + lane/4 (+8); register 4j + {0,1} / {2,3} holds
            // columns 8j + 2 (lane % 4) + {0, 1} of the first / second of those rows
            int mg, n_tile;
            tile_coords(tile, n_fastest, m_band, m_groups, n_tiles, mg, n_tile);
            const int row0 = (mg * CL + (int)rank) * GM + (wg - 1) * 64 + warp * 16 + (lane >> 2);
            const int col0 = n_tile * GN + 2 * (lane & 3);
            float* Cs = C ? C + (int64_t)(u % k_slices) * slice_stride : nullptr;
            T* const S[3] = {C_s1, C_s2, C_s3};                             // the split outputs (C_s3: 3xBF16 only)
            const float* const bq = bias_s + 2 * (lane & 3);               // the bias of column col0 + 8 j + e is bq[8 j + e]
            int ov = 0;
            mbar_wait(bias_full, ui & 1);
            unit_trace(tr, ui, 2);
            // The epilogue is compiled twice: for tiles whose 128 columns all lie below N (every n tile but a ragged
            // last one), with no per-column bounds checks, and for the edge tile, with them.  On a full tile every
            // check is true, so both give the same stores; the full form drops the checks and the single-column
            // fallback stores from the code the tensor cores wait on (DESIGN.md section 10).
            auto epilogue = [&](auto full) {
                constexpr bool kFull = decltype(full)::value;
                if constexpr (HEAD) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = row0 + 8 * h;
                        // the row's logits, computed once in place (acc is not read again) and read by the three passes
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                float& x = acc[4 * j + 2 * h + e];
                                x = kFull || col0 + 8 * j + e < N ? x * w_unscale + bq[8 * j + e] : -INFINITY;
                            }
                        }
                        auto xv = [&](int j, int e) { return acc[4 * j + 2 * h + e]; };
                        // the mask words are loaded before the reductions, whose arithmetic hides their latency
                        const uint32_t* mrow = he.mask + (int64_t)row * he.mask_words;
                        uint32_t w[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) w[i] = row < M && (kFull || n_tile * 4 + i < he.mask_words) ? mrow[n_tile * 4 + i] : 0u;
                        // the 4 lanes of a quad hold the row's 128 columns: reduce across them (all lanes take part)
                        float mx = -INFINITY;
#pragma unroll
                        for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(xv(j, 0), xv(j, 1)));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                        float se = 0.f;
                        if (mx > -INFINITY) {
#pragma unroll
                            for (int j = 0; j < 16; ++j) se += expf(xv(j, 0) - mx) + expf(xv(j, 1) - mx);
                        }
                        se += __shfl_xor_sync(0xffffffffu, se, 1);
                        se += __shfl_xor_sync(0xffffffffu, se, 2);
                        if (row >= M) continue;
                        if ((lane & 3) == 0) he.stats[(int64_t)row * n_tiles + n_tile] = make_float2(mx, se);
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int n = col0 + 8 * j + e, bit = 8 * (j & 3) + 2 * (lane & 3) + e;
                                if ((kFull || n < N) && (n_tile == 0 || ((w[j >> 2] >> bit) & 1u) || n == he.eos || n == he.pad)) Cs[(int64_t)row * ldc + n] = xv(j, e);
                            }
                        }
                    }
                } else {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = row0 + 8 * h;
                        if (row >= M) continue;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int n = col0 + 8 * j;
                            float v[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) v[e] = epi_act<ACT>(acc[4 * j + 2 * h + e] * w_unscale + bq[8 * j + e]);
                            store_pair<kFull>(Cs, S, (int64_t)row * ldc + n, n, N, v[0], v[1], ov);
                        }
                    }
                }
            };
            if ((n_tile + 1) * GN <= N) epilogue(std::true_type{});
            else epilogue(std::false_type{});
            __syncwarp();
            if (lane == 0) mbar_arrive(bias_empty);                        // this warp has read the bias slice
            if (ov) atomicExch(overflow, 1);
            unit_trace(tr, ui, 3);
            if (first && t == 0 && wg == 1) gemm_trace(5);
            first = false;
        }
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();                                        // no CTA leaves while the peer may still signal it
    if (threadIdx.x == 0) gemm_trace(6);
}

// Finishes a split-K GEMM: out = act((sum_s part[s]) * w_unscale + bias), slices summed in index order
// (deterministic), written as fp32 and/or as format T's split the next GEMM consumes: T = __half (C_h1, C_h2) or
// __nv_bfloat16 (C_h1, C_h2, C_h3).
template <int ACT, typename T = __half>
__global__ void __launch_bounds__(256) gemm_splitk_finish_kernel(int64_t M, int N, int ldc, int k_slices, int64_t slice_stride,
                                                                 const float* __restrict__ part, const float* __restrict__ bias,
                                                                 float w_unscale, float* __restrict__ C, T* __restrict__ C_h1,
                                                                 T* __restrict__ C_h2, int* __restrict__ overflow, T* __restrict__ C_h3) {
    const int64_t total = M * (int64_t)(ldc / 4);
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = e / (ldc / 4);
        const int n = (int)(e % (ldc / 4)) * 4;
        if (n >= N) continue;
        const int64_t off = row * ldc + n;
        float4 acc = *reinterpret_cast<const float4*>(part + off);
        for (int sl = 1; sl < k_slices; ++sl) {
            const float4 p = *reinterpret_cast<const float4*>(part + sl * slice_stride + off);
            acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
        }
        float v[4] = {acc.x, acc.y, acc.z, acc.w};
        T* const S[3] = {C_h1, C_h2, C_h3};
        int ov = 0;
        for (int u = 0; u < 4; ++u) {
            if (n + u >= N) continue;
            float x = v[u] * w_unscale + (bias ? bias[n + u] : 0.f);
            x = epi_act<ACT>(x);
            if (C) C[off + u] = x;
            if (C_h1) store_split<T, 1>(S, off + u, {x}, ov);
        }
        if (ov) atomicExch(overflow, 1);
    }
}

}  // namespace sealb200
