// Limits and plain structs shared by the decode kernel headers and the host units of the decode library (model.cu,
// gemm.cu, forward.cu, generate.cu).  No device code: any unit may include it without compiling a kernel.  The structs
// are kernel parameters, so their layout is part of the kernels' interface.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace sealb200 {

constexpr int kHeadDim = 64;
constexpr int kMaxLen = 128;           // max_length <= 128 (SEAL: 10 body, 15 title, README.md:209-216 uses 100)
// The longest source the T5 path takes: the encoder bucket table covers distances -(kT5MaxSource-1) .. kT5MaxSource-1.
constexpr int kT5MaxSource = 1024;

constexpr int GM = 128;                              // GEMM tile rows (two consumer warpgroups of 64)
constexpr int GN = 128;                              // GEMM tile columns (wgmma N)

// Epilogue activation (template argument ACT): none, BART's exact-erf GELU, T5's ReLU (torch.relu: NaN stays NaN)
constexpr int kActNone = 0, kActGelu = 1, kActRelu = 2;

// A GEMM output that may still be in split-K form: ks > 1 -> value = (sum_s part[s * stride + off]) * unscale + bias[col],
// the slices summed in index order exactly like gemm_splitk_finish_kernel; ks <= 1 -> plain[off].  Lets the consumer of a
// small-batch GEMM (add+LN, the attention kernels) do the finish pass itself instead of a separate launch.
struct SplitSrc { const float* part = nullptr; int ks = 0; int64_t stride = 0; const float* bias = nullptr; float unscale = 1.f; };

// lm_head epilogue of a constrained-decode step (HEAD = true, 3xFP16, CL = 1, no split-K).  Per (row, n tile) it writes
// the partial log-softmax statistics (max, sum exp(x - max)) over the tile's columns n < N to stats[row * n_tiles +
// n_tile], which topk_rows_kernel combines in place of streaming the row, and it stores x only at the columns the select
// kernels read (the read set): the row's bits of `mask` ([M][mask_words]), eos and pad (topk_rows_kernel, row_bits),
// and the whole first n tile, columns 0..127 (select_merge_kernel's -inf fill-ins, see generate_enqueue).
struct HeadEpi {
    float2* stats = nullptr; const uint32_t* mask = nullptr; int mask_words = 0; int eos = -1, pad = -1;
};

// sealbart_get_stat(model, "last_paths"): one bit per kernel branch of the BART forward (include/sealdec.h), set on
// the host next to the launch it names
enum : uint32_t {
    kPathEncPacked = 1u << 0, kPathEncUnpacked = 1u << 1,
    kPathSelfQuery = 1u << 2, kPathSelfRounds3 = 1u << 3, kPathSelfRounds8 = 1u << 4, kPathSelfLong = 1u << 5,
    kPathCrossSmall = 1u << 6, kPathCrossGrouped = 1u << 7,
    kPathAddLnRow = 1u << 8, kPathAddLnWarp = 1u << 9,
    kPathSplitKDeferred = 1u << 10, kPathSplitKFinish = 1u << 11, kPathGemmFullTile = 1u << 12, kPathGemmCluster = 1u << 13,
    kPathGemmTf32 = 1u << 14, kPathQuerySlices = 1u << 15,
    kPathT5EncAttn = 1u << 16, kPathT5DecAttn = 1u << 17, kPathT5Rms = 1u << 18, kPathT5Relu = 1u << 19, kPathT5Gate = 1u << 20,
    kPathT5RmsWide = 1u << 21, kPathPreLn = 1u << 22, kPathPreLnEmbedLn = 1u << 23, kPathGemmBf16 = 1u << 24,
};

}  // namespace sealb200
