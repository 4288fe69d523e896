// Internal (non-ABI) access to the device view of an sealfm_t for the other translation units.
#pragma once
#include "../../include/sealfm.h"
#include "fm_device.cuh"

#include <cuda_runtime.h>

#include <vector>

namespace sealb200 {
FmView sealfm_view(const sealfm_t* h);   // defined in fm_kernels.cu; throws ApiError if not on a device
// the handle's stream (created on first use); makes the handle's device current.  Throws ApiError if not on a device.
cudaStream_t sealfm_stream(const sealfm_t* h);
// document start offsets given to sealfm_set_beginnings (empty before)
const std::vector<uint64_t>& sealfm_beginnings(const sealfm_t* h);
// allowed-token bitmask rows of R SA ranges (fm_kernels.cu); `wide` = expand_scratch_bytes(L, R) of device scratch
size_t expand_scratch_bytes(uint32_t L, uint64_t R);
void launch_expand_masks(const FmView& v, cudaStream_t s, uint64_t R, const uint64_t* lo_d, const uint64_t* hi_d, uint32_t* mask_d,
                         uint32_t ld_words, uint32_t vocab, uint32_t shift, unsigned long long* wide);
}
