// Host-side representation of the FM-index: construction, sdsl .fmi parsing, native container.
// The logical content mirrors sdsl::csa_wt_int<> (sdsl/csa_wt.hpp:68-297) so that sections can be
// compared byte-for-byte with a reference-built index; the DEVICE layout derived from it
// (fm_device.cuh) is our own.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/sealfm.h"

namespace sealb200 {

struct HostIndex {
    uint64_t size = 0;        // n+1, BWT length incl. sentinel            (csa.size())
    uint32_t max_level = 0;   // L, wavelet tree height                     (sdsl/wt_int.hpp:189-193)
    uint64_t sigma = 0;       // distinct symbols incl. the sentinel
    // level-concatenated wavelet-tree bits, sdsl word order (bit p -> word p>>6, bit p&63),
    // ceil(size*L/64) words                                              (sdsl/wt_int.hpp:202-242)
    std::vector<uint64_t> tree;
    std::vector<uint64_t> alphabet;     // ascending symbols (comp order)   (csa_alphabet_strategy.hpp:494-534)
    std::vector<uint64_t> C;            // sigma+1 cumulative counts
    std::vector<uint64_t> sa_samples;   // SA[32*i]                         (csa_sampling_strategy.hpp:85-99)
    std::vector<uint64_t> isa_samples;  // ISA[64*i]                        (csa_sampling_strategy.hpp:626-641)
};

// All throw std::runtime_error with a message on failure.
void build_index(const uint64_t* symbols, uint64_t n, HostIndex& out);
void build_index_from_file(const std::string& path, int width_bytes, HostIndex& out);
// Same result as build_index, constructed on CUDA device `device` (fm_build.cu); n + 1 < 2^32 and 40 B x n of free device memory.
void build_index_gpu(const uint64_t* symbols, uint64_t n, int device, HostIndex& out);
// Same result for n + 1 < 2^40 with the suffix array in pinned host memory (fm_build_large.cu); symbols are
// `width_bytes` (4 or 8) wide.  Throws ApiError (SEALFM_EINVAL / SEALFM_ENOMEM / SEALFM_ECUDA).
void build_index_gpu_large(const void* symbols, uint64_t n, int width_bytes, int device, const sealfm_build_opts_t* opts,
                           HostIndex& out);
const sealfm_build_stats_t& build_gpu_large_last_stats();        // of the calling thread's last successful build
void load_index(const std::string& path, HostIndex& out);        // sdsl .fmi or native, auto-detect
void save_index_native(const HostIndex& idx, const std::string& path);
// The byte stream sdsl::store_to_file(csa_wt_int<>) writes for this index: loads in the unmodified reference.
void save_index_sdsl(const HostIndex& idx, const std::string& path);

}  // namespace sealb200
