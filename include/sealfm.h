/* sealfm.h — C ABI of the H100-native FM-index for SEAL's constrained decoding.
 *
 * This is the drop-in boundary for the reference's native module `seal.cpp_modules.fm_index`
 * (SWIG wrapper over class FMIndex, /root/reference/seal/cpp_modules/fm_index.hpp:20-45,
 * fm_index.i:7-20).  Every entry point names the reference method it replaces.  Plain pointers
 * and sizes only; no torch / C++ types cross this line.  INTEGRATION.md shows the binding a SEAL
 * maintainer would add (seal_b200/cpp_modules/fm_index.py is that binding, via ctypes).
 *
 * Conventions
 *   - all index integers are uint64 at the ABI, as in the reference (fm_index.hpp:16-18);
 *   - every function returns 0 on success, a negative SEALFM_E* code otherwise, and never aborts
 *     the process; sealfm_last_error() returns a thread-local message for the last failure;
 *   - "symbols" are the reference's shifted ids (token + 10, seal/index.py:16); 0 is the sentinel;
 *   - construction / (de)serialisation run on the host; EVERY query runs on the GPU the handle was
 *     bound to with sealfm_to_device().  There is no CPU query path: without a CUDA device the
 *     query entry points fail with SEALFM_ENODEVICE.
 *   - a handle is immutable after construction: concurrent queries from several host threads /
 *     CUDA streams are safe.  Device state does not survive fork().
 */
#ifndef SEALFM_H
#define SEALFM_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sealfm sealfm_t;
typedef void* sealfm_stream_t;          /* a cudaStream_t; NULL = the legacy default stream */

#define SEALFM_OK          0
#define SEALFM_EINVAL     -1            /* bad argument                                        */
#define SEALFM_EIO        -2            /* file missing / truncated / not an index             */
#define SEALFM_ENOMEM     -3
#define SEALFM_ENODEVICE  -4            /* no CUDA device, or handle not bound to one          */
#define SEALFM_ECUDA      -5            /* a CUDA call failed; see sealfm_last_error()         */
#define SEALFM_ECAPACITY  -6            /* caller-provided output buffer too small             */

const char* sealfm_last_error(void);
int         sealfm_abi_version(void);

/* ---- construction / IO (host) -------------------------------------------------------------- */

/* FMIndex::initialize(const vector<u64>&)            fm_index.cpp:33-41  (construct_im)
 * symbols[0..n) must be > 0; the 0 sentinel is appended internally like sdsl::construct does. */
int sealfm_build(const uint64_t* symbols, uint64_t n, sealfm_t** out);
/* Same index as sealfm_build (identical sections, byte for byte), constructed on CUDA device `device`:
 * radix-sort prefix doubling -> BWT -> level-wise wavelet tree -> samples (replaces sdsl::construct_im's
 * qsufsort + wt_int construction, sdsl/construct.hpp:120-166, sdsl/wt_int.hpp:169-256).  n + 1 < 2^32 (32-bit
 * ranks) and ~40 bytes of free device memory per symbol (SEALFM_ENOMEM otherwise); larger texts: sealfm_build_gpu_ex
 * or sealfm_build.
 * SEALFM_ENODEVICE without a GPU. */
int sealfm_build_gpu(const uint64_t* symbols, uint64_t n, int device, sealfm_t** out);

/* Options of sealfm_build_gpu_ex; all-zero (or NULL) selects the defaults. */
typedef struct {
    uint64_t device_budget_bytes;   /* 0: free device memory minus 1 GiB                                         */
    uint64_t chunk_elems;           /* 0: window size derived from the budget; > 0 forces it (at least 16)        */
    int32_t  force_wide;            /* 1: 64-bit positions and labels even when m < 2^32                          */
    int32_t  reserved[7];           /* must be 0                                                                  */
} sealfm_build_opts_t;

/* Same index as sealfm_build (identical sections), constructed on CUDA device `device` for texts of up to 2^40 - 2
 * symbols.  symbols: n little-endian integers of `width_bytes` (4 or 8) each, all in [1, 2^32).
 * Suffix sorting is in-place prefix doubling (Larsson-Sadakane labels): the inverse suffix array lives on the device
 * (4 bytes per symbol while m = n + 1 < 2^32, else 8), the suffix array in pinned host memory (same width), and the
 * groups still unsorted stream through a device window of chunk_elems entries (~(2w + 34) bytes each, w the position
 * width, plus CUB scratch).  Groups larger than the window are split by key range in place.  Device memory per phase,
 * t = 2 bytes per symbol when every symbol is < 2^16, else 4:
 *   round 0 (sort by first symbol):  w*m + t*m + window
 *   doubling rounds:                 w*m + window
 *   BWT and samples:                 t*m + 4*m + window
 *   wavelet tree:                    12*m + m*L/8   (the BWT, its sorted copy, CUB's alternate keys; L = bits of the largest symbol)
 * Host: w*m pinned for the suffix array.  The largest phase must fit device_budget_bytes, else SEALFM_ENOMEM before any
 * large allocation; a pinned allocation that fails is SEALFM_ENOMEM too.  SEALFM_EINVAL: symbol 0, symbols >= 2^32,
 * m >= 2^40, a width other than 4 or 8, or nonzero reserved fields.  SEALFM_ENODEVICE without a GPU.
 * *out stays NULL on every failure. */
int sealfm_build_gpu_ex(const void* symbols, uint64_t n, int width_bytes, int device, const sealfm_build_opts_t* opts,
                        sealfm_t** out);

/* What the calling thread's last successful sealfm_build_gpu_ex did: window size, which paths ran, time per phase. */
typedef struct {
    uint64_t chunk_elems;           /* window size used                                                            */
    uint64_t windows;               /* windows sorted, all rounds                                                  */
    uint64_t max_windows_per_round;
    uint64_t spanning_groups;       /* groups that crossed a window edge: the window was cut at their first row    */
    uint64_t giant_groups;          /* groups larger than the window, split by key range                           */
    uint64_t key_partitions;        /* in-place two-way partitions done by those splits                            */
    uint64_t single_key_buckets;    /* key ranges larger than the window holding one key: relabelled, not sorted  */
    uint64_t device_peak_bytes;     /* largest sum of the builder's device allocations                             */
    uint64_t host_pinned_bytes;
    uint32_t wide;                  /* 1: 64-bit positions                                                         */
    uint32_t text_bytes;            /* bytes per symbol of the text on the device: 2 or 4                          */
    uint32_t rounds;                /* sorting rounds, round 0 (first symbol) included                             */
    uint32_t reserved;
    double   phase_s[4];            /* round 0 | doubling rounds | BWT and samples | wavelet tree                   */
    uint64_t round_unsorted[48];    /* rows in the unsorted ranges at the start of round r                          */
    double   round_s[48];           /* wall time of round r                                                        */
} sealfm_build_stats_t;
int sealfm_build_gpu_ex_stats(sealfm_build_stats_t* out);
/* Adopts index sections computed elsewhere -- exactly what sealfm_section() hands out of a built index: the
 * level-concatenated wavelet-tree bits of csa_wt_int<> (sdsl/wt_int.hpp:202-242; size * max_level bits in n_tree
 * words), the ascending alphabet (sigma symbols incl. the sentinel 0), the cumulative counts C (sigma + 1), SA[32 i]
 * (ceil(size/32) entries) and ISA[64 i] ((size-1)/64 + 1 entries).  size = n + 1.  No consistency check beyond sizes. */
int sealfm_from_sections(uint64_t size, uint32_t max_level, uint64_t sigma, const uint64_t* tree, uint64_t n_tree,
                         const uint64_t* alphabet, const uint64_t* C, const uint64_t* sa_samples, uint64_t n_sa,
                         const uint64_t* isa_samples, uint64_t n_isa, sealfm_t** out);
/* FMIndex::initialize_from_file(file, width)         fm_index.cpp:43-48
 * file = raw little-endian integers of `width_bytes` (1,2,4,8) each; SEAL passes 4
 * (seal/index.py:18,62,65). */
int sealfm_build_from_file(const char* path, int width_bytes, sealfm_t** out);
/* load_FMIndex(path)                                 fm_index.cpp:191-199
 * Reads either an sdsl-lite 2.1.0 `csa_wt_int<>` stream (the published SEAL .fmi files) or this
 * library's native container (written by sealfm_save); auto-detected. */
int sealfm_load(const char* path, sealfm_t** out);
/* Writes this library's flat native container (magic "SEALB2FM"); sealfm_load reads it back.
 * (The drop-in FMIndex.save uses sealfm_save_sdsl below.) */
int sealfm_save(const sealfm_t* h, const char* path);
/* FMIndex::save(path) in the REFERENCE'S OWN FORMAT: the byte stream sdsl::store_to_file(csa_wt_int<>) writes
 * (fm_index.cpp:186-189, sdsl/csa_wt.hpp:374-384), including the rank / select tables the reference's loader
 * expects -- an index built here loads in the unmodified reference's load_FMIndex. */
int sealfm_save_sdsl(const sealfm_t* h, const char* path);
void sealfm_free(sealfm_t* h);

uint64_t sealfm_size(const sealfm_t* h);       /* FMIndex::size() = n+1   fm_index.cpp:50-52 */
uint64_t sealfm_sigma(const sealfm_t* h);      /* index.wavelet_tree.sigma                    */
uint32_t sealfm_max_level(const sealfm_t* h);  /* index.wavelet_tree.max_level                */

/* Raw sections in sdsl's own encoding, for byte-level parity tests against a reference .fmi:
 * which = 0 tree bit words | 1 alphabet symbols (ascending) | 2 C (sigma+1) | 3 SA samples |
 *         4 ISA samples.   Pointer stays valid until sealfm_free. */
int sealfm_section(const sealfm_t* h, int which, const uint64_t** ptr, uint64_t* n_words);

/* ---- device residency ------------------------------------------------------------------------ */

/* Uploads the index (interleaved rank blocks, node tables, samples) to CUDA device `device`.
 * Must be called once before any query. */
int sealfm_to_device(sealfm_t* h, int device);
int sealfm_device(const sealfm_t* h);          /* bound device id or -1                          */
uint64_t sealfm_device_bytes(const sealfm_t* h);
/* Document start offsets (seal/index.py:50 `beginnings`), needed by sealfm_doc_index*. */
int sealfm_set_beginnings(sealfm_t* h, const uint64_t* beginnings, uint64_t n);

/* ---- queries, HOST pointers (H2D + kernel + D2H inside; synchronous) --------------------------- */

/* FMIndex::backward_search_step(sym, lo, hi_incl) -> {lo', hi'_incl}   fm_index.cpp:67-76, batched */
int sealfm_backward_search_step(const sealfm_t* h, uint64_t n, const uint64_t* sym,
                                const uint64_t* lo, const uint64_t* hi_incl,
                                uint64_t* out_lo, uint64_t* out_hi_incl);
/* FMIndex::backward_search_multi(query) -> {lo, hi_excl}               fm_index.cpp:55-65
 * nq queries, query i = symbols[offsets[i]..offsets[i+1]) */
int sealfm_backward_search_multi(const sealfm_t* h, uint64_t nq, const uint64_t* symbols,
                                 const uint64_t* offsets, uint64_t* out_lo, uint64_t* out_hi_excl);
/* FMIndex::distinct_count_multi(lows, highs)                           fm_index.cpp:111-131
 * (n = 1 is FMIndex::distinct_count, fm_index.cpp:91-109).  Output: range i's interleaved
 * (symbol,count) pairs, ascending symbol, at out[out_offsets[i]..out_offsets[i+1]).
 * out == NULL: only fills out_offsets (n+1 entries) so the caller can size `out`. */
int sealfm_distinct_count_multi(const sealfm_t* h, uint64_t n, const uint64_t* lows,
                                const uint64_t* highs, uint64_t* out_offsets,
                                uint64_t* out, uint64_t out_cap);
/* FMIndex::locate(row)                                                 fm_index.cpp:163-167, batched
 * row >= size() -> (uint64_t)-1 like the reference. */
int sealfm_locate(const sealfm_t* h, uint64_t n, const uint64_t* rows, uint64_t* out_pos);
/* seal/index.py:96-100 get_doc_index_from_row, batched: bisect_right(beginnings, locate(row)) - 1 */
int sealfm_doc_index_from_rows(const sealfm_t* h, uint64_t n, const uint64_t* rows,
                               uint64_t* out_doc);
/* FMIndex::extract_text(begin, end)                                    fm_index.cpp:169-184, batched
 * text i -> out[out_offsets[i]..); out_offsets[i] = sum_{j<i}(end_j - begin_j) is computed by
 * the callee and returned (n+1 entries). */
int sealfm_extract_text(const sealfm_t* h, uint64_t n, const uint64_t* begins,
                        const uint64_t* ends, uint64_t* out_offsets, uint64_t* out,
                        uint64_t out_cap);

/* ---- queries, DEVICE pointers (asynchronous on `stream`) --------------------------------------- */

/* batched LF step; all arrays device-resident u64[n] */
int sealfm_backward_search_step_d(const sealfm_t* h, sealfm_stream_t stream, uint64_t n,
                                  const uint64_t* sym_d, const uint64_t* lo_d,
                                  const uint64_t* hi_incl_d, uint64_t* out_lo_d,
                                  uint64_t* out_hi_incl_d);
/* Allowed-token bitmask for R half-open SA ranges: bit t of row r is set iff symbol t+shift
 * (t in [0,vocab)) occurs in BWT[lo[r], hi[r]).  mask_d: uint32[R][ld_words], zeroed by the callee.
 * This is the set seal/beam_search.py:107,131-135 scatters into its -inf mask. */
int sealfm_expand_mask_d(const sealfm_t* h, sealfm_stream_t stream, uint64_t R,
                         const uint64_t* lo_d, const uint64_t* hi_excl_d, uint32_t* mask_d,
                         uint32_t ld_words, uint32_t vocab, uint32_t shift);

/* Measurement aid for the roofline of the rank kernels: average device time (us) of `n_loads` independent random 32-byte
 * sector reads over a device buffer of `buffer_bytes` (the access pattern of a rank query; 8 loads in flight per thread). */
int sealfm_debug_sector_probe(uint64_t buffer_bytes, uint64_t n_loads, int iters, double* avg_us);

#ifdef __cplusplus
}
#endif
#endif /* SEALFM_H */
