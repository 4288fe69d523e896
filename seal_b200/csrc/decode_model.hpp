// Internal to the decode library's host units: the model handle (struct sealbart) with its weights and workspace, the
// GEMM's view of an activation, and the functions one unit calls in another, each declared next to the unit that
// defines it:
//   model.cu     weights and slot tables, creation, loading, finalize, options and stats, workspace
//   gemm.cu      GEMM dispatch (wgmma_gemm.cuh) and the weights' operand splits
//   forward.cu   the BART, pre-LayerNorm and T5 layer loops and the attention dispatch
//   generate.cu  the generate loop, its CUDA-graph cache, teacher-forced scoring, the index-mask processor
// Host-only: it includes no kernel header, so a kernel is only ever compiled in the unit that launches it.
#pragma once
#include "../../include/sealdec.h"
#include "common.cuh"
#include "decode_types.cuh"
#include "operand_split.cuh"

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

// Nothing below is part of the library's interface (include/sealdec.h): keep it out of the exported symbols.
#pragma GCC visibility push(hidden)

namespace sealb200 {

struct Lin {
    float* w = nullptr; float* b = nullptr; int out = 0, in = 0;
    float* w_hi = nullptr; float* w_lo = nullptr;          // TF32 split copies (gemm_mode 2)
    __half* w_h1 = nullptr; __half* w_h2 = nullptr;        // FP16 split copies of W * 2^s (gemm_mode 3)
    __nv_bfloat16* w_bf = nullptr;                         // gemm_mode 6: the only copy of W (w is null)
    float w_unscale = 1.f;                                 // 2^-s
    CUtensorMap map_hi{}, map_lo{}; bool maps_ready = false;
    CUtensorMap map2_hi{}, map2_lo{}; bool maps2_ready = false;   // 64-row boxes: one CTA's half of a cluster's W tile (gemm_mode 5)
};
struct LNp { float* g = nullptr; float* b = nullptr; };
struct EncLayerW { Lin qkv, o, fc1, fc2; LNp ln_attn, ln_final; };
struct DecLayerW { Lin qkv, o, cq, ckv, co, fc1, fc2; LNp ln_self, ln_cross, ln_final; };

// Every (re)allocation of a workspace buffer bumps this; a captured CUDA graph bakes buffer addresses in, so
// graphs captured under an older epoch are discarded.
extern uint64_t g_ws_epoch;           // defined in model.cu: one counter for the Bufs of every unit

// A device buffer that owns its memory: freed when the Buf goes out of scope.
struct Buf {
    void* p = nullptr; size_t bytes = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    void ensure(size_t need) {
        if (need <= bytes) return;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        CUDA_CHECK(cudaMalloc(&p, need));
        bytes = need;
        ++g_ws_epoch;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

}  // namespace sealb200

using namespace sealb200;

struct sealbart {
    sealbart_config_t cfg{};          // a T5 handle fills it from its sealt5_config_t (max_positions = kT5MaxSource)
    // architecture: 0 BART (sealbart_create), 1 T5 (sealt5_create).  For T5 the Lin biases stay zero, LNp::g holds the
    // T5LayerNorm weights (EncLayerW: ln_attn = layer.0, ln_final = layer.1; DecLayerW: ln_self / ln_cross / ln_final =
    // layer.0 / 1 / 2), enc_ln_emb / dec_ln_emb the final_layer_norm of each stack, and fc1 is wi or [wi_0; wi_1].
    // 2 pre-LayerNorm BART family (sealbart_create with a variant): BART's keys and biases; enc_ln_emb / dec_ln_emb hold
    // layernorm_embedding (allocated only if variant.layernorm_embedding), enc_ln_out / dec_ln_out the stacks' final
    // layer_norm; the position tables have max_positions + variant.position_offset rows.
    int arch = 0;
    sealbart_variant_t variant{};
    LNp enc_ln_out, dec_ln_out;
    sealt5_config_t t5{};
    float* t5_rel_enc = nullptr; float* t5_rel_dec = nullptr;          // layer-0 relative_attention_bias [buckets][heads]
    int32_t* t5_bkt_enc = nullptr; int32_t* t5_bkt_dec = nullptr;      // bucket of distance k - q, see t5_bucket_tables
    int device = 0;
    float* shared = nullptr; float* enc_pos = nullptr; float* dec_pos = nullptr;
    float* lm_head = nullptr; float* final_bias = nullptr;
    bool lm_head_given = false;
    // gemm_mode 6: the token-embedding / tied lm_head table and an untied lm_head in bf16 (shared / lm_head stay null)
    __nv_bfloat16* shared_bf = nullptr; __nv_bfloat16* lm_head_bf = nullptr;
    LNp enc_ln_emb, dec_ln_emb;
    Lin head;
    std::vector<EncLayerW> enc;
    std::vector<DecLayerW> dec;
    struct Slot { void* dst; uint64_t numel; bool bf16 = false; };     // bf16: rounded (RNE) into a bf16 matrix (gemm_mode 6)
    std::map<std::string, Slot> slots;
    std::set<std::string> loaded;
    std::vector<void*> allocs;
    uint64_t weight_bytes = 0;
    bool finalized = false;
    // workspace
    Buf enc_tok, enc_mask, ex, eqkv, etmp, ckv, src_off;
    bool enc_packed = false;          // the last encoder_forward ran on the real tokens only (src_off valid)
    Buf dx, dqkv, dtmp, dcq, logits, kc, vc;
    Buf ex_split, eattn_split, effn_split, dx_split, dattn_split, dffn_split;   // activation splits (split_view)
    Buf st_scores, st_tokens, st_lo, st_hi, st_pw, st_anc, st_mask;
    Buf st_rowmax, st_rowls, st_rule, st_cval, st_cidx, st_ccnt, st_wide;     // scratch between the kernels of a step
    Buf st_hstat;                     // [R][V / 128] lm_head tile statistics (HeadEpi)
    Buf st_thr;                       // [R][3] top-k warp statistics of each logits row (topk_threshold_kernel)
    Buf hy_score, hy_len, hy_tok, hy_valid, hy_lo, hy_hi, err, dbg_ids, a_split, splitk;
    std::vector<void*> split_allocs;
    int64_t launches = 0;
    uint32_t last_paths = 0;          // OR of the kPath* bits of every kernel branch the last model call took
    int* ovf = nullptr;              // where the producers raise "fp16 range exceeded" (set by every entry point)
    double phase_us[5] = {0, 0, 0, 0, 0};
    bool profile_gemm = false;
    int fused_head = -1;              // -1 $SEALB200_FUSED_HEAD (default on), 0 dense lm_head logits, 1 statistics epilogue
    bool poison_logits = false;
    int fused_head_steps = 0;         // steps of the last enqueued generate whose lm_head used the statistics epilogue       // testing: the logits buffer is filled with NaN before every statistics-epilogue head
    int topk_cluster_steps = 0;       // steps of the last generate whose top-k threshold ran topk_threshold_cluster_kernel
    int gemm_band = -1;               // sealdec_debug_gemm_ex: -1 tile order chosen by gemm_impl, 0 no bands, > 0 band size
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> gemm_events;
    double gemm_flops = 0;
    std::vector<cudaEvent_t> events;
    // host-buffer entry point: persistent device staging of the inputs (stable addresses -> CUDA graph reuse)
    Buf in_ids, in_mask, in_occ;
    // CUDA graphs of whole generate calls (small batches are launch-latency-bound: ~1 900 kernels per generate)
    struct GraphEntry { std::vector<uint8_t> key; uint64_t epoch = 0; cudaGraphExec_t exec = nullptr; int64_t launches = 0; uint32_t paths = 0; uint64_t stamp = 0;
                        int topk_cluster_steps = 0; };
    std::vector<GraphEntry> graphs;
    std::vector<std::vector<uint8_t>> seen_keys;     // shapes run once already (their buffers are sized): capture next time
    uint64_t graph_stamp = 0;
    int graph_policy = -1;            // -1 auto (small batches), 0 never, 1 whenever possible
    int last_used_graph = 0;
    bool tf32_ready = false;          // 3xTF32 weight splits exist (gemm_mode 2 fallback after an fp16 range overflow)
    int64_t overflow_fallbacks = 0;
    cudaStream_t stream = nullptr;    // the host-buffer entry point's own (non-blocking) stream
    // query slices (generate_enqueue): the second slice runs on slice_stream, forked from and joined back into the
    // caller's stream with two events, and has GEMM / mask-expansion scratch of its own
    int query_slices = -1;            // -1 $SEALB200_QUERY_SLICES (default on), 0 off, 1 on
    cudaStream_t slice_stream = nullptr;
    cudaEvent_t slice_fork = nullptr, slice_join = nullptr;
    Buf a_split1, splitk1, st_wide1;
    Buf effn2, dffn2;                 // T5 gated-gelu: [rows][2 d_ff] output of the [wi_0; wi_1] GEMM
    ~sealbart() { for (void* p : allocs) cudaFree(p); for (void* p : split_allocs) cudaFree(p); }
};

namespace sealb200 {

// sealbart_config_t::gemm_mode (include/sealdec.h)
enum GemmMode : int { kGemmTf32 = 2, kGemmFp16 = 3, kGemmFp16Cluster = 5, kGemmBf16 = 6 };
// 3xFP16 (one CTA per tile, or 2-CTA clusters): activations in fp16 halves, which an activation can overflow
inline bool is_3xfp16(int64_t mode) { return mode == kGemmFp16 || mode == kGemmFp16Cluster; }
// the modes whose lm_head may take the statistics epilogue (HeadEpi)
inline bool head_stats_mode(int mode) { return mode == kGemmFp16 || mode == kGemmBf16; }
// gemm_mode 6 stores every GEMM weight matrix (and the embedding table) once, in bf16; the other modes keep the fp32
// master and derive their splits from it at finalize
inline bool bf16_weights(const sealbart* m) { return m->cfg.gemm_mode == kGemmBf16; }

constexpr int64_t kAddLnRowMax = 2048;      // up to this many rows add+LN runs one CTA per row

// f(T()) with the element type T of gemm_mode's operand format (operand_split.cuh)
template <typename F> void with_format(int mode, F&& f) {
    if (mode == kGemmBf16) f(__nv_bfloat16());
    else if (is_3xfp16(mode)) f(__half());
    else f(0.f);
}

// An activation tensor as the GEMMs see it: plain fp32 x and/or its split in the gemm_mode's format T (with_format):
// p[i] is piece i, an array of T, for i < kPieces<T>; p[0] == nullptr: no split.
struct Act {
    float* x = nullptr; void* p[3] = {};
    template <typename T> T* piece(int i) const { return static_cast<T*>(p[i]); }
};

// Every split buffer holds 8 bytes per element, whatever the format: with cap = b.bytes / 8 elements, piece i of format
// T starts at element i * cap of T.  The view of b from element off on, with plain (if not null) as the fp32 copy.
template <typename T> Act split_view(float* plain, const Buf& b, int64_t off = 0) {
    Act a{plain ? plain + off : nullptr};
    const int64_t cap = (int64_t)(b.bytes / 8);
    for (int i = 0; i < kPieces<T>; ++i) a.p[i] = b.as<T>() + i * cap + off;
    return a;
}

// The stream and the per-call state the launches of one forward share.
// pending: a split-K GEMM whose slices are still unsummed (gemm's defer_rows) -- its consumer (add+LN on small batches,
// the attention kernels) folds the finish pass in
// head: the lm_head GEMM may use the statistics epilogue (HeadEpi); head_fused reports that it did
// slice: 1 = the second query slice of a generate, which has its own GEMM scratch (a_split1, splitk1)
struct Ctx { sealbart* m; cudaStream_t s; SplitSrc pending{}; HeadEpi head{}; bool head_fused = false; int slice = 0; };

struct Dims {
    int64_t Q, S, R; int B, T, d, f, V, ld, W;
    int64_t G = 0; const int32_t* grp_query = nullptr; const int32_t* grp_start = nullptr;   // ragged row groups (re-scoring)
    // A query slice (generate_enqueue): queries [q0, q0 + Q) of a batch of Qb queries and Rb rows.  Its rows start at
    // r0 = q0 * B in every row-indexed buffer; the KV cache keeps the batch's row stride Rb, its ancestor indices are
    // relative to r0.  Qb = Rb = 0: not a slice.
    int64_t q0 = 0, r0 = 0, Qb = 0, Rb = 0;
};

template <typename Fn> void for_each_lin(sealbart* m, Fn&& fn) {
    for (auto& L : m->enc) { fn(L.qkv); fn(L.o); fn(L.fc1); fn(L.fc2); }
    for (auto& L : m->dec) { fn(L.qkv); fn(L.o); fn(L.cq); fn(L.ckv); fn(L.co); fn(L.fc1); fn(L.fc2); }
    fn(m->head);
}

// ---- model.cu
void make_lin(sealbart* m, Lin& l, int out, int in);
// n host values times scale (a power of two: exact) into device weights: rounded into bf16 or copied as fp32
void upload(void* dst, bool bf16, const float* host, uint64_t n, float scale = 1.f);
void check_model(const sealbart* m);
// Returns the number of CUDA devices; none is an error.
int require_device();
// the workspace buffers of a call of dimensions D, grown to fit
void ensure_workspace(sealbart* m, const Dims& D);
// HF's T5Attention._relative_position_bucket for one relative position (key - query)
int32_t t5_bucket(int32_t rel, bool bidirectional, int num_buckets, int max_distance);

// ---- gemm.cu
// C = A W^T + b (+ the epilogue activation act: kActNone / kActGelu / kActRelu, decode_types.cuh) on the tensor cores:
// gemm_mode 3 / 5 = 3xFP16 (one CTA per tile / clusters of 2 sharing W), 6 = 3xBF16 (bf16 weights), 2 = 3xTF32 (fp32
// range: the fallback when an activation leaves the fp16 range).  Operands arrive pre-split from the producing kernel
// (A.p); they are split here only if the producer did not.
// defer_rows: a split-K result of at most this many rows may be left unsummed in cx.pending for the kernel that consumes
// C (plain fp32 C of a biased GEMM without activation only); 0: the GEMM finishes it itself.
void gemm(Ctx& cx, int64_t M, int N, int K, const Act& A, int lda, Lin& l, const Act& C, int ldc, int act, int64_t defer_rows = 0);
// The GEMM operands of l in m's gemm_mode, derived from its loaded weights (gemm_mode 6: the bf16 matrix as loaded).
// d_max: one device word of scratch for 3xFP16, whose weight split reports into m->err.
void derive_lin(sealbart* m, Lin& l, unsigned int* d_max);
// 3xTF32 operand copies of every weight matrix (gemm_mode 2; also the range-safe fallback of the 3xFP16 modes)
void ensure_tf32_splits(sealbart* m);
void check_gemm_mode(int mode);

// ---- forward.cu
// the encoder pass of Q sources and the cross-attention K / V of every decoder layer (src_tokens_hint: forward.cu)
void encoder_forward(Ctx& cx, const Dims& D, const int64_t* ids_d, const int64_t* mask_d, int64_t src_tokens_hint = -1,
                     int32_t* hint_err = nullptr);
// one decoder step for all R rows: token at position pos = cur_len-1 -> logits [R][ld]
void decoder_step(Ctx& cx, const Dims& D, const int32_t* tokens, int cur_len, const int32_t* anc, bool want_logits,
                  cudaEvent_t ev_layers_done, bool compact = false, const HeadEpi& head = HeadEpi{});

// ---- generate.cu
// discards every cached CUDA graph of m and the shapes seen once
void drop_graphs(sealbart* m);

}  // namespace sealb200

#pragma GCC visibility pop
