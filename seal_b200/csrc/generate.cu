// The constrained beam-search decode of the decode library (include/sealdec.h): the generate loop with the fused select
// step, query slices and the CUDA-graph cache, teacher-forced scoring, and the index-mask logits processor.
#include "decode_model.hpp"
#include "decode_kernels.cuh"
#include "fm_handle.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

// gs = beams per group: the first beam of every group starts at 0, the others at -1e9 (seal/beam_search.py:214-216;
// with diverse beam groups 4.13's group_beam_search sets beam_scores[:, ::gs] = 0)
__global__ void init_state_kernel(int64_t R, int gs, int T, int start_tok, int pad, uint64_t lo0, uint64_t hi0,
                                  float* __restrict__ scores, int32_t* __restrict__ tokens, uint64_t* __restrict__ lo,
                                  uint64_t* __restrict__ hi, uint64_t* __restrict__ pw, int32_t* __restrict__ anc) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= R) return;
    scores[r] = (r % gs) == 0 ? 0.f : -1e9f;
    for (int t = 0; t < T; ++t) { tokens[r * T + t] = t == 0 ? start_tok : pad; anc[r * T + t] = (int32_t)r; }
    lo[r] = lo0; hi[r] = hi0; pw[r] = hi0 - lo0;
}

__global__ void ids_to_tokens_kernel(int64_t R, int t, int T, const int64_t* __restrict__ ids, int32_t* __restrict__ tokens,
                                     int32_t* __restrict__ anc) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= R) return;
    for (int i = 0; i < T; ++i) { tokens[r * T + i] = i < t ? (int32_t)ids[r * t + i] : 0; anc[r * T + i] = (int32_t)r; }
}

Dims make_dims(const sealbart* m, int64_t Q, int64_t S, int B, int T) {
    Dims D;
    D.Q = Q; D.S = S; D.B = B; D.R = Q * B; D.T = T;
    D.d = m->cfg.d_model; D.f = m->cfg.ffn_dim; D.V = m->cfg.vocab_size;
    D.ld = (D.V + 3) / 4 * 4; D.W = (D.V + 31) / 32;
    return D;
}

cudaEvent_t new_event(sealbart* m) {
    cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); m->events.push_back(e); return e;
}

struct GenArgs {
    const sealfm_t* fm; const uint32_t* occ_d; const sealdec_params_t* p; sealdec_groups_t grp;
    const int64_t* ids_d; const int64_t* mask_d; int64_t Q, S;
    float* o_score; int32_t* o_len; int32_t* o_tok; uint8_t* o_valid; uint64_t* o_lo; uint64_t* o_hi; int32_t* err_d;
};

// Enqueues one whole generate (encoder, every decode step, records) on cx.s.  No host synchronisation unless
// src_hint == -1.  `timing` = bracket the phases with CUDA events (not possible while the stream is being captured).
bool fused_head_on(const sealbart* m) {
    static const bool env_on = [] { const char* e = std::getenv("SEALB200_FUSED_HEAD"); return !e || std::atoi(e) != 0; }();
    return m->fused_head >= 0 ? m->fused_head != 0 : env_on;
}

bool query_slices_on(const sealbart* m) {
    static const bool env_on = [] { const char* e = std::getenv("SEALB200_QUERY_SLICES"); return !e || std::atoi(e) != 0; }();
    return m->query_slices >= 0 ? m->query_slices != 0 : env_on;
}

void set_select_smem() {
    CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<512, 8192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SelSharedT<8192>)));
    CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<256, 4096>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SelSharedT<4096>)));
    CUDA_CHECK(cudaFuncSetAttribute(topk_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopkMaxVocab * 4));
    CUDA_CHECK(cudaFuncSetAttribute(topk_threshold_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTopkMaxVocab * 4));
}

// topk_threshold_cluster_kernel on `rows` rows of 1 <= V <= kTopkClusterMaxVocab values: one cluster of
// topk_cluster_ctas(V) CTAs per row (set_select_smem() first)
void launch_topk_threshold_cluster(cudaStream_t s, int64_t rows, int V, int64_t ld, const float* logits, int top_k, float* row_thr) {
    const int n = topk_cluster_ctas(V);
    if (rows * n > INT32_MAX) throw ApiError(SEALFM_EINVAL, "too many logits rows for one top-k threshold launch");
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)n; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)(rows * n)); cfg.blockDim = dim3(kTopkThreads);
    cfg.dynamicSmemBytes = (size_t)topk_cluster_chunk(V) * 4; cfg.stream = s;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, topk_threshold_cluster_kernel, V, ld, logits, top_k, row_thr));
}

// (max, log sum exp over x >= tau, tau) of `rows` logits rows of V values at stride ld into row_thr[rows][3]
// (set_select_smem() first): one CTA per row up to kTopkMaxVocab, one cluster per row above.  The generate's top-k steps
// and sealdec_debug_topk_threshold.
void launch_topk_threshold(cudaStream_t s, int64_t rows, int V, int64_t ld, const float* logits, int top_k, float* row_thr) {
    if (V > kTopkMaxVocab) { launch_topk_threshold_cluster(s, rows, V, ld, logits, top_k, row_thr); return; }
    launch_k(topk_threshold_kernel, (unsigned)rows, kTopkThreads, (size_t)V * 4, s, V, ld, logits, top_k, row_thr);
}

// One decode step's selection on Q queries: topk_threshold_kernel on a top-k step (topk_warp_step), topk_rows_kernel, then
// select_merge_kernel (set_select_smem() first).  Returns `lists`, the candidate lists per query.  The first step (cur_len 1): beams 1.. carry -1e9 and are pruned
// exactly inside one CTA per query; afterwards one CTA per row.  Diverse beam groups at the first step: lists of row 0
// (every group leader) and row 1 (every other beam) only, see select_merge_kernel.
int launch_select_step(cudaStream_t s, const FmView& view, const StepCfg& c, const StepState& st, const RowScratch& rs, int64_t Q) {
    const int B = c.num_beams, gs = B / c.num_groups;
    int lists;
    if (topk_warp_step(c))
        launch_topk_threshold(s, c.logits_shared ? Q : Q * B, c.V, c.ld, st.logits, c.top_k, rs.row_thr);
    if (c.cur_len == 1 && c.num_groups > 1) {
        lists = gs > 1 ? 2 : 1;
        launch_k(topk_rows_kernel<512, 8192>, (unsigned)(Q * lists), 512, sizeof(SelSharedT<8192>), s, c, st, rs, lists, 1);
    } else if (c.cur_len == 1) {
        lists = 1;
        launch_k(topk_rows_kernel<512, 8192>, (unsigned)Q, 512, sizeof(SelSharedT<8192>), s, c, st, rs, 1, B);
    } else {
        lists = B;
        launch_k(topk_rows_kernel<256, 4096>, (unsigned)(Q * B), 256, sizeof(SelSharedT<4096>), s, c, st, rs, B, 1);
    }
    launch_k(select_merge_kernel, (unsigned)Q, kMergeThreads, 0, s, view, c, st, rs, lists);
    return lists;
}

// The StepCfg fields every step of a generate shares: the parameters, the groups and the vocabulary size V.  The
// per-step fields are set by set_step; hyp_base and head_tiles by the caller.
StepCfg step_cfg(const sealdec_params_t* p, const sealdec_groups_t& grp, int V) {
    StepCfg c{};
    c.num_beams = p->num_beams; c.K = 2 * p->num_beams; c.V = V; c.ld = (V + 3) / 4 * 4;
    c.min_length = p->min_length; c.max_length = p->max_length;
    c.eos_token_id = p->eos_token_id; c.pad_token_id = p->pad_token_id; c.model_eos_token_id = p->model_eos_token_id;
    c.forced_eos_token_id = p->forced_eos_token_id; c.forced_bos_token_id = p->forced_bos_token_id;
    c.stop_at_count = p->stop_at_count; c.always_allow_eos = p->always_allow_eos; c.disable_fm_index = p->disable_fm_index;
    c.remove_invalid_values = p->remove_invalid_values; c.shift = p->shift; c.T = p->max_length; c.mask_words = (V + 31) / 32;
    c.hyps_per_query = sealdec_hyps_per_query(p);
    c.num_groups = grp.num_beam_groups; c.diversity_penalty = grp.diversity_penalty;
    c.top_k = p->top_k < V ? p->top_k : 0;                 // top_k >= V keeps every logit: the top_k = 0 path
    return c;
}

// The fields of step cur_len: whether every row reads the occurring mask (the first step after a forced BOS, or the
// first), whether the next step's masks are expanded, and how the logits were produced (logits_shared: one row per
// query, the compact first step; logits_ignored: the forced-EOS step, on which the model did not run).
void set_step(StepCfg& c, int cur_len, bool logits_shared, bool logits_ignored) {
    const int eff_len = cur_len - (c.forced_bos_token_id >= 0 ? 1 : 0);
    c.cur_len = cur_len;
    c.first_step_shared_mask = (!c.disable_fm_index && eff_len == 1) ? 1 : 0;
    c.expand_next = (cur_len + 1 < c.T) ? 1 : 0;
    c.logits_shared = logits_shared ? 1 : 0;
    c.logits_ignored = logits_ignored ? 1 : 0;
}

void generate_enqueue(Ctx& cx, const Dims& D, const GenArgs& a, const FmView& view, uint64_t lo0, uint64_t hi0,
                      int64_t src_hint, bool timing) {
    sealbart* m = cx.m;
    const sealdec_params_t* p = a.p;
    const int B = D.B, K = 2 * B, T = D.T;
    const int64_t Q = D.Q, R = D.R;
    for (auto e : m->events) cudaEventDestroy(e);
    m->events.clear();
    auto mark = [&]() -> cudaEvent_t {
        if (!timing) return nullptr;
        cudaEvent_t e = new_event(m);
        CUDA_CHECK(cudaEventRecord(e, cx.s));
        return e;
    };
    CUDA_CHECK(cudaMemsetAsync(a.err_d, 0, 16, cx.s));
    m->fused_head_steps = 0;
    m->topk_cluster_steps = 0;
    mark();
    encoder_forward(cx, D, a.ids_d, a.mask_d, src_hint, a.err_d + 2);
    mark();

    float* sc[2] = {m->st_scores.as<float>(), m->st_scores.as<float>() + R};
    int32_t* tk[2] = {m->st_tokens.as<int32_t>(), m->st_tokens.as<int32_t>() + R * T};
    uint64_t* lo[2] = {m->st_lo.as<uint64_t>(), m->st_lo.as<uint64_t>() + R};
    uint64_t* hi[2] = {m->st_hi.as<uint64_t>(), m->st_hi.as<uint64_t>() + R};
    uint64_t* pw[2] = {m->st_pw.as<uint64_t>(), m->st_pw.as<uint64_t>() + R};
    int32_t* an[2] = {m->st_anc.as<int32_t>(), m->st_anc.as<int32_t>() + R * T};
    uint32_t* mk[2] = {m->st_mask.as<uint32_t>(), m->st_mask.as<uint32_t>() + (size_t)R * D.W};
    const int G = a.grp.num_beam_groups, gs = B / G;
    init_state_kernel<<<(unsigned)((R + 255) / 256), 256, 0, cx.s>>>(R, gs, T, p->decoder_start_token_id, p->pad_token_id,
                                                                    lo0, hi0, sc[0], tk[0], lo[0], hi[0], pw[0], an[0]);
    CUDA_CHECK(cudaGetLastError()); m->launches++;

    const StepCfg c = step_cfg(p, a.grp, D.V);
    set_select_smem();
    // Query slices.  The rows of a decode step are independent, so after the first step (compact: one row per query,
    // run on the whole batch) queries [0, Q0) and [Q0, Q), Q0 = ceil(Q / 2), run the rest of the decode -- decoder
    // layers, lm_head, selection, mask expansion -- on two streams: the caller's and m->slice_stream.  One
    // slice's attention and add+LN kernels then run beside the other slice's GEMM CTAs (wgmma_gemm_x3_kernel leaves
    // registers and shared memory on the SM for them), and each slice's last GEMM wave is filled by the other's work.
    // A kernel computes every row the same way on a slice as on the whole batch once a slice has more than kAddLnRowMax
    // rows (add+LN takes the warp-per-row kernel either way) and no GEMM of a slice is skinny enough for split-K (more
    // than sm_count / 2 tiles at the narrowest N; bart-large from 2 049 rows on): the lm_head's banded tile order only
    // reorders independent tiles -- the records are bit-identical with slicing on or off.  Off while profile_gemm
    // brackets every GEMM with events: overlapping GEMMs would make their summed durations meaningless.
    const int64_t Q0 = (Q + 1) / 2, R1 = (Q - Q0) * B;       // R1: rows of the smaller slice
    const int64_t min_tiles = (R1 + GM - 1) / GM * ((std::min(D.d, D.V) + GN - 1) / GN);
    const bool sliced = query_slices_on(m) && !m->profile_gemm && R1 > kAddLnRowMax && 2 * min_tiles > sm_count();
    auto slice_dims = [&](int64_t q0, int64_t nq) {
        Dims S = D;
        S.Q = nq; S.R = nq * B; S.q0 = q0; S.r0 = q0 * B; S.Qb = D.Q; S.Rb = D.R;
        return S;
    };
    const int H = (int)c.hyps_per_query, head_tiles = (D.V + GN - 1) / GN;
    static const bool compact_first = [] { const char* e = std::getenv("SEALB200_COMPACT_FIRST"); return !e || std::atoi(e) != 0; }();
    static const bool skip_dead = [] { const char* e = std::getenv("SEALB200_SKIP_DEAD_STEP"); return !e || std::atoi(e) != 0; }();
    auto is_dead = [&](int cur_len) {
        // Dead step: when ForcedEOSTokenLogitsProcessor fires (cur_len == max_length - 1, HF semantics restated
        // in apply_processors) it overwrites EVERY processed score with a constant, so neither the recorded
        // hypotheses nor the (already final) beams depend on the model output of this step -- the reference
        // computes it and discards it.  Nothing later reads this position's k / v either.
        const bool forced_all = p->forced_eos_token_id >= 0 && cur_len == p->max_length - 1 && cur_len + 1 == T &&
                                !(p->forced_bos_token_id >= 0 && cur_len == 1);
        return skip_dead && forced_all;
    };
    // The model forward of step `step` on the rows of PD (the whole batch or a slice); `timed` parts record the phase
    // events (sealdec_last_phase_us).  Returns whether the lm_head took the statistics epilogue.
    auto model_part = [&](Ctx& pc, const Dims& PD, int step, bool timed) {
        const int cur = step & 1, cur_len = step + 1;
        const bool compact = compact_first && cur_len == 1;
        const bool dead = is_dead(cur_len);
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
        cudaEvent_t b = (timing && timed) ? new_event(m) : nullptr;
        // Statistics epilogue of the lm_head (HeadEpi): the select kernels then read this step's logits only at the
        // row's read set.  topk_rows_kernel reads lp[v] for v in row_bits() and select_merge_kernel (G > 1) for the
        // candidates it re-scores.  With the FM index on, past the first (shared-mask) step and with one group,
        // row_bits() is the row's mask_in bits, or eos (rule 1), or pad (rule 2), plus eos with always_allow_eos --
        // within mask bits + {eos, pad}; apply_processors only overwrites values.  select_merge_kernel's -inf fill-ins
        // (fewer than K = 2B finite candidates, want < K) read the unconstrained score of the lowest flat indices of the
        // query that are not finite candidates: fewer than K + want < 2K <= 128 flat indices from the query's first
        // row, i.e. columns 0..127 of that row (V >= 128) -- the first n tile, which HeadEpi stores in full for every
        // row.  Every other case stays dense:
        // the compact first step, disable_fm_index, forced BOS (eff_len 1 reads the occurring mask), G > 1, the top-k
        // warp (its threshold needs every logit of the row), the other GEMM modes.
        const int eff_len = cur_len - (p->forced_bos_token_id >= 0 ? 1 : 0);
        HeadEpi he{};
        if (fused_head_on(m) && !dead && !compact && !p->disable_fm_index && eff_len > 1 && G == 1 && c.top_k == 0 &&
            head_stats_mode(m->cfg.gemm_mode)) {
            he = HeadEpi{m->st_hstat.as<float2>() + PD.r0 * head_tiles, mk[cur] + PD.r0 * D.W, (int)D.W, p->eos_token_id, p->pad_token_id};
            if (m->poison_logits) CUDA_CHECK(cudaMemsetAsync(m->logits.as<float>() + PD.r0 * D.ld, 0xFF, (size_t)PD.R * D.ld * 4, pc.s));
        }
        pc.head_fused = false;
        if (!dead) decoder_step(pc, PD, tk[cur] + PD.r0 * T, cur_len, an[cur] + PD.r0 * T, true, b, compact, he);
        else if (b) CUDA_CHECK(cudaEventRecord(b, pc.s));
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
        if (timed) m->fused_head_steps += pc.head_fused ? 1 : 0;
        return pc.head_fused;
    };
    // A StepState holding only where the hypothesis records of queries q0.. go (each step's and the final beams')
    auto records = [&](int64_t q0) {
        StepState st{};
        st.hyp_score = a.o_score + q0 * H; st.hyp_len = a.o_len + q0 * H; st.hyp_tokens = a.o_tok + q0 * H * T;
        st.hyp_valid = a.o_valid + q0 * H; st.hyp_lo = a.o_lo ? a.o_lo + q0 * H : nullptr; st.hyp_hi = a.o_hi ? a.o_hi + q0 * H : nullptr;
        return st;
    };
    // The selection of step `step` on the rows of PD, from the logits model_part left (head_fused: statistics epilogue).
    auto select_part = [&](Ctx& pc, const Dims& PD, unsigned long long* wide, int step, bool head_fused, bool timed) {
        const int cur = step & 1, cur_len = step + 1;
        const bool compact = compact_first && cur_len == 1;
        const bool dead = is_dead(cur_len);
        const int64_t r0 = PD.r0, q0 = PD.q0;
        StepCfg cs = c;
        set_step(cs, cur_len, compact && !dead, dead);
        cs.head_tiles = head_fused ? head_tiles : 0;
        cs.hyp_base = step * K;
        StepState st = records(q0);
        st.beam_scores_in = sc[cur] + r0; st.beam_scores_out = sc[cur ^ 1] + r0;
        st.tokens_in = tk[cur] + r0 * T; st.tokens_out = tk[cur ^ 1] + r0 * T;
        st.lo_in = lo[cur] + r0; st.lo_out = lo[cur ^ 1] + r0; st.hi_in = hi[cur] + r0; st.hi_out = hi[cur ^ 1] + r0;
        st.pw_in = pw[cur] + r0; st.pw_out = pw[cur ^ 1] + r0;
        st.anc_in = an[cur] + r0 * T; st.anc_out = an[cur ^ 1] + r0 * T;
        st.mask_in = mk[cur] + r0 * D.W; st.mask_out = mk[cur ^ 1] + r0 * D.W;
        // the compact first step wrote one logits row per query (of the whole batch)
        st.occurring_mask = a.occ_d; st.logits = m->logits.as<float>() + (cs.logits_shared ? q0 : r0) * D.ld;
        st.head_stats = m->st_hstat.as<float2>() + r0 * head_tiles;
        st.error_flag = a.err_d;
        const RowScratch rs{m->st_rowmax.as<float>() + r0, m->st_rowls.as<float>() + r0, m->st_rule.as<uint8_t>() + r0,
                            m->st_cval.as<float>() + r0 * K, m->st_cidx.as<int32_t>() + r0 * K, m->st_ccnt.as<int32_t>() + r0,
                            m->st_thr.as<float>() + (cs.logits_shared ? q0 : r0) * 3};
        launch_select_step(pc.s, view, cs, st, rs, PD.Q);
        m->launches += topk_warp_step(cs) ? 3 : 2;
        if (timed && topk_warp_step(cs) && cs.V > kTopkMaxVocab) m->topk_cluster_steps++;
        if (cs.expand_next && !p->disable_fm_index) {          // successor sets of the new beams -> next step's masks (:107)
            launch_expand_masks(view, pc.s, (uint64_t)PD.R, lo[cur ^ 1] + r0, hi[cur ^ 1] + r0, mk[cur ^ 1] + r0 * D.W, (uint32_t)D.W,
                                (uint32_t)D.V, (uint32_t)p->shift, wide);
            m->launches += 2;
        }
        if (timing && timed) CUDA_CHECK(cudaEventRecord(new_event(m), pc.s));
    };
    auto finalize_part = [&](Ctx& pc, const Dims& PD) {
        const int cur = (T - 1) & 1;
        const int64_t r0 = PD.r0;
        StepCfg cs = c;
        set_step(cs, T, false, false);
        cs.hyp_base = (T - 1) * K;
        finalize_kernel<<<(unsigned)((PD.R + 255) / 256), 256, 0, pc.s>>>(PD.Q, cs, sc[cur] + r0, tk[cur] + r0 * T, lo[cur] + r0, hi[cur] + r0,
                                                                         records(PD.q0));
        CUDA_CHECK(cudaGetLastError()); m->launches++;
    };
    if (!sliced) {
        for (int step = 0; step + 1 < T; ++step) {
            const bool fused = model_part(cx, D, step, true);
            select_part(cx, D, m->st_wide.as<unsigned long long>(), step, fused, true);
        }
        finalize_part(cx, D);
    } else {
        // slice 0 on the caller's stream (it records the per-step phase events), slice 1 on slice_stream; the steps of
        // the two are enqueued alternately so that both streams always have work queued
        m->last_paths |= kPathQuerySlices;
        const Dims PD[2] = {slice_dims(0, Q0), slice_dims(Q0, Q - Q0)};
        unsigned long long* wide[2] = {m->st_wide.as<unsigned long long>(), m->st_wide1.as<unsigned long long>()};
        // The first step selects per slice, so that every ancestor index is slice-relative from the start, but both
        // slices do so before the fork: the compact step's logits rows (one per query of the whole batch) lie inside
        // slice 0's rows, which its next lm_head overwrites.
        const bool fused0 = model_part(cx, D, 0, true);
        for (int i = 0; i < 2; ++i) select_part(cx, PD[i], wide[i], 0, fused0, i == 0);
        CUDA_CHECK(cudaEventRecord(m->slice_fork, cx.s));
        CUDA_CHECK(cudaStreamWaitEvent(m->slice_stream, m->slice_fork, 0));
        Ctx pcx[2] = {Ctx{m, cx.s}, Ctx{m, m->slice_stream}};
        pcx[1].slice = 1;
        for (int step = 1; step + 1 < T; ++step)
            for (int i = 0; i < 2; ++i) {
                const bool fused = model_part(pcx[i], PD[i], step, i == 0);
                select_part(pcx[i], PD[i], wide[i], step, fused, i == 0);
            }
        for (int i = 0; i < 2; ++i) finalize_part(pcx[i], PD[i]);
        CUDA_CHECK(cudaEventRecord(m->slice_join, m->slice_stream));
        CUDA_CHECK(cudaStreamWaitEvent(cx.s, m->slice_join, 0));
    }
    mark();
    // events in creation order: ev0, ev_enc, then per step a, b, c, d, then end (sealdec_last_phase_us); with query
    // slices a..d of every step after the first come from slice 0
}

template <typename T> void key_put(std::vector<uint8_t>& k, const T& v) {
    const uint8_t* b = reinterpret_cast<const uint8_t*>(&v);
    k.insert(k.end(), b, b + sizeof(T));
}

// NULL = one group.  1 <= G <= num_beams, num_beams % G == 0 (BeamSearchScorerWithMemory, seal/beam_search.py:597-601);
// the penalty only exists with G > 1 and > 0 (seal/beam_search.py:447-454), it is 0 otherwise.
sealdec_groups_t checked_groups(const sealdec_groups_t* g, int num_beams) {
    sealdec_groups_t r{1, 0.f};
    if (!g) return r;
    if (g->num_beam_groups < 1 || g->num_beam_groups > num_beams || num_beams % g->num_beam_groups != 0)
        throw ApiError(SEALFM_EINVAL, "num_beam_groups must divide num_beams and be in [1, num_beams]");
    if (!std::isfinite(g->diversity_penalty)) throw ApiError(SEALFM_EINVAL, "diversity_penalty must be finite");
    r.num_beam_groups = g->num_beam_groups;
    if (r.num_beam_groups > 1 && g->diversity_penalty > 0.f) r.diversity_penalty = g->diversity_penalty;
    return r;
}

// top_k: 0 = off, > 0 TopKLogitsWarper(top_k) on every step's logits -- only on the single-group path (group_beam_search
// has no warper, seal/beam_search.py:523-532) and for rows that fit the shared memory of one cluster of
// topk_threshold_cluster_kernel.
void check_top_k(int32_t top_k, const sealdec_groups_t& grp, int V) {
    if (top_k < 0) throw ApiError(SEALFM_EINVAL, "top_k must be >= 0 (0 = off)");
    if (top_k > 0 && grp.num_beam_groups > 1) throw ApiError(SEALFM_EINVAL, "top_k > 0 needs num_beam_groups == 1");
    if (top_k > 0 && V > kTopkClusterMaxVocab)
        throw ApiError(SEALFM_EINVAL, "top_k > 0 needs vocab_size <= " + std::to_string(kTopkClusterMaxVocab));
}

// A source whose attention mask is all zero has nothing to attend to: the softmax denominator of the encoder and
// cross-attention kernels stays zero (HF instead spreads the weight over the masked keys and gives finite logits).
// SEAL never builds one; the host-buffer
// entry points reject it, the device-buffer ones document it as a precondition.  The same holds for token ids
// outside [0, V): the embedding kernels index the table with them unchecked (the reference raises IndexError).
void check_token_ids(const int64_t* ids, int64_t n, int V, const char* what) {
    for (int64_t i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= V)
            throw ApiError(SEALFM_EINVAL, std::string(what) + " token id " + std::to_string(ids[i]) + " outside [0, vocab_size)");
}

void check_sources(const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, int V) {
    for (int64_t q = 0; q < Q; ++q) {
        bool any = false;
        for (int64_t s2 = 0; s2 < S && !any; ++s2) any = mask[q * S + s2] != 0;
        if (!any) throw ApiError(SEALFM_EINVAL, "source " + std::to_string(q) + " has an all-zero attention mask");
    }
    check_token_ids(ids, Q * S, V, "source");
}

// The number of real tokens of host masks [Q][S] whose every row is right-padded ("ones then zeros"), else -1
int64_t right_padded_tokens(const int64_t* mask, int64_t Q, int64_t S) {
    int64_t n = 0;
    for (int64_t q = 0; q < Q; ++q) {
        int64_t len = 0;
        for (int64_t s2 = 0; s2 < S; ++s2) { const bool on = mask[q * S + s2] != 0; if (on && s2 != len) return -1; len += on; }
        n += len;
    }
    return n;
}

// out[r * out_stride] = log_softmax(logits[r] / temperature)[targets[r * tgt_stride]] (0 for a target outside
// [0, V)) and / or the whole row into full[r * full_ld ..]: sealdec_teacher_forced and sealdec_debug_target_logprob
void launch_target_logprob(cudaStream_t s, int64_t R, int V, int64_t ld, const float* logits, const int64_t* targets,
                           int64_t tgt_stride, float temperature, float* out, int64_t out_stride, float* full,
                           int64_t full_ld) {
    target_logprob_kernel<<<(unsigned)R, 256, 0, s>>>(R, V, ld, logits, targets, tgt_stride, temperature, out, out_stride,
                                                      full, full_ld);
    CUDA_CHECK(cudaGetLastError());
}

}  // namespace

namespace sealb200 {

void drop_graphs(sealbart* m) {
    for (auto& g : m->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    m->graphs.clear();
    m->seen_keys.clear();
}

}  // namespace sealb200

extern "C" {

int64_t sealdec_hyps_per_query(const sealdec_params_t* p) {
    if (!p) return 0;
    return (int64_t)(p->max_length - 1) * 2 * p->num_beams + p->num_beams;
}

int sealdec_generate_dx(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_d, const sealdec_params_t* p,
                        const int64_t* ids_d, const int64_t* mask_d, int64_t Q, int64_t S, sealfm_stream_t stream,
                        float* o_score, int32_t* o_len, int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo,
                        uint64_t* o_hi, int32_t* err_d, int64_t src_tokens_hint, const sealdec_groups_t* groups) {
    return guarded([&] {
        check_model(m);
        if (!p || !ids_d || !mask_d || !o_score || !o_len || !o_tok || !o_valid || !err_d) throw ApiError(SEALFM_EINVAL, "null argument");
        const int B = p->num_beams, K = 2 * B, T = p->max_length;
        if (B < 1 || B > kSelMaxBeams || K > kSelMaxK) throw ApiError(SEALFM_EINVAL, "num_beams must be in [1,32]");
        const sealdec_groups_t grp = checked_groups(groups, B);
        check_top_k(p->top_k, grp, m->cfg.vocab_size);
        if (T < 2 || T > kMaxLen) throw ApiError(SEALFM_EINVAL, "max_length must be in [2,128]");
        if (Q <= 0 || S <= 0) throw ApiError(SEALFM_EINVAL, "empty batch");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        if (src_tokens_hint < -2 || src_tokens_hint > Q * S) throw ApiError(SEALFM_EINVAL, "bad source-token hint");
        FmView view{};
        uint64_t lo0 = 0, hi0 = 0;
        if (!p->disable_fm_index) {
            if (!fm || sealfm_device(fm) != m->device) throw ApiError(SEALFM_ENODEVICE, "FM index not bound to the model's device");
            if (!occ_d) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
            view = sealfm_view(fm);
            lo0 = 0; hi0 = view.m + 1;                               // get_range([]) = (0, size()+1)  (index.py:106-110)
            if (p->n_force_decoding_from > 0) {
                std::vector<uint64_t> q(p->n_force_decoding_from), off{0, (uint64_t)p->n_force_decoding_from};
                for (int i = 0; i < p->n_force_decoding_from; ++i) q[i] = (uint64_t)p->force_decoding_from[i] + p->shift;
                int rc = sealfm_backward_search_multi(fm, 1, q.data(), off.data(), &lo0, &hi0);
                if (rc) throw ApiError(rc, sealfm_last_error());
            }
        }
        Ctx cx{m, (cudaStream_t)stream};
        m->launches = 0;
        m->last_paths = 0;
        m->ovf = err_d + 1;
        m->last_used_graph = 0;
        const Dims D = make_dims(m, Q, S, B, T);
        ensure_workspace(m, D);
        if (!p->disable_fm_index) m->st_wide.ensure(expand_scratch_bytes(view.L, (uint64_t)D.R));   // wide-row work list + BFS frontiers
        if (query_slices_on(m)) {                              // generate_enqueue may run the batch as two query slices
            if (!m->slice_stream) CUDA_CHECK(cudaStreamCreateWithFlags(&m->slice_stream, cudaStreamNonBlocking));
            if (!m->slice_fork) CUDA_CHECK(cudaEventCreateWithFlags(&m->slice_fork, cudaEventDisableTiming));
            if (!m->slice_join) CUDA_CHECK(cudaEventCreateWithFlags(&m->slice_join, cudaEventDisableTiming));
            if (!p->disable_fm_index) m->st_wide1.ensure(expand_scratch_bytes(view.L, (uint64_t)(Q / 2) * B));
        }
        const GenArgs a{fm, occ_d, p, grp, ids_d, mask_d, Q, S, o_score, o_len, o_tok, o_valid, o_lo, o_hi, err_d};

        // ---- CUDA graph of the whole call: a batch-20 generate is ~1 900 short kernels, i.e. launch-latency-bound.
        // Shapes, parameters and buffer addresses are the key; the first call of a key runs eagerly (it sizes every
        // lazily grown buffer), the second is captured, later ones are one cudaGraphLaunch.
        static const int env_graph = [] { const char* e = std::getenv("SEALB200_GRAPH"); return e ? std::atoi(e) : -1; }();
        const int policy = m->graph_policy >= 0 ? m->graph_policy : env_graph;
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        if (cx.s) CUDA_CHECK(cudaStreamIsCapturing(cx.s, &cap));
        const bool small = D.R <= 4096;
        bool want_graph = cx.s != nullptr && cap == cudaStreamCaptureStatusNone && !m->profile_gemm &&
                          (policy == 1 || (policy < 0 && small));
        // inside a graph the encoder never needs the host: small batches compute the padded rows (the key then does
        // not depend on the batch's contents), larger ones use the caller's token count
        int64_t eff_hint = src_tokens_hint;
        if (want_graph) { if (small) eff_hint = -2; else if (src_tokens_hint == -1) want_graph = false; }
        if (!want_graph) { generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, cap == cudaStreamCaptureStatusNone); m->phase_us[0] = -1; return; }

        std::vector<uint8_t> key;
        key_put(key, Q); key_put(key, S); key_put(key, eff_hint); key_put(key, lo0); key_put(key, hi0);
        key_put(key, m->cfg.gemm_mode); key_put(key, cx.s);
        sealdec_params_t pc = *p; pc.force_decoding_from = nullptr; key_put(key, pc);
        for (int i = 0; i < p->n_force_decoding_from; ++i) key_put(key, p->force_decoding_from[i]);
        key_put(key, grp.num_beam_groups); key_put(key, grp.diversity_penalty);
        key_put(key, fused_head_on(m)); key_put(key, m->poison_logits); key_put(key, query_slices_on(m));
        key_put(key, view.blocks); key_put(key, view.csym); key_put(key, view.node_tab); key_put(key, view.m);
        key_put(key, occ_d); key_put(key, ids_d); key_put(key, mask_d); key_put(key, o_score); key_put(key, o_len);
        key_put(key, o_tok); key_put(key, o_valid); key_put(key, o_lo); key_put(key, o_hi); key_put(key, err_d);
        if (!m->graphs.empty() && m->graphs.front().epoch != g_ws_epoch) drop_graphs(m);
        for (auto& g : m->graphs)
            if (g.key == key) {
                CUDA_CHECK(cudaGraphLaunch(g.exec, cx.s));
                g.stamp = ++m->graph_stamp; m->launches = g.launches; m->last_paths = g.paths; m->last_used_graph = 1;
                m->topk_cluster_steps = g.topk_cluster_steps;
                return;
            }
        bool seen = false;
        for (auto& k2 : m->seen_keys) if (k2 == key) { seen = true; break; }
        if (!seen) {                                           // first time: eager (sizes split-K / staging buffers)
            if (m->seen_keys.size() >= 16) m->seen_keys.erase(m->seen_keys.begin());
            m->seen_keys.push_back(key);
            generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, true);
            m->phase_us[0] = -1;
            return;
        }
        const uint64_t epoch0 = g_ws_epoch;
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        bool captured = false;
        if (cudaStreamBeginCapture(cx.s, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
            try {
                generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, false);
                captured = cudaStreamEndCapture(cx.s, &graph) == cudaSuccess && graph != nullptr;
            } catch (...) {
                cudaStreamEndCapture(cx.s, &graph);
                captured = false;
            }
            if (captured && g_ws_epoch == epoch0) captured = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
            else captured = false;
            if (graph) cudaGraphDestroy(graph);
        }
        if (!captured) {
            // a buffer moved while capturing, or this driver cannot capture / instantiate the call (the launches were
            // only recorded, nothing ran): run it the ordinary way, and stop trying on this model
            cudaGetLastError();
            if (g_ws_epoch == epoch0) m->graph_policy = 0;
            m->launches = 0; m->last_paths = 0;
            generate_enqueue(cx, D, a, view, lo0, hi0, eff_hint, true);
            return;
        }
        if (m->graphs.size() >= 8) {                           // evict the least recently used
            size_t victim = 0;
            for (size_t i = 1; i < m->graphs.size(); ++i) if (m->graphs[i].stamp < m->graphs[victim].stamp) victim = i;
            cudaGraphExecDestroy(m->graphs[victim].exec);
            m->graphs.erase(m->graphs.begin() + victim);
        }
        sealbart::GraphEntry ge; ge.key = std::move(key); ge.epoch = g_ws_epoch; ge.exec = exec; ge.launches = m->launches; ge.paths = m->last_paths; ge.stamp = ++m->graph_stamp;
        ge.topk_cluster_steps = m->topk_cluster_steps;
        m->graphs.push_back(std::move(ge));
        CUDA_CHECK(cudaGraphLaunch(exec, cx.s));
        m->last_used_graph = 1;
    });
}

int sealdec_last_phase_us(const sealbart_t* mc, double out5[5]) {
    return guarded([&] {
        sealbart* m = const_cast<sealbart*>(mc);
        if (!m || !out5) throw ApiError(SEALFM_EINVAL, "null argument");
        CUDA_CHECK(cudaSetDevice(m->device));
        const size_t n = m->events.size();
        if (n < 3) throw ApiError(SEALFM_EINVAL, "no generate call recorded");
        CUDA_CHECK(cudaEventSynchronize(m->events[n - 1]));
        auto ms = [&](size_t a, size_t b) { float t = 0; CUDA_CHECK(cudaEventElapsedTime(&t, m->events[a], m->events[b])); return (double)t * 1e3; };
        double enc = ms(0, 1), layers = 0, head = 0, sel = 0;
        for (size_t i = 2; i + 3 < n; i += 4) { layers += ms(i, i + 1); head += ms(i + 1, i + 2); sel += ms(i + 2, i + 3); }
        out5[0] = enc; out5[1] = layers; out5[2] = head; out5[3] = sel; out5[4] = ms(0, n - 1);
    });
}

int sealdec_generate(sealbart_t* m, const sealfm_t* fm, const uint32_t* occ_host, const sealdec_params_t* p,
                     const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, float* o_score, int32_t* o_len,
                     int32_t* o_tok, uint8_t* o_valid, uint64_t* o_lo, uint64_t* o_hi, const sealdec_groups_t* groups) {
    return guarded([&] {
        check_model(m);
        if (!p || !ids || !mask || Q <= 0 || S <= 0) throw ApiError(SEALFM_EINVAL, "null argument / empty batch");
        checked_groups(groups, p->num_beams);
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        const int64_t H = sealdec_hyps_per_query(p), T = p->max_length;
        const int W = (m->cfg.vocab_size + 31) / 32;
        // the caller's buffers are host memory: the real-token count costs nothing to know here, so the encoder
        // never has to ask the device for it (right-padded masks only; anything else takes the padded path)
        int64_t hint = right_padded_tokens(mask, Q, S);
        if (hint <= 0) hint = -2;
        if (!m->stream) CUDA_CHECK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
        cudaStream_t s = m->stream;
        m->in_ids.ensure(Q * S * 8); m->in_mask.ensure(Q * S * 8); m->in_occ.ensure((size_t)W * 4);
        m->hy_score.ensure(Q * H * 4); m->hy_len.ensure(Q * H * 4); m->hy_tok.ensure(Q * H * T * 4);
        m->hy_valid.ensure(Q * H); m->hy_lo.ensure(Q * H * 8); m->hy_hi.ensure(Q * H * 8); m->err.ensure(16);
        CUDA_CHECK(cudaMemcpyAsync(m->in_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(m->in_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        if (occ_host) CUDA_CHECK(cudaMemcpyAsync(m->in_occ.p, occ_host, (size_t)W * 4, cudaMemcpyHostToDevice, s));
        int32_t errs[4] = {0, 0, 0, 0};
        auto run = [&] {                                       // one pass on the staged inputs
            return sealdec_generate_dx(m, fm, occ_host ? m->in_occ.as<uint32_t>() : nullptr, p, m->in_ids.as<int64_t>(),
                                       m->in_mask.as<int64_t>(), Q, S, s, m->hy_score.as<float>(), m->hy_len.as<int32_t>(),
                                       m->hy_tok.as<int32_t>(), m->hy_valid.as<uint8_t>(), o_lo ? m->hy_lo.as<uint64_t>() : nullptr,
                                       o_hi ? m->hy_hi.as<uint64_t>() : nullptr, m->err.as<int32_t>(), hint, groups);
        };
        if (const int rc = run()) throw ApiError(rc, last_error());
        CUDA_CHECK(cudaMemcpyAsync(errs, m->err.p, 16, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (errs[1] && is_3xfp16(m->cfg.gemm_mode)) {
            // An activation left the fp16 range (|x| > 65504; the producers saturate and raise the flag): this pass is
            // redone with the 3xTF32 kernels, which have fp32's range -- the caller gets exact-range results either way.
            const int mode = m->cfg.gemm_mode;
            { const int r0 = sealbart_set_option(m, "gemm_mode", kGemmTf32); if (r0) throw ApiError(r0, last_error()); }
            m->overflow_fallbacks++;
            const int rc = run();
            const int rc2 = sealbart_set_option(m, "gemm_mode", mode);
            if (rc) throw ApiError(rc, last_error());
            if (rc2) throw ApiError(rc2, last_error());
            CUDA_CHECK(cudaMemcpyAsync(errs, m->err.p, 16, cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));
        }
        CUDA_CHECK(cudaMemcpyAsync(o_score, m->hy_score.p, Q * H * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_len, m->hy_len.p, Q * H * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_tok, m->hy_tok.p, Q * H * T * 4, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaMemcpyAsync(o_valid, m->hy_valid.p, Q * H, cudaMemcpyDeviceToHost, s));
        if (o_lo) CUDA_CHECK(cudaMemcpyAsync(o_lo, m->hy_lo.p, Q * H * 8, cudaMemcpyDeviceToHost, s));
        if (o_hi) CUDA_CHECK(cudaMemcpyAsync(o_hi, m->hy_hi.p, Q * H * 8, cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        if (errs[2]) throw ApiError(SEALFM_EINVAL, "internal: source-token count mismatch");
        if (errs[0]) throw ApiError(SEALFM_EINVAL, "beam: fewer than num_beams non-EOS candidates (seal/beam_search.py:687-690)");
    });
}

int sealdec_teacher_forced(sealbart_t* m, const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S,
                           const int64_t* dec_ids, const int32_t* row_query, int64_t N, int64_t T, float temperature,
                           float* out_logprob, int64_t out_full_pos, float* out_full) {
    return guarded([&] {
        check_model(m);
        if (!ids || !mask || !dec_ids || !row_query || N <= 0 || T < 1 || T > kMaxLen || Q <= 0 || S <= 0)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        if (out_full && (out_full_pos < 0 || out_full_pos >= T)) throw ApiError(SEALFM_EINVAL, "out_full_pos must be in [0, T)");
        if (m->arch != 1 && T > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "decoder inputs longer than the position table");
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        check_token_ids(dec_ids, N * T, m->cfg.vocab_size, "decoder");
        for (int64_t r = 0; r < N; ++r) {
            if (row_query[r] < 0 || row_query[r] >= Q || (r && row_query[r] < row_query[r - 1]))
                throw ApiError(SEALFM_EINVAL, "row_query must be sorted and within [0, Q)");
        }
        const int64_t kChunk = 4096;                           // decoder rows per pass (logits: 4096 x V floats)
        Dims D = make_dims(m, Q, S, 1, (int)T);
        D.R = std::min<int64_t>(N, kChunk);
        ensure_workspace(m, D);
        m->ovf = m->err.as<int>() + 1;
        cudaStream_t s = nullptr;
        CUDA_CHECK(cudaMemsetAsync(m->ovf, 0, 4, s));          // before the encoder: its producers raise it too
        Buf d_ids, d_mask, d_dec, d_gq, d_gs, d_out, d_full;
        d_ids.ensure(Q * S * 8); d_mask.ensure(Q * S * 8);
        CUDA_CHECK(cudaMemcpyAsync(d_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(d_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        Ctx cx{m, s};
        m->launches = 0;
        m->last_paths = 0;
        encoder_forward(cx, D, d_ids.as<int64_t>(), d_mask.as<int64_t>());
        d_dec.ensure(D.R * T * 8); d_gq.ensure((D.R + 1) * 4); d_gs.ensure((D.R + 2) * 4);
        if (T > 1) d_out.ensure(D.R * (T - 1) * 4);
        if (out_full) d_full.ensure((size_t)D.R * D.V * 4);
        for (int64_t r0 = 0; r0 < N; r0 += kChunk) {
            const int64_t rows = std::min(kChunk, N - r0);
            std::vector<int32_t> gq, gs;
            for (int64_t r = 0; r < rows; ++r)
                if (r == 0 || row_query[r0 + r] != row_query[r0 + r - 1]) { gq.push_back(row_query[r0 + r]); gs.push_back((int32_t)r); }
            gs.push_back((int32_t)rows);
            CUDA_CHECK(cudaMemcpyAsync(d_dec.p, dec_ids + r0 * T, rows * T * 8, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(d_gq.p, gq.data(), gq.size() * 4, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(d_gs.p, gs.data(), gs.size() * 4, cudaMemcpyHostToDevice, s));
            Dims C = D;
            C.R = rows; C.G = (int64_t)gq.size(); C.grp_query = d_gq.as<int32_t>(); C.grp_start = d_gs.as<int32_t>();
            int32_t* tk = m->st_tokens.as<int32_t>(); int32_t* an = m->st_anc.as<int32_t>();
            ids_to_tokens_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, s>>>(rows, (int)T, (int)T, d_dec.as<int64_t>(), tk, an);
            CUDA_CHECK(cudaGetLastError());
            for (int p = 0; p < T; ++p) {
                const bool need = (p + 1 < T) || (out_full && p == out_full_pos);
                if (!need) continue;                           // the last position only feeds the full-vector output
                decoder_step(cx, C, tk, p + 1, an, true, nullptr);
                launch_target_logprob(s, rows, C.V, C.ld, m->logits.as<float>(), d_dec.as<int64_t>() + (p + 1 < T ? p + 1 : 0), T,
                                      temperature, (p + 1 < T) ? d_out.as<float>() + p : nullptr, T - 1,
                                      (out_full && p == out_full_pos) ? d_full.as<float>() : nullptr, C.V);
                m->launches++;
            }
            if (T > 1 && out_logprob)
                CUDA_CHECK(cudaMemcpyAsync(out_logprob + r0 * (T - 1), d_out.p, rows * (T - 1) * 4, cudaMemcpyDeviceToHost, s));
            if (out_full)
                CUDA_CHECK(cudaMemcpyAsync(out_full + (size_t)r0 * D.V, d_full.p, (size_t)rows * D.V * 4, cudaMemcpyDeviceToHost, s));
            CUDA_CHECK(cudaStreamSynchronize(s));              // gq/gs are stack temporaries; outputs consumed per chunk
        }
        int32_t ovf = 0;
        CUDA_CHECK(cudaMemcpy(&ovf, m->err.as<int>() + 1, 4, cudaMemcpyDeviceToHost));
        if (ovf) throw ApiError(SEALFM_EINVAL, "fp16 range exceeded in the 3xFP16 GEMM path (|x| > 65504); use gemm_mode 2 (3xTF32)");
    });
}

int sealdec_apply_index_mask_d(const sealfm_t* fm, sealfm_stream_t stream, const sealdec_processor_cfg_t* cfg,
                               const int64_t* input_ids_d, int64_t R, int64_t t, const uint32_t* occ_d,
                               const float* in_d, float* out_d, int64_t V, int64_t ld) {
    return guarded([&] {
        if (!fm || !cfg || !input_ids_d || !in_d || !out_d) throw ApiError(SEALFM_EINVAL, "null argument");
        const int dev = sealfm_device(fm);
        if (dev < 0) throw ApiError(SEALFM_ENODEVICE, "index not bound to a CUDA device (call sealfm_to_device)");
        CUDA_CHECK(cudaSetDevice(dev));
        if (R <= 0 || t < 1) throw ApiError(SEALFM_EINVAL, "empty input");
        cudaStream_t s = (cudaStream_t)stream;
        const FmView view = sealfm_view(fm);
        const int W = (int)((V + 31) / 32);
        dim3 grid((unsigned)R, (unsigned)std::min<int64_t>((V + 255) / 256, 64));
        const bool fb = cfg->forced_bos_token_id >= 0;
        if (fb && t == 1) {                                                     // :66-69
            apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, nullptr, W, 1, nullptr, cfg->eos_token_id,
                                                   cfg->pad_token_id, 0, cfg->forced_bos_token_id);
            CUDA_CHECK(cudaGetLastError());
            return;
        }
        const int skip = fb ? 1 : 0;                                            // :71
        if (t - skip == 1) {                                                    // :73-77
            if (!occ_d) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
            apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, occ_d, W, 1, nullptr, cfg->eos_token_id,
                                                   cfg->pad_token_id, cfg->always_allow_eos, -1);
            CUDA_CHECK(cudaGetLastError());
            return;
        }
        // scratch: lo, hi (u64), rule (u8), masks — stream-ordered allocation, no host sync
        uint64_t* lo = nullptr; uint64_t* hi = nullptr; uint8_t* rule = nullptr; uint32_t* masks = nullptr; uint64_t* fsyms = nullptr;
        // stream-ordered frees on EVERY exit path (an ApiError / CUDA_CHECK below must not leak the scratch)
        struct Scratch { void** p[5]; cudaStream_t s; ~Scratch() { for (void** q : p) if (*q) cudaFreeAsync(*q, s); } }
            guard{{(void**)&lo, (void**)&hi, (void**)&rule, (void**)&masks, (void**)&fsyms}, s};
        CUDA_CHECK(cudaMallocAsync(&lo, R * 8, s)); CUDA_CHECK(cudaMallocAsync(&hi, R * 8, s));
        CUDA_CHECK(cudaMallocAsync(&rule, R, s)); CUDA_CHECK(cudaMallocAsync(&masks, (size_t)R * W * 4, s));
        const int nf = cfg->n_force_decoding_from;
        if (nf > 0) {
            std::vector<uint64_t> f(nf);
            for (int i = 0; i < nf; ++i) f[i] = (uint64_t)cfg->force_decoding_from[i] + cfg->shift;
            CUDA_CHECK(cudaMallocAsync(&fsyms, nf * 8, s));
            CUDA_CHECK(cudaMemcpyAsync(fsyms, f.data(), nf * 8, cudaMemcpyHostToDevice, s));
            CUDA_CHECK(cudaStreamSynchronize(s));   // f is a stack temporary
        }
        rows_fold_kernel<<<(unsigned)((R + 127) / 128), 128, 0, s>>>(view, R, (int)t, input_ids_d, skip, cfg->eos_token_id,
                                                                    cfg->pad_token_id, cfg->stop_at_count, fsyms, nf, cfg->shift,
                                                                    lo, hi, rule);
        CUDA_CHECK(cudaGetLastError());
        int rc = sealfm_expand_mask_d(fm, s, R, lo, hi, masks, W, (uint32_t)V, (uint32_t)cfg->shift);
        if (rc) throw ApiError(rc, sealfm_last_error());
        apply_mask_kernel<<<grid, 256, 0, s>>>(R, (int)V, ld, in_d, out_d, masks, W, 0, rule, cfg->eos_token_id,
                                               cfg->pad_token_id, cfg->always_allow_eos, -1);
        CUDA_CHECK(cudaGetLastError());
    });
}

}  // extern "C"

// ---- test hooks ------------------------------------------------------------------------------------------------

namespace {

// deterministic pseudo-random logits in [-8, 8) and `per_row` allowed tokens per row
__global__ void debug_fill_rows_kernel(int64_t R, int V, int ld, int W, int per_row, float* __restrict__ logits, uint32_t* __restrict__ mask) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R * ld; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t h = (uint32_t)i * 2654435761u; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
        logits[i] = (float)(h >> 8) * (16.f / 16777216.f) - 8.f;
        if (i < R * per_row) {
            const int64_t r = i / per_row;
            const int v = (int)((uint64_t)(i % per_row + 1) * 7919u * (uint64_t)(r + 1) % (uint64_t)V);
            atomicOr(&mask[r * W + (v >> 5)], 1u << (v & 31));
        }
    }
}

// sealdec_debug_topk_threshold (cluster = false: V <= kTopkMaxVocab, the generate's dispatch) and
// sealdec_debug_topk_threshold_cluster (cluster = true: topk_threshold_cluster_kernel for V <= kTopkClusterMaxVocab)
int debug_topk_threshold(bool cluster, int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k, float* out_thr,
                         float* out_max, float* out_logsum) {
    return guarded([&] {
        if (R <= 0 || V <= 0 || ld < V || !logits || top_k < 1 || !out_thr || !out_max || !out_logsum || (uint64_t)R > INT32_MAX)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        const int max_v = cluster ? kTopkClusterMaxVocab : kTopkMaxVocab;
        if (V > max_v) throw ApiError(SEALFM_EINVAL, "V must be <= " + std::to_string(max_v));
        require_device();
        Buf d_lg, d_thr;
        d_lg.ensure((size_t)R * ld * 4); d_thr.ensure((size_t)R * 3 * 4);
        CUDA_CHECK(cudaMemcpy(d_lg.p, logits, (size_t)R * ld * 4, cudaMemcpyHostToDevice));
        CUDA_CHECK(cudaMemset(d_thr.p, 0xFF, (size_t)R * 3 * 4));
        set_select_smem();
        if (cluster) launch_topk_threshold_cluster(nullptr, R, V, ld, d_lg.as<float>(), top_k, d_thr.as<float>());
        else launch_topk_threshold(nullptr, R, V, ld, d_lg.as<float>(), top_k, d_thr.as<float>());
        CUDA_CHECK(cudaDeviceSynchronize());
        std::vector<float> h((size_t)R * 3);
        CUDA_CHECK(cudaMemcpy(h.data(), d_thr.p, h.size() * 4, cudaMemcpyDeviceToHost));
        for (int64_t r = 0; r < R; ++r) { out_max[r] = h[r * 3]; out_logsum[r] = h[r * 3 + 1]; out_thr[r] = h[r * 3 + 2]; }
    });
}

}  // namespace

extern "C" {

int sealdec_debug_step_logits(sealbart_t* m, const int64_t* ids, const int64_t* mask, int64_t Q, int64_t S, int32_t B,
                              const int64_t* dec_ids, int64_t t, const int32_t* anc, int64_t src_tokens_hint,
                              float* out_logits) {
    return guarded([&] {
        check_model(m);
        if (!ids || !mask || !dec_ids || !out_logits || t < 1 || t > kMaxLen || Q <= 0 || S <= 0 || B < 1)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        if (S > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "source longer than max_positions");
        check_sources(ids, mask, Q, S, m->cfg.vocab_size);
        // a count is only valid for right-padded masks; checked here, where the mask is host memory
        if (src_tokens_hint != -1 && src_tokens_hint != -2 && right_padded_tokens(mask, Q, S) != src_tokens_hint)
            throw ApiError(SEALFM_EINVAL, "src_tokens_hint does not match a right-padded mask");
        const int T = (int)t;
        if (m->arch != 1 && T > m->cfg.max_positions) throw ApiError(SEALFM_EINVAL, "decoder inputs longer than the position table");
        const Dims D = make_dims(m, Q, S, B, T);
        check_token_ids(dec_ids, D.R * T, m->cfg.vocab_size, "decoder");
        if (anc)
            for (int64_t i = 0; i < D.R * T; ++i)
                if (anc[i] < 0 || anc[i] >= D.R) throw ApiError(SEALFM_EINVAL, "ancestor row out of range");
        ensure_workspace(m, D);
        m->ovf = m->err.as<int>() + 1;
        Buf d_ids, d_mask;
        d_ids.ensure(Q * S * 8); d_mask.ensure(Q * S * 8); m->dbg_ids.ensure(D.R * t * 8);
        cudaStream_t s = nullptr;
        CUDA_CHECK(cudaMemcpyAsync(d_ids.p, ids, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(d_mask.p, mask, Q * S * 8, cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(m->dbg_ids.p, dec_ids, D.R * t * 8, cudaMemcpyHostToDevice, s));
        Ctx cx{m, s};
        m->launches = 0;
        m->last_paths = 0;
        encoder_forward(cx, D, d_ids.as<int64_t>(), d_mask.as<int64_t>(), src_tokens_hint);
        int32_t* tk = m->st_tokens.as<int32_t>(); int32_t* an = m->st_anc.as<int32_t>();
        ids_to_tokens_kernel<<<(unsigned)((D.R + 255) / 256), 256, 0, s>>>(D.R, T, T, m->dbg_ids.as<int64_t>(), tk, an);
        CUDA_CHECK(cudaGetLastError());
        if (anc) CUDA_CHECK(cudaMemcpyAsync(an, anc, (size_t)D.R * T * 4, cudaMemcpyHostToDevice, s));   // replaces the identity
        for (int cur_len = 1; cur_len <= T; ++cur_len) decoder_step(cx, D, tk, cur_len, an, cur_len == T, nullptr);
        CUDA_CHECK(cudaMemcpy2DAsync(out_logits, (size_t)D.V * 4, m->logits.p, (size_t)D.ld * 4, (size_t)D.V * 4, D.R,
                                     cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int sealdec_debug_select_step(const sealfm_t* fm, const sealdec_params_t* p, const sealdec_groups_t* groups, int64_t Q,
                              int32_t V, int32_t cur_len, int32_t logits_shared, int32_t logits_ignored,
                              const float* logits, const float* head_stats, const uint32_t* masks,
                              const uint32_t* occurring_mask, const float* beam_scores, const int32_t* tokens,
                              const int32_t* ancestry, const uint64_t* lo, const uint64_t* hi, const uint64_t* pw,
                              float* row_max, float* row_logsum, uint8_t* row_rule, float* cand_val, int32_t* cand_idx,
                              int32_t* cand_cnt, int32_t* lists, float* beam_scores_out, int32_t* tokens_out,
                              int32_t* ancestry_out, uint64_t* lo_out, uint64_t* hi_out, uint64_t* pw_out,
                              float* rec_score, int32_t* rec_len, int32_t* rec_tokens, uint8_t* rec_valid,
                              uint64_t* rec_lo, uint64_t* rec_hi, int32_t* error_flag) {
    return guarded([&] {
        if (!p || !beam_scores || !tokens || !ancestry || !lo || !hi || !pw || !row_max || !row_logsum || !row_rule ||
            !cand_val || !cand_idx || !cand_cnt || !lists || !beam_scores_out || !tokens_out || !ancestry_out || !lo_out ||
            !hi_out || !pw_out || !rec_score || !rec_len || !rec_tokens || !rec_valid || !rec_lo || !rec_hi || !error_flag)
            throw ApiError(SEALFM_EINVAL, "null argument");
        // only configurations a generate produces (generate_enqueue)
        const int B = p->num_beams, K = 2 * B, T = p->max_length;
        if (B < 1 || B > kSelMaxBeams || K > kSelMaxK) throw ApiError(SEALFM_EINVAL, "num_beams must be in [1,32]");
        const sealdec_groups_t grp = checked_groups(groups, B);
        if (T < 2 || T > kMaxLen) throw ApiError(SEALFM_EINVAL, "max_length must be in [2,128]");
        if (cur_len < 1 || cur_len > T - 1) throw ApiError(SEALFM_EINVAL, "cur_len must be in [1, max_length - 1]");
        if (Q <= 0 || V <= 0 || (int64_t)B * V > INT32_MAX) throw ApiError(SEALFM_EINVAL, "bad Q / V");
        if (p->eos_token_id < 0 || p->eos_token_id >= V || p->pad_token_id < 0 || p->pad_token_id >= V ||
            p->model_eos_token_id >= V || p->forced_eos_token_id >= V || p->forced_bos_token_id >= V)
            throw ApiError(SEALFM_EINVAL, "token ids must be below V");
        const bool fb_step = p->forced_bos_token_id >= 0 && cur_len == 1;
        const int eff_len = cur_len - (p->forced_bos_token_id >= 0 ? 1 : 0);
        const bool fm_on = !p->disable_fm_index;
        const bool shared_mask = fm_on && eff_len == 1;
        if (logits_ignored && !(p->forced_eos_token_id >= 0 && cur_len == T - 1 && !fb_step))
            throw ApiError(SEALFM_EINVAL, "logits_ignored: only on the forced-EOS step");
        if (logits_shared && (cur_len != 1 || logits_ignored)) throw ApiError(SEALFM_EINVAL, "logits_shared: only at cur_len 1");
        if (!logits_ignored && !logits) throw ApiError(SEALFM_EINVAL, "logits missing");
        if (head_stats && !(fm_on && eff_len > 1 && grp.num_beam_groups == 1 && V >= GN && !logits_ignored && !logits_shared))
            throw ApiError(SEALFM_EINVAL, "head statistics: only after the first step, with the FM index on, one group and V >= 128");
        check_top_k(p->top_k, grp, V);
        if (head_stats && p->top_k > 0) throw ApiError(SEALFM_EINVAL, "head statistics: not with top_k > 0 (dense logits)");
        if (fm_on && !fb_step && !shared_mask && !masks) throw ApiError(SEALFM_EINVAL, "masks missing");
        if (shared_mask && !occurring_mask) throw ApiError(SEALFM_EINVAL, "occurring mask missing");
        FmView view{};
        if (fm_on) {
            if (!fm || sealfm_device(fm) < 0) throw ApiError(SEALFM_ENODEVICE, "FM index not on a device");
            CUDA_CHECK(cudaSetDevice(sealfm_device(fm)));
            view = sealfm_view(fm);
        } else
            require_device();
        const int64_t R = Q * B;
        for (int64_t r = 0; r < R; ++r) {
            if (lo[r] > hi[r] || (fm_on && hi[r] > view.m + 1)) throw ApiError(SEALFM_EINVAL, "SA range out of the index");
            for (int i = 0; i < T; ++i)
                if (ancestry[r * T + i] < 0 || ancestry[r * T + i] >= R) throw ApiError(SEALFM_EINVAL, "ancestor row out of range");
        }
        const int ld = (V + 3) / 4 * 4, W = (V + 31) / 32, tiles = (V + GN - 1) / GN;
        const int64_t lrows = logits_shared ? Q : R;

        Buf d_lg, d_hs, d_mk, d_occ, d_sc, d_tk, d_an, d_lo, d_hi, d_pw, d_rmax, d_rls, d_rule, d_cval, d_cidx, d_ccnt, d_sco, d_tko,
            d_ano, d_loo, d_hio, d_pwo, d_hsc, d_hlen, d_htk, d_hval, d_hlo, d_hhi, d_err, d_thr;
        auto up = [&](Buf& d, const void* h, size_t bytes) {
            d.ensure(bytes);
            if (h) CUDA_CHECK(cudaMemcpy(d.p, h, bytes, cudaMemcpyHostToDevice));
            else CUDA_CHECK(cudaMemset(d.p, 0, bytes));
        };
        // outputs and scratch start as NaN / all-ones bits: a value read before it is written, or never written, shows
        auto poisoned = [&](Buf& d, size_t bytes) { d.ensure(bytes); CUDA_CHECK(cudaMemset(d.p, 0xFF, bytes)); };
        poisoned(d_lg, (size_t)lrows * ld * 4);                 // the padding columns ld - V stay NaN
        if (!logits_ignored)
            CUDA_CHECK(cudaMemcpy2D(d_lg.p, (size_t)ld * 4, logits, (size_t)V * 4, (size_t)V * 4, lrows, cudaMemcpyHostToDevice));
        if (head_stats) up(d_hs, head_stats, (size_t)R * tiles * 8);
        up(d_mk, masks, (size_t)R * W * 4);
        up(d_occ, occurring_mask, (size_t)W * 4);
        up(d_sc, beam_scores, R * 4); up(d_tk, tokens, (size_t)R * T * 4); up(d_an, ancestry, (size_t)R * T * 4);
        up(d_lo, lo, R * 8); up(d_hi, hi, R * 8); up(d_pw, pw, R * 8);
        poisoned(d_rmax, R * 4); poisoned(d_rls, R * 4); poisoned(d_rule, R); poisoned(d_thr, (size_t)R * 3 * 4);
        poisoned(d_cval, (size_t)R * K * 4); poisoned(d_cidx, (size_t)R * K * 4); poisoned(d_ccnt, R * 4);
        poisoned(d_sco, R * 4); poisoned(d_tko, (size_t)R * T * 4); poisoned(d_ano, (size_t)R * T * 4);
        poisoned(d_loo, R * 8); poisoned(d_hio, R * 8); poisoned(d_pwo, R * 8);
        poisoned(d_hsc, (size_t)Q * K * 4); poisoned(d_hlen, (size_t)Q * K * 4); poisoned(d_htk, (size_t)Q * K * T * 4);
        poisoned(d_hval, (size_t)Q * K); poisoned(d_hlo, (size_t)Q * K * 8); poisoned(d_hhi, (size_t)Q * K * 8);
        d_err.ensure(16); CUDA_CHECK(cudaMemset(d_err.p, 0, 16));

        StepCfg c = step_cfg(p, grp, V);
        set_step(c, cur_len, logits_shared, logits_ignored);
        c.hyps_per_query = K; c.hyp_base = 0;                  // the step's 2B records of each query
        c.head_tiles = head_stats ? tiles : 0;
        StepState st{};
        st.beam_scores_in = d_sc.as<float>(); st.beam_scores_out = d_sco.as<float>();
        st.tokens_in = d_tk.as<int32_t>(); st.tokens_out = d_tko.as<int32_t>();
        st.lo_in = d_lo.as<uint64_t>(); st.lo_out = d_loo.as<uint64_t>(); st.hi_in = d_hi.as<uint64_t>(); st.hi_out = d_hio.as<uint64_t>();
        st.pw_in = d_pw.as<uint64_t>(); st.pw_out = d_pwo.as<uint64_t>();
        st.anc_in = d_an.as<int32_t>(); st.anc_out = d_ano.as<int32_t>();
        st.mask_in = d_mk.as<uint32_t>(); st.occurring_mask = d_occ.as<uint32_t>();
        st.logits = d_lg.as<float>(); st.head_stats = head_stats ? d_hs.as<float2>() : nullptr;
        st.hyp_score = d_hsc.as<float>(); st.hyp_len = d_hlen.as<int32_t>(); st.hyp_tokens = d_htk.as<int32_t>();
        st.hyp_valid = d_hval.as<uint8_t>(); st.hyp_lo = d_hlo.as<uint64_t>(); st.hyp_hi = d_hhi.as<uint64_t>();
        st.error_flag = d_err.as<int32_t>();
        RowScratch rs{d_rmax.as<float>(), d_rls.as<float>(), d_rule.as<uint8_t>(), d_cval.as<float>(), d_cidx.as<int32_t>(),
                      d_ccnt.as<int32_t>(), d_thr.as<float>()};
        set_select_smem();
        *lists = launch_select_step(nullptr, view, c, st, rs, Q);
        CUDA_CHECK(cudaDeviceSynchronize());
        auto down = [&](void* h, const Buf& d, size_t bytes) { CUDA_CHECK(cudaMemcpy(h, d.p, bytes, cudaMemcpyDeviceToHost)); };
        down(row_max, d_rmax, R * 4); down(row_logsum, d_rls, R * 4); down(row_rule, d_rule, R);
        down(cand_val, d_cval, (size_t)R * K * 4); down(cand_idx, d_cidx, (size_t)R * K * 4); down(cand_cnt, d_ccnt, R * 4);
        down(beam_scores_out, d_sco, R * 4); down(tokens_out, d_tko, (size_t)R * T * 4); down(ancestry_out, d_ano, (size_t)R * T * 4);
        down(lo_out, d_loo, R * 8); down(hi_out, d_hio, R * 8); down(pw_out, d_pwo, R * 8);
        down(rec_score, d_hsc, (size_t)Q * K * 4); down(rec_len, d_hlen, (size_t)Q * K * 4); down(rec_tokens, d_htk, (size_t)Q * K * T * 4);
        down(rec_valid, d_hval, (size_t)Q * K); down(rec_lo, d_hlo, (size_t)Q * K * 8); down(rec_hi, d_hhi, (size_t)Q * K * 8);
        down(error_flag, d_err, 4);
    });
}

int sealdec_debug_topk_rows(int64_t R, int32_t V, int32_t num_beams, int32_t per_row, int32_t iters, double* avg_us) {
    return guarded([&] {
        if (R <= 0 || V <= 0 || num_beams < 1 || num_beams > kSelMaxBeams || R % num_beams || per_row < 0 || iters <= 0 || !avg_us)
            throw ApiError(SEALFM_EINVAL, "bad argument");
        require_device();
        const int ld = (V + 3) / 4 * 4, W = (V + 31) / 32, B = num_beams, K = 2 * B, T = 3;
        Buf lg, mk, sc, tk, pw, rmax, rls, rule, cval, cidx, ccnt;
        lg.ensure((size_t)R * ld * 4); mk.ensure((size_t)R * W * 4); sc.ensure((size_t)R * 4); tk.ensure((size_t)R * T * 4);
        pw.ensure((size_t)R * 8); rmax.ensure((size_t)R * 4); rls.ensure((size_t)R * 4); rule.ensure((size_t)R);
        cval.ensure((size_t)R * K * 4); cidx.ensure((size_t)R * K * 4); ccnt.ensure((size_t)R * 4);
        CUDA_CHECK(cudaMemset(mk.p, 0, (size_t)R * W * 4)); CUDA_CHECK(cudaMemset(sc.p, 0, (size_t)R * 4));
        CUDA_CHECK(cudaMemset(tk.p, 0, (size_t)R * T * 4)); CUDA_CHECK(cudaMemset(pw.p, 0, (size_t)R * 8));
        debug_fill_rows_kernel<<<sm_count() * 8, 256>>>(R, V, ld, W, per_row, lg.as<float>(), mk.as<uint32_t>());
        CUDA_CHECK(cudaGetLastError());
        // a later step (cur_len 2) of plain constrained beam search: every row is its own candidate list
        StepCfg c{};
        c.num_beams = B; c.K = K; c.V = V; c.ld = ld; c.cur_len = 2; c.min_length = 0; c.max_length = T;
        c.eos_token_id = 2; c.pad_token_id = 1; c.model_eos_token_id = 2; c.forced_eos_token_id = -1; c.forced_bos_token_id = -1;
        c.T = T; c.mask_words = W; c.expand_next = 1; c.num_groups = 1;
        StepState st{};
        st.beam_scores_in = sc.as<float>(); st.tokens_in = tk.as<int32_t>(); st.pw_in = pw.as<uint64_t>();
        st.mask_in = mk.as<uint32_t>(); st.logits = lg.as<float>();
        RowScratch rs{rmax.as<float>(), rls.as<float>(), rule.as<uint8_t>(), cval.as<float>(), cidx.as<int32_t>(), ccnt.as<int32_t>(),
                      nullptr};
        using RowsLater = SelSharedT<4096>;
        CUDA_CHECK(cudaFuncSetAttribute(topk_rows_kernel<256, 4096>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RowsLater)));
        launch_k(topk_rows_kernel<256, 4096>, (unsigned)R, 256, sizeof(RowsLater), nullptr, c, st, rs, B, 1);
        CUDA_CHECK(cudaDeviceSynchronize());
        cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0, nullptr));
        for (int i = 0; i < iters; ++i) launch_k(topk_rows_kernel<256, 4096>, (unsigned)R, 256, sizeof(RowsLater), nullptr, c, st, rs, B, 1);
        CUDA_CHECK(cudaEventRecord(e1, nullptr));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *avg_us = (double)ms * 1e3 / iters;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    });
}

int sealdec_debug_topk_threshold(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k, float* out_thr,
                                 float* out_max, float* out_logsum) {
    return debug_topk_threshold(false, R, V, ld, logits, top_k, out_thr, out_max, out_logsum);
}

int sealdec_debug_topk_threshold_cluster(int64_t R, int32_t V, int64_t ld, const float* logits, int32_t top_k,
                                         float* out_thr, float* out_max, float* out_logsum) {
    return debug_topk_threshold(true, R, V, ld, logits, top_k, out_thr, out_max, out_logsum);
}

int sealdec_debug_target_logprob(int64_t R, int32_t V, int64_t ld, const float* logits, const int64_t* targets,
                                 int64_t tgt_stride, float temperature, float* out, int64_t out_stride, float* full,
                                 int64_t full_ld) {
    return guarded([&] {
        // only what sealdec_teacher_forced passes: ld >= V, a positive finite temperature, at least one output
        if (R <= 0 || V <= 0 || ld < V || !logits || (!out && !full)) throw ApiError(SEALFM_EINVAL, "bad argument");
        if (!(temperature > 0.f) || !std::isfinite(temperature)) throw ApiError(SEALFM_EINVAL, "temperature must be positive and finite");
        if (out && (!targets || tgt_stride < 1 || out_stride < 1)) throw ApiError(SEALFM_EINVAL, "bad target / output stride");
        if (full && full_ld < V) throw ApiError(SEALFM_EINVAL, "full_ld must be >= V");
        if ((uint64_t)R > INT32_MAX) throw ApiError(SEALFM_EINVAL, "too many rows");
        require_device();
        Buf d_lg, d_tg, d_out, d_full;
        const size_t n_out = out ? (size_t)(R - 1) * out_stride + 1 : 0;
        const size_t n_tg = out ? (size_t)(R - 1) * tgt_stride + 1 : 0;
        const size_t n_full = full ? (size_t)(R - 1) * full_ld + V : 0;
        d_lg.ensure((size_t)R * ld * 4);
        CUDA_CHECK(cudaMemcpy(d_lg.p, logits, (size_t)R * ld * 4, cudaMemcpyHostToDevice));
        // the outputs start as NaN: an element the kernel does not write comes back that way
        if (out) {
            d_tg.ensure(n_tg * 8); d_out.ensure(n_out * 4);
            CUDA_CHECK(cudaMemcpy(d_tg.p, targets, n_tg * 8, cudaMemcpyHostToDevice));
            CUDA_CHECK(cudaMemset(d_out.p, 0xFF, n_out * 4));
        }
        if (full) { d_full.ensure(n_full * 4); CUDA_CHECK(cudaMemset(d_full.p, 0xFF, n_full * 4)); }
        launch_target_logprob(nullptr, R, V, ld, d_lg.as<float>(), out ? d_tg.as<int64_t>() : nullptr, tgt_stride, temperature,
                              out ? d_out.as<float>() : nullptr, out_stride, full ? d_full.as<float>() : nullptr, full_ld);
        CUDA_CHECK(cudaDeviceSynchronize());
        if (out) CUDA_CHECK(cudaMemcpy(out, d_out.p, n_out * 4, cudaMemcpyDeviceToHost));
        if (full) CUDA_CHECK(cudaMemcpy(full, d_full.p, n_full * 4, cudaMemcpyDeviceToHost));
    });
}

}  // extern "C"
