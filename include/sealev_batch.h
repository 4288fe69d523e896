/* sealev_batch.h -- evidence aggregation (seal/keys.py:178-497) for a whole batch of queries.
 *
 * seal_b200.keys.batch_aggregate_evidence returns, for every query, exactly what seal_b200.keys.aggregate_evidence
 * returns for that query alone (same document order, key order and floats).  It prepares the keys of all queries with
 * the host functions below, computes every distinct SA range in one sealfm_backward_search_multi launch, and runs the
 * two per-query loops of sealev.h -- the first stage and the full scoring of the shortlisted documents -- as CUDA
 * kernels over the whole batch (sealev_batch_first_stage, sealev_batch_score_docs).
 *
 * Scalar scoring: the reference's Python float arithmetic, evaluated with the C library's log / exp / pow (what
 * CPython's math.log, math.exp and float ** float call) in the same order.  Where Python raises, these return
 * SEALFM_EINVAL and sealev_last_error() holds Python's message ("math domain error", "math range error",
 * "0.0 cannot be raised to a negative power").
 *
 * Batch entry points: per-query key sets are flattened like sealev.h's (key k = key_tok[key_off[k] ..
 * key_off[k+1])), and query q owns keys query_key_off[q] .. query_key_off[q+1]).  Key indices in outputs are local to
 * their query.  They run on the device and stream of the FM handle, synchronously, and return 0 or a SEALFM_E* code
 * (sealev_last_error() for the message).  Batches whose located rows or document tokens exceed the device budget
 * (sealev_set_device_budget) are processed in chunks of whole queries; the results do not depend on the chunking. */
#ifndef SEALEV_BATCH_H
#define SEALEV_BATCH_H
#include <stdint.h>
#include "sealfm.h"
#ifdef __cplusplus
extern "C" {
#endif

/* _Evidence.key_score (seal_b200/keys.py; seal/keys.py:208-235) of n keys: sr[i] = the key's decoder score,
 * count[i] its corpus count, len[i] its length, cutoff[i] its query's cutoff (read only when use_fm_index_frequency
 * is 0).  ntokens = float(len(index)). */
int sealev_key_scores(int64_t n, const double* sr, const int64_t* count, const int64_t* len, const double* cutoff,
                      double ntokens, double alpha, double length_penalty, double smoothing,
                      int32_t use_fm_index_frequency, double* out);

/* The first top_k tokens of argsort(-scores[q], kind="stable") that are not in the query's `given` set
 * (given_tok[given_off[q] .. given_off[q+1])), for each of n_queries rows of V scores.  top_k follows Python slice
 * semantics (negative: all but the last -top_k).  out_tok: n_queries rows of min(V, max(top_k, 0)) entries (a negative
 * top_k: V entries); out_n[q] = tokens written to row q. */
int sealev_unigram_topk(int64_t n_queries, int64_t V, const double* scores, int64_t top_k, const int64_t* given_off,
                        const int64_t* given_tok, int64_t* out_tok, int64_t* out_n);

/* The unigram table entries (_Evidence.unigram_table; seal/keys.py:237-272) of n kept tokens: s[i] = the token's
 * unigram score, count[i] its corpus count, cutoff[i] its query's cutoff. */
int sealev_unigram_scores(int64_t n, const double* s, const int64_t* count, const double* cutoff, double ntokens,
                          double alpha, double smoothing, int32_t use_fm_index_frequency, double* out);

/* add_best_unigrams_to_ngrams (seal/keys.py:274-278): sorted(range(V), key=-table[t])[:n_extra[q]] for each query's
 * table, given sparse (its nonzero entries tab_tok / tab_val[tab_off[q] .. tab_off[q+1]), any order) over V[q]
 * tokens.  Writes min(n_extra[q], V[q]) tokens and their table values from out_off[q]; out_off has n_queries + 1
 * entries and is filled by the callee. */
int sealev_best_unigrams(int64_t n_queries, const int64_t* V, const int64_t* tab_off, const int64_t* tab_tok,
                         const double* tab_val, const int64_t* n_extra, int64_t* out_off, int64_t* out_tok,
                         double* out_val, int64_t out_cap);

/* Device bytes one chunk of a batch call may use for its located rows or document tokens (0: 2 GiB).  Smaller values
 * force smaller chunks; a single query is never split. */
void sealev_set_device_budget(uint64_t bytes);

/* sealev_first_stage for every query at once.  Key k's located rows are SA rows key_lo[k] .. key_lo[k] + key_rows[k]
 * (the caller caps them at max_occurrences_1); empty_count[q] = query q's count of the empty key.  Shortlist of query
 * q: out_docs[out_off[q] .. out_off[q+1]), at most max_docs documents; out_cap >= sum_q min(max_docs, rows of q). */
int sealev_batch_first_stage(const sealfm_t* h, int64_t n_queries, const int64_t* query_key_off, const int64_t* key_tok,
                             const int64_t* key_off, const double* key_score, const int64_t* key_count,
                             const uint64_t* key_lo, const int64_t* key_rows, const int64_t* empty_count,
                             int32_t sort_mode, int32_t allow_overlaps, double beta, double single_key, int64_t max_docs,
                             int64_t* out_off, int64_t* out_docs, int64_t out_cap);

/* sealev_score_docs for every query at once.  Query q scores documents docs[query_doc_off[q] .. query_doc_off[q+1])
 * (document ids of the index; their tokens are extracted on the device, symbol - shift, and laid out as the
 * reference's [2] + doc[:-1]) against its keys.  Its unigram table is uni_tok / uni_val[query_uni_off[q] ..
 * query_uni_off[q+1]) (nonzero entries, any order) over uni_size[q] tokens; uni_size[q] < 0: the query has no unigram
 * scores.  Outputs per document d of the batch: its tokens doc_tok[doc_tok_off[d] .. doc_tok_off[d+1]) (doc_tok_off is
 * filled by the callee; tok_cap >= sum of max(length, 1)), out_score, out_best (local key index or -1) /
 * out_best_score, and picks pick_key / pick_score[pick_off[d] .. pick_off[d+1]) as in sealev_score_docs.  If the picks
 * exceed pick_cap the call returns SEALFM_ECAPACITY with *pick_needed set to the exact count. */
int sealev_batch_score_docs(const sealfm_t* h, int64_t n_queries, const int64_t* query_key_off, const int64_t* key_tok,
                            const int64_t* key_off, const double* key_score, const int64_t* key_count,
                            const int64_t* empty_count, const int64_t* query_doc_off, const int64_t* docs,
                            const int64_t* query_uni_off, const int64_t* uni_tok, const double* uni_val,
                            const int64_t* uni_size, int64_t shift, int32_t sort_mode, int32_t allow_overlaps,
                            int32_t ignore_free_places, int32_t single_key_add_unigrams, double beta, double single_key,
                            int64_t* doc_tok_off, int64_t* doc_tok, int64_t tok_cap, double* out_score, int64_t* out_best,
                            double* out_best_score, int64_t* pick_off, int64_t* pick_key, double* pick_score,
                            int64_t pick_cap, int64_t* pick_needed);

/* Wall time (microseconds) of the phases of the calling thread's last batch call: [0] ranges-to-rows + locate,
 * [1] the rest of the first stage, [2] extraction, [3] scoring (chunks summed; device work timed by synchronising). */
void sealev_batch_phase_us(double* out4);

#ifdef __cplusplus
}
#endif
#endif
