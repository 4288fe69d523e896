// Host preparation of batched evidence aggregation (include/sealev_batch.h): the scalar scoring of
// seal_b200/keys.py's _Evidence (key_score, contrast, unigram_table) and the add_best_unigrams_to_ngrams extras, for
// every key of a batch in one call.  Python's float arithmetic in Python's order, on the C library's log / exp / pow
// (what math.log, math.exp and float ** float call), raising where Python raises.  No CUDA here.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <new>
#include <numeric>
#include <stdexcept>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../include/sealev_batch.h"

namespace sealb200 { void sealev_set_error(const std::string& msg); }   // evidence_host.cpp

namespace {

struct ApiError : std::runtime_error {
    int code;
    ApiError(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

// status code + sealev_last_error() message; no exception leaves the ABI
template <typename Fn>
int guarded(Fn&& fn) {
    try { fn(); return 0; }
    catch (const ApiError& e) { sealb200::sealev_set_error(e.what()); return e.code; }
    catch (const std::bad_alloc&) { sealb200::sealev_set_error("out of host memory"); return SEALFM_ENOMEM; }
    catch (const std::exception& e) { sealb200::sealev_set_error(e.what()); return SEALFM_EINVAL; }
}

// math.log: ValueError for x <= 0 (Modules/mathmodule.c m_log)
double py_log(double x) {
    if (std::isnan(x)) return x;
    if (x <= 0.0) throw ApiError(SEALFM_EINVAL, "math domain error");
    return std::log(x);
}

// math.exp: OverflowError when a finite argument overflows
double py_exp(double x) {
    const double r = std::exp(x);
    if (std::isinf(r) && std::isfinite(x)) throw ApiError(SEALFM_EINVAL, "math range error");
    return r;
}

// float ** float (Objects/floatobject.c float_pow): its error cases; the value is the C library's pow
double py_pow(double x, double y) {
    if (std::isfinite(x) && std::isfinite(y)) {
        if (x == 0.0 && y < 0.0) throw ApiError(SEALFM_EINVAL, "0.0 cannot be raised to a negative power");
        if (x < 0.0 && y != std::floor(y)) throw ApiError(SEALFM_EINVAL, "math domain error");
    }
    const double r = std::pow(x, y);
    if (std::isinf(r) && std::isfinite(x) && std::isfinite(y)) throw ApiError(SEALFM_EINVAL, "math range error");
    return r;
}

// max(x, 0.0): the first argument unless 0.0 > x (so NaN and -0.0 stay)
inline double py_max0(double x) { return 0.0 > x ? 0.0 : x; }

// _Evidence.contrast (seal/keys.py:220-223, :250-253)
double contrast(double sr, int64_t count, double ntokens, double smoothing) {
    const double snr = py_log(((double)count + smoothing) / (ntokens + smoothing));
    return (sr + py_log(1 - py_exp(snr))) - (snr + py_log(1 - py_exp(sr)));
}

// sort order of (-score, token): Python's stable sort of the negated scores
inline bool neg_before(double sa, int64_t ta, double sb, int64_t tb) {
    const double na = -sa, nb = -sb;
    if (na < nb) return true;
    if (nb < na) return false;
    return ta < tb;
}

}  // namespace

extern "C" {

int sealev_key_scores(int64_t n, const double* sr, const int64_t* count, const int64_t* len, const double* cutoff,
                      double ntokens, double alpha, double length_penalty, double smoothing,
                      int32_t use_fm_index_frequency, double* out) {
    return guarded([&] {
        if (n < 0 || (n && (!sr || !count || !len || !out || (!use_fm_index_frequency && !cutoff))))
            throw ApiError(SEALFM_EINVAL, "null argument");
        for (int64_t i = 0; i < n; ++i) {                       // _Evidence.key_score
            if (count[i] == 0) { out[i] = 0.0; continue; }
            const double decay = py_pow(1.0 - length_penalty, (double)len[i] - 1.0);
            double sc;
            if (use_fm_index_frequency) sc = py_max0(contrast((sr[i] - 1e-10) * decay, count[i], ntokens, smoothing));
            else sc = py_max0(sr[i] - cutoff[i]) * decay;
            out[i] = py_pow(sc, alpha);
        }
    });
}

int sealev_unigram_topk(int64_t n_queries, int64_t V, const double* scores, int64_t top_k, const int64_t* given_off,
                        const int64_t* given_tok, int64_t* out_tok, int64_t* out_n) {
    return guarded([&] {
        if (n_queries < 0 || V < 0 || (n_queries && (!scores || !given_off || !out_tok || !out_n)))
            throw ApiError(SEALFM_EINVAL, "null argument");
        const int64_t kk = top_k >= 0 ? std::min(top_k, V) : std::max<int64_t>(V + top_k, 0);
        std::vector<int64_t> idx(V);
        std::unordered_set<int64_t> given;
        for (int64_t q = 0; q < n_queries; ++q) {
            const double* s = scores + q * V;
            std::iota(idx.begin(), idx.end(), 0);
            // (-score, token) is a total order, so a partial sort gives the stable argsort's first kk entries
            std::partial_sort(idx.begin(), idx.begin() + kk, idx.end(),
                              [&](int64_t a, int64_t b) { return neg_before(s[a], a, s[b], b); });
            given.clear();
            for (int64_t i = given_off[q]; i < given_off[q + 1]; ++i) given.insert(given_tok[i]);
            int64_t w = 0;
            for (int64_t i = 0; i < kk; ++i)
                if (!given.count(idx[i])) out_tok[q * kk + w++] = idx[i];
            out_n[q] = w;
        }
    });
}

int sealev_unigram_scores(int64_t n, const double* s, const int64_t* count, const double* cutoff, double ntokens,
                          double alpha, double smoothing, int32_t use_fm_index_frequency, double* out) {
    return guarded([&] {
        if (n < 0 || (n && (!s || !count || !out || (!use_fm_index_frequency && !cutoff))))
            throw ApiError(SEALFM_EINVAL, "null argument");
        for (int64_t i = 0; i < n; ++i) {                       // _Evidence.unigram_table, one kept token
            if (count[i] == 0) { out[i] = 0.0; continue; }
            if (use_fm_index_frequency) out[i] = py_max0(contrast(s[i], count[i], ntokens, smoothing));
            else out[i] = py_pow(py_max0(s[i] - cutoff[i]), alpha);
        }
    });
}

int sealev_best_unigrams(int64_t n_queries, const int64_t* V, const int64_t* tab_off, const int64_t* tab_tok,
                         const double* tab_val, const int64_t* n_extra, int64_t* out_off, int64_t* out_tok,
                         double* out_val, int64_t out_cap) {
    return guarded([&] {
        if (n_queries < 0 || !out_off || (n_queries && (!V || !tab_off || !n_extra)))
            throw ApiError(SEALFM_EINVAL, "null argument");
        out_off[0] = 0;
        std::vector<std::pair<int64_t, double>> nz;
        std::unordered_set<int64_t> nz_set;
        for (int64_t q = 0; q < n_queries; ++q) {
            const int64_t m = std::max<int64_t>(0, std::min(n_extra[q], V[q]));
            out_off[q + 1] = out_off[q] + m;
            if (out_off[q + 1] > out_cap) throw ApiError(SEALFM_ECAPACITY, "output buffer too small");
            // the table's nonzero entries (all positive) come first by (-value, token), then its zeros by token
            nz.clear(); nz_set.clear();
            for (int64_t i = tab_off[q]; i < tab_off[q + 1]; ++i)
                if (tab_val[i] != 0.0) { nz.emplace_back(tab_tok[i], tab_val[i]); nz_set.insert(tab_tok[i]); }
            std::sort(nz.begin(), nz.end(), [](const std::pair<int64_t, double>& a, const std::pair<int64_t, double>& b) {
                return neg_before(a.second, a.first, b.second, b.first);
            });
            int64_t w = out_off[q];
            for (size_t i = 0; i < nz.size() && w < out_off[q + 1]; ++i) { out_tok[w] = nz[i].first; out_val[w] = nz[i].second; ++w; }
            for (int64_t t = 0; t < V[q] && w < out_off[q + 1]; ++t)
                if (!nz_set.count(t)) { out_tok[w] = t; out_val[w] = 0.0; ++w; }
        }
    });
}

}  // extern "C"
