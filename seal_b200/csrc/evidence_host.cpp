// Native host logic of evidence aggregation (include/sealev.h): the two order-defining loops of
// seal/keys.py:316-491 that remain on the host once every FM-index access has been batched onto the GPU
// (seal_b200/keys.py).  Plain C++ on doubles in the reference's own evaluation order, so the results are the
// reference's bit for bit (tests/golden/keys_golden.json was produced by the reference function itself).
// No CUDA here; compiled into libsealb200.so.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/sealev.h"
#include "../../include/sealfm.h"

namespace {

struct KeyView {
    const int64_t* tok; int len;
    bool operator==(const KeyView& o) const { return len == o.len && std::memcmp(tok, o.tok, sizeof(int64_t) * len) == 0; }
};

// Python tuple ordering: element-wise, a proper prefix is smaller
inline int cmp_keys(const KeyView& a, const KeyView& b) {
    const int n = std::min(a.len, b.len);
    for (int i = 0; i < n; ++i) if (a.tok[i] != b.tok[i]) return a.tok[i] < b.tok[i] ? -1 : 1;
    return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}

// keys.py:186-191 `repetition`: score damped by the share of a key's token TYPES already covered
struct Coverage {
    std::unordered_set<int64_t> seen;
    double damp(const int64_t* tok, int len, double score, double beta, std::vector<int64_t>& scratch) const {
        if (seen.empty()) return score;
        scratch.assign(tok, tok + len);
        std::sort(scratch.begin(), scratch.end());
        scratch.erase(std::unique(scratch.begin(), scratch.end()), scratch.end());
        size_t fresh = 0;
        for (int64_t t : scratch) fresh += seen.count(t) ? 0 : 1;
        return (1.0 - beta + (beta * (double)fresh / (double)scratch.size())) * score;
    }
    void add(const int64_t* tok, int len) { seen.insert(tok, tok + len); }
};

thread_local std::string g_err;
bool g_compensated_sum = true;      // how the host interpreter's built-in sum() adds floats (sealev_set_sum_mode)

}  // namespace

namespace sealb200 {
// the message sealev_last_error() returns, for the batched entry points (include/sealev_batch.h)
void sealev_set_error(const std::string& msg) { g_err = msg; }
bool sealev_compensated_sum() { return g_compensated_sum; }
}  // namespace sealb200

extern "C" {

const char* sealev_last_error(void) { return g_err.c_str(); }
void sealev_set_sum_mode(int compensated) { g_compensated_sum = compensated != 0; }

int sealev_first_stage(int64_t n_keys, const int64_t* key_tok, const int64_t* key_off, const double* key_score,
                       const int64_t* key_count, int64_t empty_count, const int64_t* span_off,
                       const uint64_t* pos, const int64_t* doc, int32_t sort_mode, int32_t allow_overlaps, double beta,
                       double single_key, int64_t max_docs, int64_t* out_docs, int64_t* out_n) {
    try {
        if (n_keys < 0 || !key_off || !span_off || !out_docs || !out_n) { g_err = "null argument"; return SEALFM_EINVAL; }
        struct Entry { int64_t doc; double sum; std::vector<std::pair<int64_t, double>> credits; int64_t best; double best_score; };
        std::vector<Entry> entries;                              // insertion order = first touch (defaultdict semantics, :334-345)
        std::unordered_map<int64_t, size_t> slot;
        std::unordered_set<uint64_t> covered;                    // token positions claimed by an earlier key (:316, :339-342)
        auto klen = [&](int64_t k) { return k < 0 ? (int64_t)0 : key_off[k + 1] - key_off[k]; };
        auto kcount = [&](int64_t k) { return k < 0 ? empty_count : key_count[k]; };
        std::unordered_set<int64_t> credited;
        for (int64_t k = 0; k < n_keys; ++k) {
            const int64_t n = klen(k);
            const double sc = key_score[k];
            credited.clear();
            for (int64_t j = span_off[k]; j < span_off[k + 1]; ++j) {
                const uint64_t end = pos[j];
                const int64_t d = doc[j];
                auto it = slot.find(d);
                if (it == slot.end()) { it = slot.emplace(d, entries.size()).first; entries.push_back(Entry{d, 0.0, {}, -1, 0.0}); }
                Entry& e = entries[it->second];
                bool better;                                     // :326-337: (len, score) | (-count, score) | score, strictly greater
                if (sort_mode == 1) better = n != klen(e.best) ? n > klen(e.best) : sc > e.best_score;
                else if (sort_mode == 2) better = kcount(k) != kcount(e.best) ? -kcount(k) > -kcount(e.best) : sc > e.best_score;
                else better = sc > e.best_score;
                if (better) { e.best = k; e.best_score = sc; }
                bool fresh = true;
                for (int64_t t = 0; t < n && fresh; ++t) fresh = !covered.count(end - (uint64_t)n + (uint64_t)t);
                if (fresh) for (int64_t t = 0; t < n; ++t) covered.insert(end - (uint64_t)n + (uint64_t)t);
                if ((fresh || allow_overlaps) && !credited.count(d)) { credited.insert(d); e.sum += sc; e.credits.emplace_back(k, sc); }
            }
        }
        std::vector<int64_t> scratch;
        for (Entry& e : entries) {                               // :353-365
            Coverage cov; double total = 0.0;
            for (auto& c : e.credits) {
                const int64_t* t = key_tok + key_off[c.first]; const int len = (int)klen(c.first);
                total += cov.damp(t, len, c.second, beta, scratch);
                cov.add(t, len);
            }
            e.sum = total;
        }
        std::vector<size_t> order(entries.size());
        for (size_t i = 0; i < order.size(); ++i) order[i] = i;
        auto rank = [&](size_t i) { return (1.0 - single_key) * (-entries[i].sum) + single_key * (-entries[i].best_score); };
        std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return rank(a) < rank(b); });   // :367-368
        const int64_t n_out = std::min<int64_t>((int64_t)order.size(), max_docs < 0 ? 0 : max_docs);
        for (int64_t i = 0; i < n_out; ++i) out_docs[i] = entries[order[i]].doc;
        *out_n = n_out;
        return 0;
    } catch (const std::exception& ex) { g_err = ex.what(); return SEALFM_ENOMEM; }
}

int sealev_score_docs(int64_t n_keys, const int64_t* key_tok, const int64_t* key_off, const double* key_score,
                      const int64_t* key_count, int64_t empty_count, int64_t n_docs, const int64_t* doc_tok,
                      const int64_t* doc_off, const double* unigram, int64_t n_unigram, int32_t sort_mode,
                      int32_t allow_overlaps, int32_t ignore_free_places, int32_t single_key_add_unigrams, double beta,
                      double single_key, double* out_score, int64_t* out_best, double* out_best_score,
                      int64_t* pick_off, int64_t* pick_key, double* pick_score, int64_t pick_cap) {
    try {
        if (!key_off || !doc_off || !out_score || !out_best || !out_best_score || !pick_off) { g_err = "null argument"; return SEALFM_EINVAL; }
        // trie over the scored keys (:378-385); node 0 = root
        struct Node { std::unordered_map<int64_t, int32_t> next; int64_t key = -1; };
        std::vector<Node> trie(1);
        for (int64_t k = 0; k < n_keys; ++k) {
            int32_t cur = 0;
            for (int64_t i = key_off[k]; i < key_off[k + 1]; ++i) {
                auto it = trie[cur].next.find(key_tok[i]);
                if (it == trie[cur].next.end()) { const int32_t nn = (int32_t)trie.size(); trie[cur].next.emplace(key_tok[i], nn); trie.emplace_back(); cur = nn; }
                else cur = it->second;
            }
            trie[cur].key = k;
        }
        auto kview = [&](int64_t k) { return KeyView{key_tok + key_off[k], (int)(key_off[k + 1] - key_off[k])}; };
        auto klen = [&](int64_t k) { return k < 0 ? (int64_t)0 : key_off[k + 1] - key_off[k]; };
        auto kcount = [&](int64_t k) { return k < 0 ? empty_count : key_count[k]; };
        struct Place { int64_t key; int32_t a, b; };
        std::vector<std::pair<int32_t, int32_t>> live, keep;     // (start, trie node)
        std::vector<int64_t> hit_order; std::vector<std::vector<std::pair<int32_t, int32_t>>> places(n_keys);
        std::vector<char> hit(n_keys, 0);
        std::vector<Place> queue;
        std::vector<int64_t> scratch;
        int64_t n_pick = 0;
        pick_off[0] = 0;
        for (int64_t d = 0; d < n_docs; ++d) {
            const int64_t* toks = doc_tok + doc_off[d];
            const int32_t L = (int32_t)(doc_off[d + 1] - doc_off[d]);
            // ---- all occurrences, discovered in the order of the reference's open-match list (:396-409) ----
            for (int64_t k : hit_order) { hit[k] = 0; places[k].clear(); }
            hit_order.clear(); live.clear();
            for (int32_t i = 0; i < L; ++i) {
                keep.clear();
                auto visit = [&](int32_t a, int32_t node) {
                    auto it = trie[node].next.find(toks[i]);
                    if (it == trie[node].next.end()) return;
                    keep.emplace_back(a, it->second);
                    const int64_t k = trie[it->second].key;
                    if (k >= 0) { if (!hit[k]) { hit[k] = 1; hit_order.push_back(k); } places[k].emplace_back(a, i + 1); }
                };
                visit(i, 0);                                     // the match starting here is popped first
                for (size_t m = live.size(); m-- > 0;) visit(live[m].first, live[m].second);
                live.swap(keep);
            }
            // ---- best single key (:413-432) and the greedy queue ----
            int64_t best = -1; double best_score = 0.0;
            queue.clear();
            for (int64_t k : hit_order) {
                const double s = key_score[k];
                bool ahead;                                      // strictly smaller (−len, −s) | (count, −s) | −s
                if (sort_mode == 1) ahead = klen(k) != klen(best) ? -klen(k) < -klen(best) : -s < -best_score;
                else if (sort_mode == 2) ahead = kcount(k) != kcount(best) ? kcount(k) < kcount(best) : -s < -best_score;
                else ahead = -s < -best_score;
                if (ahead) { best = k; best_score = s; }
                for (auto& p : places[k]) queue.push_back(Place{k, p.first, p.second});
            }
            std::sort(queue.begin(), queue.end(), [&](const Place& x, const Place& y) {          // heap order (:420, :441)
                const double sx = key_score[x.key], sy = key_score[y.key];
                if (-sx != -sy) return -sx < -sy;
                if (x.key != y.key) { const int c = cmp_keys(kview(x.key), kview(y.key)); if (c) return c < 0; }
                if (x.a != y.a) return x.a < y.a;
                return x.b < y.b;
            });
            Coverage cov;
            std::vector<char> free_(L, 1);
            const int64_t first_pick = n_pick;
            int64_t prev = -1; double prev_adj = 0.0;
            auto same_key = [&](int64_t x, int64_t y) { return x == y || (x >= 0 && y >= 0 && kview(x) == kview(y)); };
            for (const Place& p : queue) {                       // :434-470
                const KeyView kv = kview(p.key);
                double adj;
                if (prev >= 0 && same_key(prev, p.key)) adj = prev_adj;
                else adj = cov.damp(kv.tok, kv.len, key_score[p.key], beta, scratch);
                if (adj <= 0.0) continue;
                if (!allow_overlaps) { bool ok = true; for (int32_t t = p.a; t < p.b && ok; ++t) ok = free_[t]; if (!ok) continue; }
                if (!(prev >= 0 && same_key(prev, p.key))) {
                    prev = p.key; prev_adj = adj;
                    cov.add(kv.tok, kv.len);
                    if (n_pick >= pick_cap) { g_err = "pick buffer too small"; return SEALFM_ECAPACITY; }
                    pick_key[n_pick] = p.key; pick_score[n_pick] = adj; ++n_pick;
                }
                for (int32_t t = p.a; t < p.b; ++t) free_[t] = 0;
            }
            if (ignore_free_places) std::fill(free_.begin(), free_.end(), 1);
            // :476 is Python's built-in sum(): since CPython 3.12 that is Neumaier-compensated for floats
            // (Python/bltinmodule.c); the fixtures were produced by the reference under 3.12, so this is what "the
            // reference's result" is here (a naive left-to-right sum differs in the last bit on 1 document of 200)
            double total = 0.0;
            if (!g_compensated_sum) {                           // CPython < 3.12: plain left-to-right sum()
                for (int64_t i = first_pick; i < n_pick; ++i) total += pick_score[i];
            } else if (n_pick > first_pick) {
                total = pick_score[first_pick];
                double comp = 0.0;
                for (int64_t i = first_pick + 1; i < n_pick; ++i) {
                    const double x = pick_score[i], t = total + x;
                    if (std::fabs(total) >= std::fabs(x)) comp += (total - t) + x; else comp += (x - t) + total;
                    total = t;
                }
                if (comp != 0.0 && std::isfinite(comp)) total += comp;
            }
            double uni = 0.0;
            if (unigram) {                                       // :479-486: free token types in order of first appearance
                std::unordered_set<int64_t> done;
                for (int32_t i = 0; i < L; ++i) {
                    if (!free_[i] || !done.insert(toks[i]).second) continue;
                    const int64_t t = toks[i];
                    if (t < 0 || t >= n_unigram) { g_err = "token id outside the unigram table"; return SEALFM_EINVAL; }
                    double s = unigram[t];
                    if (s > 0.0) {
                        s = cov.damp(&t, 1, s, beta, scratch);
                        if (s != 0.0) {
                            uni += s;
                            if (n_pick >= pick_cap) { g_err = "pick buffer too small"; return SEALFM_ECAPACITY; }
                            pick_key[n_pick] = -1 - t; pick_score[n_pick] = s; ++n_pick;      // unigram pick: -(token) - 1
                        }
                    }
                }
            }
            const double lone = best_score + (single_key_add_unigrams ? uni : 0.0);
            total += uni;
            out_score[d] = (1.0 - single_key) * total + single_key * lone;
            out_best[d] = best; out_best_score[d] = best_score;
            pick_off[d + 1] = n_pick;
        }
        return 0;
    } catch (const std::exception& ex) { g_err = ex.what(); return SEALFM_ENOMEM; }
}

}  // extern "C"
