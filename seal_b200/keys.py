"""Drop-in for ``seal.keys`` (/root/reference/seal/keys.py): the decoder-side helpers that run right
after every generate pass (SURVEY.md §8f rank 1) -- ``rescore_keys`` (:64-141) and
``compute_unigram_scores`` (:145-176), on the kernels behind ``sealdec_teacher_forced``
(include/sealdec.h) -- and the evidence aggregation (§8f rank 2) ``aggregate_evidence`` (:178-497),
whose FM-index accesses are three batched GPU launches.  Same signatures and return values.
No CPU path."""
import ctypes as C
from typing import List, Optional

import sys

import numpy as np

from ._lib import lib, check
from .beam_search import _engine_for


def strip(seq, symbols_start, symbols_end):                     # keys.py:53-61
    i = 0
    while i < len(seq) and seq[i] in symbols_start:
        i += 1
    j = len(seq)
    while j > i and seq[j - 1] in symbols_end:
        j -= 1
    return seq[i:j]


def _pad_inputs(batch_in, pad):
    maxlen = max(len(i) for i in batch_in)
    ids = np.full((len(batch_in), maxlen), pad, dtype=np.int64)
    for r, i in enumerate(batch_in):
        ids[r, :len(i)] = i
    return ids, (ids != pad).astype(np.int64)                   # keys.py:78-82


def _teacher_forced(eng, ids, mask, dec, row_query, temperature=1.0, full_pos=-1):
    N, T = dec.shape
    Q, S = ids.shape
    V = int(eng.config.vocab_size)
    out = np.zeros((N, max(T - 1, 1)), dtype=np.float32)
    full = np.empty((N, V), dtype=np.float32) if full_pos >= 0 else None
    rq = np.ascontiguousarray(row_query, dtype=np.int32)
    check(lib.sealdec_teacher_forced(eng._h, ids.ctypes.data, mask.ctypes.data, Q, S, dec.ctypes.data, rq.ctypes.data, N, T,
                                     C.c_float(temperature), out.ctypes.data if T > 1 else None, full_pos,
                                     full.ctypes.data if full is not None else None))
    return out[:, :T - 1], full


def rescore_keys(model, inputs, list_of_decoded, batch_size=100, length_penalty=0.0, progress_bar=False, prefix=[],
                 strip_from_bos=[], strip_from_eos=[]):
    """keys.py:64-141.  `batch_size` is accepted for signature compatibility; the native pass chunks rows itself."""
    eng = _engine_for(model)
    cfg = eng.config
    if inputs is None:                                                           # :70-73
        batch_in = [[cfg.bos_token_id, cfg.eos_token_id]] * len(list_of_decoded)
    else:
        batch_in = [list(i) for i in inputs]
    list_of_decoded = [[x[1] if isinstance(x[0], float) else x for x in xx] for xx in list_of_decoded]   # :75
    ids, mask = _pad_inputs(batch_in, cfg.pad_token_id)
    rows, row_query, orig = [], [], []
    for idx, ddi in enumerate(list_of_decoded):                                  # :87-104
        for di in ddi:
            di = list(di.tolist() if hasattr(di, "tolist") else di)
            stripped = [cfg.decoder_start_token_id] + list(prefix) + strip(di, strip_from_bos, strip_from_eos)
            rows.append(stripped); row_query.append(idx); orig.append(di)
    all_out = {i: [] for i in range(len(list_of_decoded))}
    if not rows:
        return [v for k, v in sorted(all_out.items())]
    T = max(len(r) for r in rows)
    dec = np.full((len(rows), T), cfg.pad_token_id, dtype=np.int64)              # :110-116
    for r, toks in enumerate(rows):
        dec[r, :len(toks)] = toks
    lp, _ = _teacher_forced(eng, ids, mask, dec, row_query)
    lp[dec[:, 1:] < 2] = 0.0                                                     # :132
    lp = lp[:, len(prefix):].sum(-1, dtype=np.float32)                           # :133-134 (the reference sums the fp32 tensor)
    for q, di, ll in zip(row_query, orig, lp.tolist()):
        all_out[q].append((ll / (len(di) ** length_penalty), di))                # :138-139
    return [v for k, v in sorted(all_out.items())]


def compute_unigram_scores(model, inputs, index=None, tokenizer=None, tolist=True, temperature=1.0, prefix=[]):
    """keys.py:145-176: full-vocabulary log-probs of the first decoded position (after `prefix`)."""
    eng = _engine_for(model)
    cfg = eng.config
    if isinstance(inputs[0], str):
        batch = tokenizer(inputs, padding=True, return_tensors="np")
        ids = np.ascontiguousarray(batch["input_ids"], dtype=np.int64)
        mask = np.ascontiguousarray(batch["attention_mask"], dtype=np.int64)
    else:
        ids, mask = _pad_inputs([list(i) for i in inputs], cfg.pad_token_id)
    dec = np.full((ids.shape[0], 1 + len(prefix)), cfg.decoder_start_token_id, dtype=np.int64)   # :164-166
    for i, t in enumerate(prefix, start=1):
        dec[:, i] = t
    _, full = _teacher_forced(eng, ids, mask, dec, np.arange(ids.shape[0]), temperature=temperature, full_pos=len(prefix))
    return full.tolist() if tolist else full


# ------------------------------------------------------------------------------------------------
# Evidence aggregation (SURVEY.md §8f rank 2; /root/reference/seal/keys.py:178-497).
#
# The reference walks the FM-index one call at a time from Python: get_count per key (twice), per
# vocabulary entry, then locate + get_doc_index per SA row (up to max_occurrences_1 rows per key) and
# get_doc per shortlisted document.  Here every index access of a call is one of three batched GPU
# launches -- all interval searches (sealfm_backward_search_multi), all row locations (sealfm_locate)
# and all document extractions (sealfm_extract_text); the ordering / set logic that defines the
# result stays on the host, arranged around those three batches.  Same signature, same return value
# (document order, key order and every float identical to the reference's).
# ------------------------------------------------------------------------------------------------
import math as _math
from collections import Counter as _Counter


class _Evidence:
    def __init__(self, index, p):
        self.index, self.p = index, p
        self.ntokens = float(index.beginnings[-1])                                          # keys.py:193
        self.range_of = {}                       # token tuple -> (lo, hi) half-open SA range

    # -- batch 1: SA ranges ------------------------------------------------------------------------
    def need_ranges(self, seqs):
        todo = [s for s in dict.fromkeys(tuple(s) for s in seqs) if s not in self.range_of]
        if todo:
            lo, hi = self.index.get_range_batch([list(s) for s in todo])
            for s, l, h in zip(todo, lo.tolist(), hi.tolist()):
                self.range_of[s] = (l, h)

    def count(self, seq):
        lo, hi = self.range_of[tuple(seq)]
        return hi - lo

    # -- scalar scoring (kept in Python floats: the reference's exact arithmetic) ------------------
    def contrast(self, sr, count):                                                          # :220-223, :250-253
        p = self.p
        snr = _math.log((count + p["smoothing"]) / (self.ntokens + p["smoothing"]))
        return (sr + _math.log(1 - _math.exp(snr))) - (snr + _math.log(1 - _math.exp(sr)))

    def damp(self, types, score, seen):                                                     # :186-191
        if not seen:
            return score
        types = set(types)
        beta = self.p["beta"]
        return (1.0 - beta + (beta * len(types.difference(seen)) / len(types))) * score

    def key_score(self, key, sr, cutoff):                                                   # :208-235
        p = self.p
        c = self.count(key)
        if c == 0:
            return 0.0
        decay = (1.0 - p["length_penalty"]) ** (len(key) - 1.0)
        if p["use_fm_index_frequency"]:
            sc = max(self.contrast((sr - 1e-10) * decay, c), 0.0)
        else:
            sc = max(sr - cutoff, 0.0) * decay
        return sc ** p["alpha"]

    def unigram_table(self, unigram_scores, given, cutoff):                                 # :237-272
        p = self.p
        V = len(unigram_scores)
        # sorted(range(V), reverse=True, key=score)[:k] (:240-241): a stable sort of the negated scores keeps the
        # lower token id first among ties, like reverse=True on a stable sort does
        us = np.asarray(unigram_scores, dtype=np.float64)
        order = np.argsort(-us, kind="stable")[:p["use_top_k_unigrams"]].tolist()
        kept = [t for t in order if t not in given]
        unigram_scores = us.tolist() if not isinstance(unigram_scores, list) else unigram_scores
        self.need_ranges([(t,) for t in kept])               # only the kept ones can score above zero
        table = [0.0] * V
        for t in kept:
            c = self.count((t,))
            if c == 0:
                continue
            if p["use_fm_index_frequency"]:
                sc = max(self.contrast(unigram_scores[t], c), 0.0)
            else:
                sc = max(unigram_scores[t] - cutoff, 0.0) ** p["alpha"]
            if sc != 0.0:
                table[t] = sc
        return table


def aggregate_evidence(ngrams_and_scores, unigram_scores: Optional[List[float]] = None, index=None,
                       max_occurrences_1: int = 1500, max_occurrences_2: int = 10_000_000,
                       n_docs_complete_score: int = 500, alpha: float = 2.0, beta: float = 0.8,
                       length_penalty: float = 0.0, use_fm_index_frequency: bool = True,
                       add_best_unigrams_to_ngrams: bool = False, use_top_k_unigrams=1000, sort_by_length=False,
                       sort_by_freq=False, smoothing=5.0, allow_overlaps=False, single_key=0.0,
                       single_key_add_unigrams=False, unigrams_ignore_free_places=False):
    """seal/keys.py:178-497.  Returns (results, all_ngrams): results = {doc: [score, [(key, score)...],
    None, doc_tokens, [best key, best score]]} sorted by descending score; all_ngrams = {key: score}."""
    ev = _Evidence(index, dict(alpha=alpha, beta=beta, length_penalty=length_penalty, smoothing=smoothing,
                               use_fm_index_frequency=use_fm_index_frequency, use_top_k_unigrams=use_top_k_unigrams))
    keys = [((k.tolist() if hasattr(k, "tolist") else list(k)), s) for k, s in ngrams_and_scores]
    cutoff = None
    if not use_fm_index_frequency:                                                          # :198-205
        cutoff = min(keys, key=lambda ks: ks[1])[1] - 0.1 if keys else [][0]
    ev.need_ranges([k for k, _ in keys])
    counts = {(): len(index)}                                                               # :196
    for k, _ in keys:
        counts[tuple(k)] = ev.count(k)
    given = {0, 1, 2} | {k[0] for k, _ in keys if len(k) == 1}                              # :207-211
    keys = [(k, ev.key_score(k, s, cutoff)) for k, s in keys]

    if unigram_scores is not None:
        unigram_scores = ev.unigram_table(unigram_scores, given, cutoff)
        if add_best_unigrams_to_ngrams:                                                     # :274-278
            extra = sorted(range(len(unigram_scores)), key=lambda t: -unigram_scores[t])[:len(keys)]
            ev.need_ranges([(t,) for t in extra])
            for t in extra:
                counts[(t,)] = ev.count((t,))
                keys.append(([t], unigram_scores[t]))

    # rare keys drive the first stage; frequent ones only take part in the full scoring  (:280-314)
    rare, freq = {}, {}
    for k, sc in keys:
        c = ev.count(k)
        if c > max_occurrences_2 or sc == 0.0:
            continue
        (freq if (c > max_occurrences_1 or sc < 0.0) else rare)[tuple(k)] = sc
    by_score = lambda kv: kv[1]
    rare = dict(sorted(rare.items(), key=by_score, reverse=True))
    freq = dict(sorted(freq.items(), key=by_score, reverse=True))
    all_ngrams = dict(sorted(list(rare.items()) + list(freq.items()), key=by_score, reverse=True))

    # -- batch 2: every SA row of every rare key, located and mapped to its document at once ------
    spans = []
    for k in rare:
        lo, hi = ev.range_of[k]
        spans.append((lo, max(lo, min(hi, lo + max_occurrences_1))))
    if any(b > a for a, b in spans):
        rows = np.concatenate([np.arange(a, b, dtype=np.uint64) for a, b in spans])
        pos, doc = index.locate_rows(rows)
    else:
        pos, doc = np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.int64)
    sort_mode = 1 if sort_by_length else (2 if sort_by_freq else 0)
    empty_count = int(counts[()])

    # first stage (:316-368) in native code: coverage of token positions, one credit per (key, document), damping
    # of repeated token types, shortlist of the n_docs_complete_score best documents
    rk = _FlatKeys(list(rare.items()), counts)
    span_off = np.zeros(len(spans) + 1, dtype=np.int64)
    np.cumsum([b - a for a, b in spans], out=span_off[1:])
    shortlist = np.zeros(max(len(pos), 1), dtype=np.int64); n_short = C.c_int64(0)
    _evcheck(lib.sealev_first_stage(len(rk), rk.tok.ctypes.data, rk.off.ctypes.data, rk.score.ctypes.data, rk.count.ctypes.data,
                                    empty_count, span_off.ctypes.data, np.ascontiguousarray(pos, dtype=np.uint64).ctypes.data,
                                    np.ascontiguousarray(doc, dtype=np.int64).ctypes.data, sort_mode, int(bool(allow_overlaps)),
                                    float(beta), float(single_key), int(n_docs_complete_score), shortlist.ctypes.data,
                                    C.byref(n_short)))
    shortlist = shortlist[:n_short.value].tolist()

    # -- batch 3: the shortlisted documents' tokens -----------------------------------------------
    fetch = getattr(index, "get_docs_arrays", None)
    texts = fetch(shortlist) if fetch else [np.asarray(t, dtype=np.int64) for t in index.get_docs(shortlist)]
    docs_arr = []
    for t in texts:                                                                         # :389: [2] + doc[:-1]
        a = np.empty(max(len(t), 1), dtype=np.int64)
        a[0] = 2; a[1:] = t[:-1]
        docs_arr.append(a)
    docs_tok = [a.tolist() for a in docs_arr]
    scored = [(k, v) for k, v in all_ngrams.items() if len(k) >= 1 and v > 0.0]             # trie contents, :378-385
    sk = _FlatKeys(scored, counts)
    doc_off = np.zeros(len(docs_tok) + 1, dtype=np.int64)
    np.cumsum([len(t) for t in docs_tok], out=doc_off[1:])
    flat = np.concatenate(docs_arr) if docs_arr else np.zeros(0, dtype=np.int64)
    uni = np.ascontiguousarray(unigram_scores, dtype=np.float64) if unigram_scores is not None else None
    n = len(docs_tok)
    out_score = np.zeros(max(n, 1)); out_best = np.zeros(max(n, 1), dtype=np.int64); out_best_score = np.zeros(max(n, 1))
    pick_off = np.zeros(n + 1, dtype=np.int64)
    # a document cannot pick more keys + unigram types than it has tokens -- when overlaps are forbidden.  With
    # allow_overlaps every nested / overlapping match is picked, so the buffer simply grows on SEALFM_ECAPACITY.
    cap = int(doc_off[-1]) * 2 + 16
    lib.sealev_set_sum_mode(1 if sys.version_info >= (3, 12) else 0)     # how this interpreter's sum() adds floats (:476)
    while True:
        pick_key = np.zeros(cap, dtype=np.int64); pick_score = np.zeros(cap)
        rc = lib.sealev_score_docs(len(sk), sk.tok.ctypes.data, sk.off.ctypes.data, sk.score.ctypes.data, sk.count.ctypes.data,
                                   empty_count, n, flat.ctypes.data, doc_off.ctypes.data,
                                   uni.ctypes.data if uni is not None else None, len(uni) if uni is not None else 0, sort_mode,
                                   int(bool(allow_overlaps)), int(bool(unigrams_ignore_free_places)),
                                   int(bool(single_key_add_unigrams)), float(beta), float(single_key), out_score.ctypes.data,
                                   out_best.ctypes.data, out_best_score.ctypes.data, pick_off.ctypes.data, pick_key.ctypes.data,
                                   pick_score.ctypes.data, cap)
        if rc == -6 and cap < (1 << 34):             # SEALFM_ECAPACITY
            cap *= 4
            continue
        _evcheck(rc)
        break
    results = {}
    pk, ps, po = pick_key.tolist(), pick_score.tolist(), pick_off.tolist()
    for i, d in enumerate(shortlist):
        picked = [((scored[k][0] if k >= 0 else (-1 - k,)), s) for k, s in zip(pk[po[i]:po[i + 1]], ps[po[i]:po[i + 1]])]
        b = int(out_best[i])
        best = [scored[b][0], float(out_best_score[i])] if b >= 0 else [[], 0.0]
        results[d] = [float(out_score[i]), picked, None, docs_tok[i], best]
    return dict(sorted(results.items(), key=lambda kv: -kv[1][0])), all_ngrams              # :496-497


class _FlatKeys:
    """(key tuple, score) pairs flattened for the native calls (include/sealev.h)."""

    def __init__(self, items, counts):
        self.off = np.zeros(len(items) + 1, dtype=np.int64)
        np.cumsum([len(k) for k, _ in items], out=self.off[1:])
        self.tok = np.fromiter((t for k, _ in items for t in k), dtype=np.int64, count=int(self.off[-1])) if items else np.zeros(0, dtype=np.int64)
        if len(self.tok) == 0:
            self.tok = np.zeros(1, dtype=np.int64)
        self.score = np.array([s for _, s in items], dtype=np.float64) if items else np.zeros(1)
        self.count = np.array([counts[tuple(k)] for k, _ in items], dtype=np.int64) if items else np.zeros(1, dtype=np.int64)
        self.n = len(items)

    def __len__(self):
        return self.n


def _evcheck(code):
    if code != 0:
        from ._lib import SealB200Error
        raise SealB200Error(code, lib.sealev_last_error().decode(errors="replace"))


_END = -1                                         # trie slot holding (key, score) of a complete key


def _build_trie(scored):
    root = {}
    for k, sc in scored.items():
        node = root
        for t in k:
            node = node.setdefault(t, {})
        node[_END] = (k, sc)
    return root


def _scan_keys(toks, root):
    """All occurrences of the scored keys in one document -> {key: [score, [(start, end)...]]}, keys in the
    order the reference's open-match list discovers them (it is popped from its END at every position,
    keys.py:400-409, so the visiting order of the live partial matches flips from one token to the next;
    only the order in which equal-scored keys are met depends on it).  Partial matches are (start, trie node)
    pairs, so a position costs one dict lookup per live match instead of a tuple slice and two set probes."""
    hits = {}
    live = []
    for i, t in enumerate(toks):
        keep = []
        node = root.get(t)                        # the match starting here is visited first
        if node is not None:
            keep.append((i, node))
            end = node.get(_END)
            if end is not None:
                hits.setdefault(end[0], [end[1], []])[1].append((i, i + 1))
        for a, node in reversed(live):
            node = node.get(t)
            if node is not None:
                keep.append((a, node))
                end = node.get(_END)
                if end is not None:
                    hits.setdefault(end[0], [end[1], []])[1].append((a, i + 1))
        live = keep
    return hits


# ------------------------------------------------------------------------------------------------
# Batched evidence aggregation: aggregate_evidence for a whole batch of queries (include/sealev_batch.h).
#
# The scalar scoring of every key and unigram of the batch runs in native host code (sealev_key_scores,
# sealev_unigram_topk / _scores, sealev_best_unigrams), every distinct SA range of the batch is computed in one
# backward_search_multi launch, and the two per-query loops -- the first stage and the full scoring of the
# shortlisted documents -- run as CUDA kernels over all queries at once.  What stays in Python per query is the dict
# bookkeeping that defines the orders (rare / frequent split, stable sorts by score) and building the result dicts.
# ------------------------------------------------------------------------------------------------
import inspect as _inspect
import time as _time

_AGG_DEFAULTS = {n: q.default for n, q in _inspect.signature(aggregate_evidence).parameters.items()
                 if n not in ("ngrams_and_scores", "unigram_scores", "index")}

_PY_ERRORS = {"math domain error": ValueError, "math range error": OverflowError,
              "0.0 cannot be raised to a negative power": ZeroDivisionError}


def _evcheck_py(code):
    """Native scalar scoring: the exception Python's own arithmetic raises, else SealB200Error."""
    if code != 0:
        msg = lib.sealev_last_error().decode(errors="replace")
        if msg in _PY_ERRORS:
            raise _PY_ERRORS[msg](msg)
        _evcheck(code)


def _i64(x):
    return np.ascontiguousarray(x, dtype=np.int64) if len(x) else np.zeros(1, dtype=np.int64)


def _f64(x):
    return np.ascontiguousarray(x, dtype=np.float64) if len(x) else np.zeros(1)


def batch_aggregate_evidence(list_of_ngrams_and_scores, list_of_unigram_scores=None, index=None, **kw):
    """aggregate_evidence for a batch of queries: a list of (results, all_ngrams), element q equal (same document
    order, key order, dict order and floats) to aggregate_evidence(list_of_ngrams_and_scores[q],
    list_of_unigram_scores[q], index, **kw).  `kw` takes aggregate_evidence's keywords, with its defaults.  Key
    scores are read with float()."""
    bad = sorted(set(kw) - set(_AGG_DEFAULTS))
    if bad:
        raise TypeError(f"batch_aggregate_evidence() got an unexpected keyword argument {bad[0]!r}")
    return _batch_evidence(list(list_of_ngrams_and_scores), list_of_unigram_scores, index, {**_AGG_DEFAULTS, **kw})


def _batch_evidence(queries, unis, index, p, phases=None):
    t0 = _time.perf_counter()
    held = []                              # arrays whose addresses are passed to the native calls below

    def ptr(a):
        held.append(a)
        return a.ctypes.data

    Q = len(queries)
    if Q == 0:
        return []
    unis = [None] * Q if unis is None else list(unis)
    if len(unis) != Q:
        raise ValueError("list_of_unigram_scores must have one entry per query")
    from .index import SHIFT
    fmfreq = bool(p["use_fm_index_frequency"])
    ntokens = float(index.beginnings[-1])
    keys = [[((k.tolist() if hasattr(k, "tolist") else list(k)), float(s)) for k, s in q] for q in queries]
    cutoff = [0.0] * Q
    if not fmfreq:                                                                          # :198-205
        cutoff = [min(ks, key=lambda ks: ks[1])[1] - 0.1 if ks else [][0] for ks in keys]

    # -- unigram candidates: the first use_top_k_unigrams of the stable argsort, minus the given tokens ----------
    top_k = p["use_top_k_unigrams"]
    kept = [None] * Q                     # int64 arrays of kept tokens
    V = [-1] * Q
    uarr = [None] * Q                     # float64 unigram scores
    out_n = np.zeros(1, dtype=np.int64)
    for q, us in enumerate(unis):
        if us is None:
            continue
        a = uarr[q] = np.ascontiguousarray(us, dtype=np.float64)
        v = V[q] = len(a)
        g = np.fromiter({0, 1, 2} | {k[0] for k, _ in keys[q] if len(k) == 1}, dtype=np.int64)   # :207-211
        goff = np.array([0, len(g)], dtype=np.int64)
        kk = v if top_k is None else (min(top_k, v) if top_k >= 0 else max(v + top_k, 0))
        out = np.zeros(max(kk, 1), dtype=np.int64)
        _evcheck_py(lib.sealev_unigram_topk(1, v, a.ctypes.data if v else None, v if top_k is None else int(top_k),
                                            goff.ctypes.data, ptr(_i64(g)), out.ctypes.data, out_n.ctypes.data))
        kept[q] = out[:out_n[0]]

    # -- every distinct SA range of the batch in one launch: multi-token keys by tuple, single tokens by value ------
    multi = {}
    singles = []
    for ks in keys:
        for k, _ in ks:
            if len(k) == 1:
                singles.append(k[0])
            else:
                multi.setdefault(tuple(k), len(multi))
    uniq = np.unique(np.concatenate([np.asarray(singles, dtype=np.int64)] + [a for a in kept if a is not None]))
    seqs_multi = list(multi)
    lens = np.concatenate([np.fromiter((len(s) for s in seqs_multi), dtype=np.int64, count=len(seqs_multi)),
                           np.ones(len(uniq), dtype=np.int64)])
    nseq = len(lens)
    t1 = _time.perf_counter()
    lo_m = hi_m = lo_u = hi_u = np.zeros(0, dtype=np.int64)
    if nseq:
        offs = np.zeros(nseq + 1, dtype=np.uint64); np.cumsum(lens, out=offs[1:])
        flat = np.concatenate([np.fromiter((t + SHIFT for s in seqs_multi for t in s), dtype=np.int64,
                                           count=int(lens[:len(seqs_multi)].sum())), uniq + SHIFT]).astype(np.uint64)
        if len(flat) == 0:
            flat = np.zeros(1, dtype=np.uint64)
        lo = np.zeros(nseq, dtype=np.uint64); hi = np.zeros(nseq, dtype=np.uint64)
        check(lib.sealfm_backward_search_multi(index._dev(), nseq, flat.ctypes.data, offs.ctypes.data,
                                               lo.ctypes.data, hi.ctypes.data))
        lo = lo.astype(np.int64); hi = hi.astype(np.int64)
        lo_m, hi_m, lo_u, hi_u = lo[:len(multi)], hi[:len(multi)], lo[len(multi):], hi[len(multi):]
    t2 = _time.perf_counter()
    lo_m, hi_m = lo_m.tolist(), hi_m.tolist()

    def ranges_of(ks):                     # (lo, hi) of each key of a list
        sing = np.asarray([k[0] for k, _ in ks if len(k) == 1], dtype=np.int64)
        at = np.searchsorted(uniq, sing)
        sl, sh = lo_u[at].tolist(), hi_u[at].tolist()
        out, i = [], 0
        for k, _ in ks:
            if len(k) == 1:
                out.append((sl[i], sh[i])); i += 1
            else:
                j = multi[tuple(k)]; out.append((lo_m[j], hi_m[j]))
        return out

    # -- scalar scoring of every key of the batch ----------------------------------------------------------------
    rng = [ranges_of(ks) for ks in keys]
    flat_keys = [(q, k, s, r) for q, ks in enumerate(keys) for (k, s), r in zip(ks, rng[q])]
    n = len(flat_keys)
    sr = _f64([s for _, _, s, _ in flat_keys]); cnt = _i64([r[1] - r[0] for _, _, _, r in flat_keys])
    kl = _i64([len(k) for _, k, _, _ in flat_keys]); co = _f64([cutoff[q] for q, _, _, _ in flat_keys])
    ksc = np.zeros(max(n, 1))
    _evcheck_py(lib.sealev_key_scores(n, sr.ctypes.data, cnt.ctypes.data, kl.ctypes.data, co.ctypes.data, ntokens,
                                      float(p["alpha"]), float(p["length_penalty"]), float(p["smoothing"]), int(fmfreq),
                                      ksc.ctypes.data))
    ksc = ksc[:n].tolist()
    # unigram tables (nonzero entries) and the add_best_unigrams_to_ngrams extras
    uq = [q for q in range(Q) if kept[q] is not None]
    tab = [None] * Q
    extras = [[] for _ in range(Q)]
    if uq:
        ut = np.concatenate([kept[q] for q in uq]) if uq else np.zeros(0, dtype=np.int64)
        at = np.searchsorted(uniq, ut)
        uc = _i64(hi_u[at] - lo_u[at]) if len(ut) else _i64([])
        us = _f64(np.concatenate([uarr[q][kept[q]] for q in uq]))
        uco = _f64(np.concatenate([np.full(len(kept[q]), cutoff[q]) for q in uq]))
        uv = np.zeros(max(len(ut), 1))
        _evcheck_py(lib.sealev_unigram_scores(len(ut), us.ctypes.data, uc.ctypes.data, uco.ctypes.data, ntokens,
                                              float(p["alpha"]), float(p["smoothing"]), int(fmfreq), uv.ctypes.data))
        uv = uv[:len(ut)]
        o = 0
        toff = [0]
        for q in uq:
            m = len(kept[q]); t, v = kept[q], uv[o:o + m]; o += m
            nz = v != 0.0
            tab[q] = (t[nz], v[nz])
            toff.append(toff[-1] + int(nz.sum()))
        if p["add_best_unigrams_to_ngrams"]:                                                # :274-278
            tt = _i64(np.concatenate([tab[q][0] for q in uq])); tv = _f64(np.concatenate([tab[q][1] for q in uq]))
            nx = _i64([len(keys[q]) for q in uq]); vv = _i64([V[q] for q in uq])
            cap = int(sum(min(len(keys[q]), V[q]) for q in uq))
            xo = np.zeros(len(uq) + 1, dtype=np.int64); xt = np.zeros(max(cap, 1), dtype=np.int64); xv = np.zeros(max(cap, 1))
            _evcheck_py(lib.sealev_best_unigrams(len(uq), vv.ctypes.data, ptr(_i64(toff)), tt.ctypes.data,
                                                 tv.ctypes.data, nx.ctypes.data, xo.ctypes.data, xt.ctypes.data,
                                                 xv.ctypes.data, cap))
            xt, xv, xo = xt.tolist(), xv.tolist(), xo.tolist()
            for i, q in enumerate(uq):
                extras[q] = list(zip(xt[xo[i]:xo[i + 1]], xv[xo[i]:xo[i + 1]]))

    # -- per query: rare / frequent split and all_ngrams, in the reference's dict and sort orders (:280-314) ------
    mo1, mo2 = p["max_occurrences_1"], p["max_occurrences_2"]
    by_score = lambda kv: kv[1]
    uni_at = {}                            # token -> (lo, hi) of the tokens extras can add with a nonzero score
    fs_tok, fs_off, fs_score, fs_count, fs_lo, fs_rows, fs_q = [], [0], [], [], [], [], [0]
    sc_tok, sc_off, sc_score, sc_count, sc_q = [], [0], [], [], [0]
    all_ng, scored_q, empty_count = [], [], []
    i_key = 0
    for q in range(Q):
        ks = keys[q]
        scores = ksc[i_key:i_key + len(ks)]; i_key += len(ks)
        rq = rng[q]
        items = [(tuple(k), sc, r) for (k, _), sc, r in zip(ks, scores, rq)]
        if extras[q]:
            ex = [t for t, v in extras[q] if v != 0.0]
            if ex:
                at = np.searchsorted(uniq, np.asarray(ex, dtype=np.int64))
                for t, l, h in zip(ex, lo_u[at].tolist(), hi_u[at].tolist()):
                    uni_at[t] = (l, h)
            items += [((t,), v, uni_at.get(t) if v != 0.0 else None) for t, v in extras[q]]
        counts = {(): len(index)}
        for k, _, r in items:
            if r is not None:
                counts[k] = r[1] - r[0]
        rare, freq, rr = {}, {}, {}
        for k, sc, r in items:
            if sc == 0.0:
                continue
            c = r[1] - r[0]
            if c > mo2:
                continue
            (freq if (c > mo1 or sc < 0.0) else rare)[k] = sc
            rr[k] = r
        rare = dict(sorted(rare.items(), key=by_score, reverse=True))
        freq = dict(sorted(freq.items(), key=by_score, reverse=True))
        all_ngrams = dict(sorted(list(rare.items()) + list(freq.items()), key=by_score, reverse=True))
        all_ng.append(all_ngrams)
        empty_count.append(int(counts[()]))
        for k, sc in rare.items():
            l, h = rr[k]
            fs_tok.extend(k); fs_off.append(len(fs_tok)); fs_score.append(sc); fs_count.append(counts[k])
            fs_lo.append(l); fs_rows.append(max(0, min(h, l + mo1) - l))
        fs_q.append(len(fs_score))
        scored = [(k, v) for k, v in all_ngrams.items() if len(k) >= 1 and v > 0.0]        # trie contents, :378-385
        scored_q.append(scored)
        for k, v in scored:
            sc_tok.extend(k); sc_off.append(len(sc_tok)); sc_score.append(v); sc_count.append(counts[k])
        sc_q.append(len(sc_score))
    t3 = _time.perf_counter()

    # -- GPU first stage ---------------------------------------------------------------------------------------
    h = index._dev()
    sort_mode = 1 if p["sort_by_length"] else (2 if p["sort_by_freq"] else 0)
    ec = _i64(empty_count)
    nd_max = int(p["n_docs_complete_score"])
    rows_q = [sum(fs_rows[fs_q[q]:fs_q[q + 1]]) for q in range(Q)]
    cap = sum(min(max(nd_max, 0), r) for r in rows_q)
    so = np.zeros(Q + 1, dtype=np.int64); sd = np.zeros(max(cap, 1), dtype=np.int64)
    _evcheck(lib.sealev_batch_first_stage(h, Q, ptr(_i64(fs_q)), ptr(_i64(fs_tok)), ptr(_i64(fs_off)),
                                          ptr(_f64(fs_score)), ptr(_i64(fs_count)),
                                          ptr(np.ascontiguousarray(_i64(fs_lo), dtype=np.uint64)),
                                          ptr(_i64(fs_rows)), ec.ctypes.data, sort_mode, int(bool(p["allow_overlaps"])),
                                          float(p["beta"]), float(p["single_key"]), nd_max, so.ctypes.data, sd.ctypes.data, cap))
    fs_us = np.zeros(4)
    lib.sealev_batch_phase_us(fs_us.ctypes.data)
    t4 = _time.perf_counter()

    # -- GPU scoring of the shortlisted documents -----------------------------------------------------------------
    so_l = so.tolist()
    docs = sd[:so_l[-1]]
    b = np.asarray(index.beginnings, dtype=np.int64)
    dl = np.maximum(b[docs + 1] - b[docs], 1) if len(docs) else np.zeros(0, dtype=np.int64)
    tok_cap = int(dl.sum())
    uo, ut, uv = [0], [], []
    for q in range(Q):
        if tab[q] is not None:
            ut.append(tab[q][0]); uv.append(tab[q][1]); uo.append(uo[-1] + len(tab[q][0]))
        else:
            uo.append(uo[-1])
    ut = _i64(np.concatenate(ut) if ut else []); uv = _f64(np.concatenate(uv) if uv else [])
    nd = len(docs)
    dto = np.zeros(nd + 1, dtype=np.int64); dtok = np.zeros(max(tok_cap, 1), dtype=np.int64)
    out_score = np.zeros(max(nd, 1)); out_best = np.zeros(max(nd, 1), dtype=np.int64); out_bs = np.zeros(max(nd, 1))
    po = np.zeros(nd + 1, dtype=np.int64)
    need = C.c_int64(0)
    pcap = tok_cap * 2 + 16
    lib.sealev_set_sum_mode(1 if sys.version_info >= (3, 12) else 0)     # how this interpreter's sum() adds floats (:476)
    args_head = (h, Q, ptr(_i64(sc_q)), ptr(_i64(sc_tok)), ptr(_i64(sc_off)), ptr(_f64(sc_score)),
                 ptr(_i64(sc_count)), ec.ctypes.data, so.ctypes.data, ptr(_i64(docs)), ptr(_i64(uo)),
                 ut.ctypes.data, uv.ctypes.data, ptr(_i64(V)), SHIFT, sort_mode, int(bool(p["allow_overlaps"])),
                 int(bool(p["unigrams_ignore_free_places"])), int(bool(p["single_key_add_unigrams"])), float(p["beta"]),
                 float(p["single_key"]), dto.ctypes.data, dtok.ctypes.data, tok_cap, out_score.ctypes.data,
                 out_best.ctypes.data, out_bs.ctypes.data, po.ctypes.data)
    while True:
        pk = np.zeros(max(pcap, 1), dtype=np.int64); ps = np.zeros(max(pcap, 1))
        rc = lib.sealev_batch_score_docs(*args_head, pk.ctypes.data, ps.ctypes.data, pcap, C.byref(need))
        if rc == -6 and need.value > pcap:               # SEALFM_ECAPACITY: the exact count is known now
            pcap = need.value
            continue
        _evcheck(rc)
        break
    sc_us = np.zeros(4)
    lib.sealev_batch_phase_us(sc_us.ctypes.data)
    t5 = _time.perf_counter()

    # -- result dicts, as aggregate_evidence builds them ---------------------------------------------------------
    flat_tok = dtok[:int(dto[-1])].tolist(); dto = dto.tolist()
    n_pk = int(po[-1])
    pk, ps, po = pk[:n_pk].tolist(), ps[:n_pk].tolist(), po.tolist()
    osc, ob, obs = out_score.tolist(), out_best.tolist(), out_bs.tolist()
    docs = docs.tolist()
    out = []
    for q in range(Q):
        scored = scored_q[q]
        results = {}
        for i in range(so_l[q], so_l[q + 1]):
            picked = [((scored[k][0] if k >= 0 else (-1 - k,)), s) for k, s in zip(pk[po[i]:po[i + 1]], ps[po[i]:po[i + 1]])]
            bk = ob[i]
            best = [scored[bk][0], obs[i]] if bk >= 0 else [[], 0.0]
            results[docs[i]] = [osc[i], picked, None, flat_tok[dto[i]:dto[i + 1]], best]
        out.append((dict(sorted(results.items(), key=lambda kv: -kv[1][0])), all_ng[q]))   # :496-497
    t6 = _time.perf_counter()
    if phases is not None:
        for name, v in (("host_prep", (t1 - t0) + (t3 - t2)), ("ranges", t2 - t1), ("locate", fs_us[0] * 1e-6),
                        ("first_stage", fs_us[1] * 1e-6), ("extract", sc_us[2] * 1e-6), ("score", sc_us[3] * 1e-6),
                        ("python_assembly", (t4 - t3 - (fs_us[0] + fs_us[1]) * 1e-6) + (t5 - t4 - (sc_us[2] + sc_us[3]) * 1e-6) + (t6 - t5))):
            phases[name] = phases.get(name, 0.0) + v
    return out
