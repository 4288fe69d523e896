"""batch_aggregate_evidence on the GPU: every query's (results, all_ngrams) equals aggregate_evidence's for that query
alone -- same document order, key order, dict order, floats (==) and token lists -- for every keyword variant, at
batch sizes 1 to 1 000, across chunk boundaries, and on the edge cases of the decomposition."""
import json

import numpy as np
import pytest

from seal_b200.synthetic import make_corpus
from test_evidence import flatten, load_gold

pytestmark = pytest.mark.gpu

SEARCHER = dict(max_occurrences_1=1500, n_docs_complete_score=1500, use_top_k_unigrams=5000, add_best_unigrams_to_ngrams=True)


def per_query(keys, unis, index, **kw):
    from seal_b200.keys import aggregate_evidence
    return [aggregate_evidence(k, u, index, **kw) for k, u in zip(keys, unis)]


def check_equal(got, exp):
    assert len(got) == len(exp)
    for q, ((gr, ga), (er, ea)) in enumerate(zip(got, exp)):
        assert list(ga.items()) == list(ea.items()), q
        assert list(gr) == list(er), q                     # document order
        assert gr == er, q                                 # every float, key order, token list, best key


@pytest.fixture(scope="module")
def corpus():
    from seal_b200.index import FMIndex
    docs = make_corpus(n_docs=4000, doc_len=40, n_phrases=3000, seed=9, vocab=3000)
    seqs = [list(map(int, d)) for d in docs]
    rep = [7, 8] * 30 + [7] * 40 + [9, 9, 9, 10] * 10         # a highly repetitive document (last one)
    seqs.append(rep)
    idx = FMIndex(); idx.initialize(seqs)
    return np.asarray(docs), idx


def make_batch(docs, n_queries, seed, n_keys=60, with_uni=0.8, vocab=3000):
    rng = np.random.default_rng(seed)
    keys, unis = [], []
    for q in range(n_queries):
        kk = []
        for _ in range(int(rng.integers(0, n_keys + 1))):
            d = int(rng.integers(0, docs.shape[0])); L = int(rng.integers(1, 9)); a = int(rng.integers(0, docs.shape[1] - L))
            k = docs[d, a:a + L].astype(np.int64).tolist()
            if rng.random() < 0.05:
                k[-1] = int(rng.integers(4, vocab))           # mostly zero-count keys
            kk.append((k, float(-rng.exponential(4.0) - 0.01)))
        if rng.random() < 0.2:
            kk.append(([11, 12, 13], -0.5))                    # the same key in many queries
        keys.append(kk)
        if rng.random() < with_uni:
            z = rng.standard_normal(vocab) * 3.0
            unis.append((z - np.log(np.exp(z).sum())).tolist())
        else:
            unis.append(None)
    return keys, unis


def test_golden_cases_as_batches():
    """Every keys_golden.json case; cases that share keywords run as one batch."""
    from seal_b200.index import FMIndex
    from seal_b200.keys import batch_aggregate_evidence
    g = load_gold()
    idx = FMIndex(); idx.initialize([list(map(int, d)) for d in make_corpus(**g["corpus"])])
    groups = {}
    for c in g["cases"]:
        groups.setdefault(json.dumps(c["kw"], sort_keys=True), []).append(c)
    for kw, cases in groups.items():
        out = batch_aggregate_evidence([[(list(k), s) for k, s in c["keys"]] for c in cases],
                                       [c["unigram_scores"] for c in cases], idx, **json.loads(kw))
        for c, (res, alln) in zip(cases, out):
            got_r, got_a = flatten(res, alln)
            assert got_a == c["all_ngrams"], c["name"]
            assert got_r == c["results"], c["name"]


VARIANTS = [dict(), dict(sort_by_length=True), dict(sort_by_freq=True), dict(allow_overlaps=True),
            dict(single_key=0.5), dict(single_key=1.0, single_key_add_unigrams=True), dict(unigrams_ignore_free_places=True),
            dict(use_fm_index_frequency=False), dict(add_best_unigrams_to_ngrams=True), dict(max_occurrences_1=1),
            dict(max_occurrences_1=25), dict(max_occurrences_1=1500), dict(n_docs_complete_score=0),
            dict(n_docs_complete_score=1), dict(n_docs_complete_score=1500), SEARCHER,
            dict(SEARCHER, allow_overlaps=True, sort_by_length=True, single_key=0.3)]


@pytest.mark.parametrize("kw", VARIANTS, ids=[json.dumps(v, sort_keys=True) for v in VARIANTS])
def test_batch_equals_per_query_every_keyword(corpus, kw):
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    keys, unis = make_batch(docs, 24, seed=len(json.dumps(kw, sort_keys=True)))
    keys[0] = []                                               # a query without keys
    keys[1] = [([2999, 2998, 2997, 2996], -0.3)]               # only zero-count keys
    if kw.get("use_fm_index_frequency", True) is False:
        # the reference raises IndexError for a query without keys here (its cutoff is min() of no scores)
        with pytest.raises(IndexError):
            per_query(keys[:1], unis[:1], idx, **kw)
        with pytest.raises(IndexError):
            batch_aggregate_evidence(keys, unis, idx, **kw)
        keys[0] = [([11, 12], -1.5)]
    check_equal(batch_aggregate_evidence(keys, unis, idx, **kw), per_query(keys, unis, idx, **kw))


@pytest.mark.parametrize("compensated", [0, 1])
def test_both_sum_modes(corpus, compensated, monkeypatch):
    import sys
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    monkeypatch.setattr(sys, "version_info", (3, 12) if compensated else (3, 11))
    keys, unis = make_batch(docs, 16, seed=40 + compensated)
    check_equal(batch_aggregate_evidence(keys, unis, idx, **SEARCHER), per_query(keys, unis, idx, **SEARCHER))


@pytest.mark.parametrize("n", [1, 2, 20, 137, 1000])
def test_batch_sizes(corpus, n):
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    keys, unis = make_batch(docs, n, seed=n, n_keys=30 if n == 1000 else 60)
    check_equal(batch_aggregate_evidence(keys, unis, idx, **SEARCHER), per_query(keys, unis, idx, **SEARCHER))


def test_repetitive_document_long_components_and_self_overlap(corpus):
    """Keys inside the repetitive document: self-overlapping occurrences (7 8 7, 9 9) form long overlap components."""
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    keys = [[([7, 8], -0.5), ([8, 7], -0.6), ([7, 8, 7], -0.7), ([7], -1.0), ([7, 7, 7], -0.4), ([9, 9], -0.2),
             ([9, 9, 10], -0.3), ([7, 8, 7, 8, 7, 8], -0.1)],
            [([7, 7], -0.5), ([9], -2.0), ([10, 9, 9, 9], -0.3)]]
    for kw in (dict(), dict(allow_overlaps=True), dict(sort_by_length=True, single_key=0.4), SEARCHER):
        check_equal(batch_aggregate_evidence(keys, [None, None], idx, **kw), per_query(keys, [None, None], idx, **kw))


def test_keys_in_no_shortlisted_document(corpus):
    """A shortlist of one document: most keys (rare and frequent) occur in no scored document."""
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    keys, unis = make_batch(docs, 8, seed=5)
    kw = dict(n_docs_complete_score=1, max_occurrences_1=3)
    check_equal(batch_aggregate_evidence(keys, unis, idx, **kw), per_query(keys, unis, idx, **kw))


def test_picks_beyond_the_first_capacity_guess(corpus):
    """allow_overlaps picks every distinct key of a document: 500 substrings of one 40-token document exceed the
    first pick-buffer guess (2 x tokens + 16)."""
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    d = docs[17].astype(np.int64).tolist()
    subs = list(dict.fromkeys(tuple(d[a:b]) for a in range(len(d)) for b in range(a + 1, min(len(d), a + 12) + 1)))[:500]
    keys = [[(list(k), -1.0 - 0.001 * i) for i, k in enumerate(subs)]]
    kw = dict(allow_overlaps=True, n_docs_complete_score=1)
    got = batch_aggregate_evidence(keys, [None], idx, **kw)
    check_equal(got, per_query(keys, [None], idx, **kw))
    assert sum(len(v[1]) for v in got[0][0].values()) > 2 * 40 + 16


def test_forced_chunking_equals_one_chunk(corpus):
    from seal_b200._lib import lib
    from seal_b200.keys import batch_aggregate_evidence
    docs, idx = corpus
    keys, unis = make_batch(docs, 40, seed=8)
    whole = batch_aggregate_evidence(keys, unis, idx, **SEARCHER)
    try:
        lib.sealev_set_device_budget(1 << 16)                   # a few queries per chunk in both stages
        chunked = batch_aggregate_evidence(keys, unis, idx, **SEARCHER)
    finally:
        lib.sealev_set_device_budget(0)
    check_equal(chunked, whole)
    check_equal(whole, per_query(keys, unis, idx, **SEARCHER))


def test_searcher_defaults_on_real_decode_records(corpus):
    """Keys as SEALSearcher gets them: beam-15, length-10 constrained decode records of a small BART on this corpus,
    unigram scores from compute_unigram_scores; aggregated at SEALSearcher's defaults."""
    from oracle.decode_oracle import make_bart
    from seal_b200.beam_search import generate_records
    from seal_b200.keys import batch_aggregate_evidence, compute_unigram_scores
    docs, idx = corpus
    model = make_bart(seed=0, layers=2, vocab=3000, d_model=128)
    rng = np.random.default_rng(1)
    ids = rng.integers(4, 3000, size=(12, 10)).astype(np.int64); ids[:, 0] = 0; ids[:, -1] = 2
    mask = np.ones_like(ids)
    rec = generate_records(model, idx, ids, mask, min_length=10, max_length=10, length_penalty=0.0, num_beams=15,
                           forced_bos_token_id=None)
    keys = []
    for q in range(ids.shape[0]):
        best = {}
        for h in np.flatnonzero(rec["valid"][q]):
            k = tuple(int(t) for t in rec["tokens"][q, h, :rec["lens"][q, h]] if t > 2)
            if k:
                best[k] = max(best.get(k, -np.inf), float(rec["scores"][q, h]))
        keys.append([(list(k), s) for k, s in best.items()])
    assert sum(len(k) for k in keys) > 100
    unis = compute_unigram_scores(model, ids)
    check_equal(batch_aggregate_evidence(keys, unis, idx, **SEARCHER), per_query(keys, unis, idx, **SEARCHER))
