"""Batched evidence aggregation, host side: the native scalar scoring (include/sealev_batch.h) against
seal_b200.keys._Evidence bit for bit, and SEALSearcher.batch_retrieve_from_keys as seal_b200.compat installs it."""
import json
import math
import struct
import sys
import types

import numpy as np
import pytest

from seal_b200.synthetic import make_corpus
from test_evidence import _BatchedOracleIndex, load_gold


def bits(x):
    return struct.pack("<d", x)


def native_key_scores(sr, count, length, cutoff, ntokens, p):
    from seal_b200._lib import lib
    from seal_b200.keys import _evcheck_py
    n = len(sr)
    a = [np.ascontiguousarray(v, dtype=t) for v, t in ((sr, np.float64), (count, np.int64), (length, np.int64), (cutoff, np.float64))]
    out = np.zeros(max(n, 1))
    _evcheck_py(lib.sealev_key_scores(n, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, a[3].ctypes.data, ntokens,
                                      p["alpha"], p["length_penalty"], p["smoothing"], int(p["use_fm_index_frequency"]),
                                      out.ctypes.data))
    return out[:n].tolist()


def native_unigram_table(us, given, cutoff, counts_of, ntokens, p):
    """sealev_unigram_topk + sealev_unigram_scores -> the dense table _Evidence.unigram_table returns"""
    from seal_b200._lib import lib
    from seal_b200.keys import _evcheck_py
    V = len(us)
    mat = np.ascontiguousarray(us, dtype=np.float64)
    g = np.array(sorted(given), dtype=np.int64); goff = np.array([0, len(g)], dtype=np.int64)
    k = p["use_top_k_unigrams"]
    kk = min(k, V) if k >= 0 else max(V + k, 0)
    out = np.zeros(max(kk, 1), dtype=np.int64); n = np.zeros(1, dtype=np.int64)
    _evcheck_py(lib.sealev_unigram_topk(1, V, mat.ctypes.data, k, goff.ctypes.data, g.ctypes.data, out.ctypes.data, n.ctypes.data))
    kept = out[:n[0]]
    s = np.ascontiguousarray(mat[kept]); c = np.ascontiguousarray([counts_of(int(t)) for t in kept], dtype=np.int64)
    co = np.full(max(len(kept), 1), cutoff if cutoff is not None else 0.0)
    val = np.zeros(max(len(kept), 1))
    _evcheck_py(lib.sealev_unigram_scores(len(kept), s.ctypes.data, c.ctypes.data, co.ctypes.data, ntokens, p["alpha"],
                                          p["smoothing"], int(p["use_fm_index_frequency"]), val.ctypes.data))
    table = [0.0] * V
    for t, v in zip(kept.tolist(), val[:len(kept)].tolist()):
        if v != 0.0:
            table[t] = v
    return table


def _params(kw):
    from seal_b200.keys import _AGG_DEFAULTS
    p = {**_AGG_DEFAULTS, **kw}
    return dict(alpha=float(p["alpha"]), beta=p["beta"], length_penalty=float(p["length_penalty"]), smoothing=float(p["smoothing"]),
                use_fm_index_frequency=p["use_fm_index_frequency"], use_top_k_unigrams=p["use_top_k_unigrams"])


@pytest.fixture(scope="module")
def gold_index():
    from oracle.fm_oracle import OracleIndex
    g = load_gold()
    return _BatchedOracleIndex(OracleIndex([list(map(int, d)) for d in make_corpus(**g["corpus"])]))


@pytest.mark.parametrize("case", range(len(load_gold()["cases"])))
def test_native_scalar_scoring_matches_python_on_golden_cases(case, gold_index):
    from seal_b200.keys import _Evidence
    c = load_gold()["cases"][case]
    p = _params(c["kw"])
    ev = _Evidence(gold_index, p)
    keys = [(list(k), s) for k, s in c["keys"]]
    cutoff = (min(s for _, s in keys) - 0.1) if (keys and not p["use_fm_index_frequency"]) else None
    ev.need_ranges([k for k, _ in keys])
    exp = [ev.key_score(k, s, cutoff) for k, s in keys]
    got = native_key_scores([s for _, s in keys], [ev.count(k) for k, _ in keys], [len(k) for k, _ in keys],
                            [cutoff or 0.0] * len(keys), ev.ntokens, p)
    assert [bits(x) for x in got] == [bits(x) for x in exp]
    if c["unigram_scores"] is not None:
        given = {0, 1, 2} | {k[0] for k, _ in keys if len(k) == 1}
        exp_t = ev.unigram_table(c["unigram_scores"], given, cutoff)
        ev.need_ranges([(t,) for t in range(len(c["unigram_scores"]))])
        got_t = native_unigram_table(c["unigram_scores"], given, cutoff, lambda t: ev.count((t,)), ev.ntokens, p)
        assert [bits(x) for x in got_t] == [bits(x) for x in exp_t]


def test_native_scalar_scoring_fuzz_near_the_log1mexp_edge():
    """Scores a hair below 0 (1 - exp(sr) near 0), counts up to the corpus size (1 - exp(snr) near 0), every length
    penalty / alpha / smoothing combination: same bits as _Evidence, or the same exception."""
    from seal_b200.keys import _Evidence

    class _Idx:
        beginnings = [0, 1_000_003]

    rng = np.random.default_rng(5)
    checked = raised = 0
    for trial in range(400):
        p = dict(alpha=float(rng.choice([0.5, 1.0, 2.0, 3.0])), beta=0.8, length_penalty=float(rng.choice([0.0, 0.1, 0.5, -0.2])),
                 smoothing=float(rng.choice([0.0, 5.0, 1e-3])), use_fm_index_frequency=bool(rng.random() < 0.8),
                 use_top_k_unigrams=1000)
        ev = _Evidence(_Idx(), p)
        n = 64
        sr = np.concatenate([-10.0 ** rng.uniform(-17, -1, n // 2), -rng.exponential(3.0, n // 4), rng.uniform(-1e-9, 1e-9, n // 4)])
        cnt = rng.choice([0, 1, 2, 17, 999_999, 1_000_002, 1_000_003, 1_000_010], n)
        length = rng.integers(0, 12, n)
        cutoff = float(sr.min() - 0.1)
        for s, c, L in zip(sr.tolist(), cnt.tolist(), length.tolist()):
            key = tuple(range(L))
            ev.range_of[key] = (0, c)
            try:
                e = ev.key_score(list(key), s, cutoff)
            except (ValueError, OverflowError, ZeroDivisionError) as err:
                with pytest.raises(type(err)):
                    native_key_scores([s], [c], [L], [cutoff], ev.ntokens, p)
                raised += 1
                continue
            assert bits(native_key_scores([s], [c], [L], [cutoff], ev.ntokens, p)[0]) == bits(e), (s, c, L, p)
            checked += 1
        us = list(np.concatenate([-10.0 ** rng.uniform(-17, -1, 40), -rng.exponential(3.0, 40)]))
        us[3] = us[5] = us[7]                                    # ties keep the lower token id first
        counts = {t: int(rng.choice([0, 1, 50, 1_000_003])) for t in range(len(us))}
        for t, c in counts.items():
            ev.range_of[(t,)] = (0, c)
        given = {0, 1, 2, 9}
        p["use_top_k_unigrams"] = int(rng.choice([5, 30, 1000, -3]))
        try:
            exp_t = ev.unigram_table(us, given, cutoff)
        except (ValueError, OverflowError) as err:
            with pytest.raises(type(err)):
                native_unigram_table(us, given, cutoff, counts.__getitem__, ev.ntokens, p)
            continue
        got_t = native_unigram_table(us, given, cutoff, counts.__getitem__, ev.ntokens, p)
        assert [bits(x) for x in got_t] == [bits(x) for x in exp_t]
    assert checked > 10_000 and raised > 0


def test_native_best_unigrams_match_python_sort():
    from seal_b200._lib import lib
    rng = np.random.default_rng(2)
    for trial in range(50):
        V = int(rng.integers(1, 60))
        table = [0.0] * V
        for t in rng.choice(V, int(rng.integers(0, V + 1)), replace=False).tolist():
            table[t] = float(rng.choice([0.5, 1.25, 3.0]))              # ties among the nonzero entries
        m = int(rng.integers(0, 2 * V))
        exp = sorted(range(V), key=lambda t: -table[t])[:m]
        nz = [t for t in range(V) if table[t] != 0.0]
        tt = np.array(nz or [0], dtype=np.int64); tv = np.array([table[t] for t in nz] or [0.0])
        toff = np.array([0, len(nz)], dtype=np.int64); vv = np.array([V], dtype=np.int64); nx = np.array([m], dtype=np.int64)
        xo = np.zeros(2, dtype=np.int64); xt = np.zeros(max(m, 1), dtype=np.int64); xv = np.zeros(max(m, 1))
        assert lib.sealev_best_unigrams(1, vv.ctypes.data, toff.ctypes.data, tt.ctypes.data, tv.ctypes.data, nx.ctypes.data,
                                        xo.ctypes.data, xt.ctypes.data, xv.ctypes.data, m) == 0
        assert xt[:xo[1]].tolist() == exp
        assert xv[:xo[1]].tolist() == [table[t] for t in exp]


# ---- SEALSearcher.batch_retrieve_from_keys under seal_b200.compat ------------------------------------------------

class _StandInSearcher:
    """The attribute and method names of seal.retrieval.SEALSearcher that retrieval reads (seal/retrieval.py:399-760)."""

    def __init__(self, jobs, batch_size):
        self.jobs, self.batch_size, self.fm_index = jobs, batch_size, object()
        self.max_hits, self.fully_score, self.score_exponent, self.repetition_penalty = 1500, 1500, 2.0, 0.8
        self.scoring_length_penalty, self.use_fm_index_frequency, self.add_best_unigrams_to_ngrams = 0.25, True, True
        self.use_top_k_ngrams, self.sort_by_length, self.sort_by_freq, self.smoothing = 5000, False, True, 5.0
        self.allow_overlaps, self.single_key, self.unigrams_ignore_free_places = False, 0.5, True

    def batch_retrieve_from_keys(self, keys):
        raise AssertionError("the reference method should have been replaced")

    def _mp_batch_retrieve_from_keys(self, keys):
        raise AssertionError("forks a process pool")


@pytest.fixture
def installed(monkeypatch):
    saved = {k: v for k, v in sys.modules.items() if k == "seal" or k.startswith("seal.")}
    seal = types.ModuleType("seal"); seal.__path__ = []
    retrieval = types.ModuleType("seal.retrieval"); retrieval.SEALSearcher = _StandInSearcher
    for k in saved:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.setitem(sys.modules, "seal", seal)
    monkeypatch.setitem(sys.modules, "seal.retrieval", retrieval)
    orig = _StandInSearcher.batch_retrieve_from_keys
    import multiprocessing
    import multiprocessing.pool

    def no_pool(*a, **k):
        raise AssertionError("multiprocessing used")
    monkeypatch.setattr(multiprocessing, "Pool", no_pool)
    monkeypatch.setattr(multiprocessing.pool, "Pool", no_pool)
    from seal_b200 import compat
    compat.install()
    calls = []

    def fake_batch(ngs, unis, index=None, **kw):
        calls.append((list(ngs), list(unis), index, kw))
        return [(("results", json.dumps(k)), ("ngrams", u)) for k, u in zip(ngs, unis)]
    import seal_b200.keys as sk
    monkeypatch.setattr(sk, "batch_aggregate_evidence", fake_batch)
    yield calls
    _StandInSearcher.batch_retrieve_from_keys = orig
    for k in [k for k in sys.modules if k == "seal" or k.startswith("seal.")]:
        del sys.modules[k]
    sys.modules.update(saved)


@pytest.mark.parametrize("jobs", [1, 75])
def test_compat_batch_retrieve_in_process_in_chunks(installed, jobs):
    from seal_b200.compat import batch_retrieve_from_keys
    assert _StandInSearcher.batch_retrieve_from_keys is batch_retrieve_from_keys
    s = _StandInSearcher(jobs=jobs, batch_size=3)
    inputs = []
    for q in range(8):                                           # the four input forms retrieve_from_keys accepts
        kk = [([q, q + 1], -1.0 - q)]
        inputs.append([kk, (kk,), (kk, [0.0, -float(q)]), (kk, [-1.0], ["doc"])][q % 4])
    gen = s.batch_retrieve_from_keys(iter(inputs))
    assert installed == []                                        # lazy: nothing runs before the first next()
    out = list(gen)
    assert len(out) == 8
    for q, (res, ng) in enumerate(out):                          # one (results, ngrams) per query, in order
        assert res == ("results", json.dumps([([q, q + 1], -1.0 - q)]).replace("(", "[").replace(")", "]"))
        assert ng == ("ngrams", [None, None, [0.0, -float(q)], [-1.0]][q % 4])
    assert [len(c[0]) for c in installed] == [3, 3, 2]           # chunks of self.batch_size
    for _, _, index, kw in installed:
        assert index is s.fm_index
        assert kw == dict(max_occurrences_1=1500, n_docs_complete_score=1500, alpha=2.0, beta=0.8, length_penalty=0.25,
                          use_fm_index_frequency=True, add_best_unigrams_to_ngrams=True, use_top_k_unigrams=5000,
                          sort_by_length=False, sort_by_freq=True, smoothing=5.0, allow_overlaps=False, single_key=0.5,
                          unigrams_ignore_free_places=True)


def test_batch_aggregate_evidence_rejects_unknown_keywords():
    from seal_b200.keys import batch_aggregate_evidence, _AGG_DEFAULTS
    with pytest.raises(TypeError):
        batch_aggregate_evidence([[]], None, None, not_a_keyword=1)
    assert _AGG_DEFAULTS["max_occurrences_2"] == 10_000_000 and _AGG_DEFAULTS["single_key_add_unigrams"] is False
    assert math.isclose(_AGG_DEFAULTS["beta"], 0.8)
