"""`seal_b200.compat.install()` registers this package under the reference's module names so that
unmodified SEAL callers (`from seal.index import FMIndex`, `from seal.beam_search import
fm_index_generate`, `from seal.cpp_modules.fm_index import load_FMIndex`) resolve to the H100 path.
See INTEGRATION.md."""
import importlib
import itertools
import sys
import types


def install():
    from . import index, beam_search, keys
    from .cpp_modules import fm_index
    import seal_b200.cpp_modules as cppm
    seal = sys.modules.get("seal") or types.ModuleType("seal")
    seal.FMIndex = index.FMIndex
    seal.fm_index_generate = beam_search.fm_index_generate
    seal.IndexBasedLogitsProcessor = beam_search.IndexBasedLogitsProcessor
    sys.modules["seal"] = seal
    sys.modules["seal.index"] = index
    sys.modules["seal.beam_search"] = beam_search
    # seal.keys: the decoder-side helpers and the evidence aggregation are replaced in place when the
    # reference module is importable (its remaining helpers -- deduplicate, decompose_query_into_keys --
    # stay the reference's own)
    ref_keys = sys.modules.get("seal.keys")
    if ref_keys is not None:
        ref_keys.rescore_keys = keys.rescore_keys
        ref_keys.compute_unigram_scores = keys.compute_unigram_scores
        ref_keys.aggregate_evidence = keys.aggregate_evidence
    # seal.retrieval: SEALSearcher aggregates the evidence of a whole chunk of queries in one batched call, in this
    # process, for every `jobs` value (the reference forks a multiprocessing pool for jobs >= 2, and device state does
    # not survive fork())
    ref_retrieval = sys.modules.get("seal.retrieval")
    if ref_retrieval is None and hasattr(seal, "__path__"):
        try:
            ref_retrieval = importlib.import_module("seal.retrieval")
        except ImportError:
            ref_retrieval = None
    if ref_retrieval is not None and hasattr(ref_retrieval, "SEALSearcher"):
        ref_retrieval.SEALSearcher.batch_retrieve_from_keys = batch_retrieve_from_keys
    sys.modules["seal.cpp_modules"] = cppm
    sys.modules["seal.cpp_modules.fm_index"] = fm_index
    return seal


def _split_keys(keys):
    """SEALSearcher.retrieve_from_keys's input forms (seal/retrieval.py:720-729): keys, (keys,), (keys, unigram
    scores) or (keys, unigram scores, added documents) -> (keys, unigram scores)."""
    if isinstance(keys, tuple) and len(keys) == 1:
        return keys[0], None
    if isinstance(keys, tuple) and len(keys) == 2:
        return keys
    if isinstance(keys, tuple) and len(keys) == 3:
        return keys[0], keys[1]
    return keys, None


def batch_retrieve_from_keys(self, keys):
    """SEALSearcher.batch_retrieve_from_keys (seal/retrieval.py:756-760) without a process pool: takes the key
    generator in chunks of self.batch_size and yields (results, ngrams) per query, in order, each equal to what
    self.retrieve_from_keys returns for it -- same arguments to the aggregation, run by
    seal_b200.keys.batch_aggregate_evidence for the whole chunk."""
    from . import keys as _keys
    it = iter(keys)
    size = max(int(getattr(self, "batch_size", 1) or 1), 1)
    while True:
        chunk = [_split_keys(k) for k in itertools.islice(it, size)]
        if not chunk:
            return
        yield from _keys.batch_aggregate_evidence(
            [k for k, _ in chunk], [u for _, u in chunk], index=self.fm_index,
            max_occurrences_1=self.max_hits,
            n_docs_complete_score=self.fully_score,
            alpha=self.score_exponent,
            beta=self.repetition_penalty,
            length_penalty=self.scoring_length_penalty,
            use_fm_index_frequency=self.use_fm_index_frequency,
            add_best_unigrams_to_ngrams=self.add_best_unigrams_to_ngrams,
            use_top_k_unigrams=self.use_top_k_ngrams,
            sort_by_length=self.sort_by_length,
            sort_by_freq=self.sort_by_freq,
            smoothing=self.smoothing,
            allow_overlaps=self.allow_overlaps,
            single_key=self.single_key,
            unigrams_ignore_free_places=self.unigrams_ignore_free_places)
