"""`seal_b200.compat.install()` registers this package under the reference's module names so that
unmodified SEAL callers (`from seal.index import FMIndex`, `from seal.beam_search import
fm_index_generate`, `from seal.cpp_modules.fm_index import load_FMIndex`) resolve to the H100 path.
See INTEGRATION.md."""
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
    sys.modules["seal.cpp_modules"] = cppm
    sys.modules["seal.cpp_modules.fm_index"] = fm_index
    return seal
