"""seal_b200 — H100-native constrained beam-search decode for SEAL.

Mirrors ``seal/__init__.py:7-9`` for the hot path: ``FMIndex``, ``fm_index_generate``,
``IndexBasedLogitsProcessor``.  Touching any of them loads libsealb200.so (CUDA, sm_90a); there is no CPU
fallback.  The names are resolved lazily (PEP 562) so that the pure-numpy helpers (``seal_b200.synthetic``,
``seal_b200.sharding``'s layout code) can be imported by tooling — e.g. the CPU reference arm of ``bench.py`` —
without mapping the CUDA library into that process.
"""
__all__ = ["FMIndex", "fm_index_generate", "IndexBasedLogitsProcessor", "SealBartEngine"]


def __getattr__(name):
    if name == "FMIndex":
        from .index import FMIndex
        return FMIndex
    if name in ("fm_index_generate", "IndexBasedLogitsProcessor", "SealBartEngine"):
        from . import beam_search
        return getattr(beam_search, name)
    raise AttributeError(f"module 'seal_b200' has no attribute {name!r}")
