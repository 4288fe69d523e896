import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    # `-m gpu` tests must fail loudly if there is no GPU rather than silently skipping
    pass


def random_text(seed, n, vocab, lo=10):
    rng = np.random.default_rng(seed)
    return rng.integers(lo, lo + vocab, size=n).astype(np.uint64)


@pytest.fixture(scope="session")
def small_corpus():
    """2 000 phrase-structured docs x 40 tokens (80 k tokens) in SEAL's symbol convention."""
    from seal_b200.synthetic import make_corpus
    return make_corpus(n_docs=2000, doc_len=40, n_phrases=5000, seed=7)


@pytest.fixture(scope="session")
def oracle_backend_cls():
    """The compiled reference when present (this container / shipped .so), else the C port."""
    from oracle.fm_oracle import RefFM, PortFM, ref_available
    return RefFM if ref_available() else PortFM
