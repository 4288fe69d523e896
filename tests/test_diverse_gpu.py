"""GPU parity of diverse beam groups (fm_index_generate's diverse_bs_groups / diverse_bs_penalty; include/sealdec.h
sealdec_groups_t) against the restatement of transformers 4.13's group_beam_search (tests/group_oracle.py) driving
transformers' BART in eager fp32.  Compared like test_decode_gpu.compare_generate: the sorted hypotheses that pass the
caller's get_count > 0 filter, scores within 1e-4.  Queries where a -inf tie-filled beam's token entered a later
group's penalty (`tie_sensitive`: torch.topk's choice among -inf ties is unspecified) are left out and counted."""
import json
import os

import numpy as np
import pytest

from test_decode_gpu import compare_generate, make_inputs, tiny_setup

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


@pytest.fixture(scope="module")
def tiny():
    return tiny_setup()


def compare_untied(got, exp, tie, ora, **kw):
    keep = [q for q in range(len(got)) if not tie[q]]
    worst = compare_generate([got[q] for q in keep], [exp[q] for q in keep], ora, **kw)
    return worst, len(keep)


GRID = [dict(num_beams=6, diverse_bs_groups=G, diverse_bs_penalty=pen, min_length=0, max_length=7, length_penalty=0.0)
        for G in (2, 3, 6) for pen in (0.0, 0.5, 2.0)]
OPTIONS = [
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0, stop_at_count=3),
    dict(num_beams=6, diverse_bs_groups=2, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0, always_allow_eos=True),
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=6, length_penalty=0.0, forced_bos_token_id=0),
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=2.0, min_length=0, max_length=6, length_penalty=0.0, disable_fm_index=True),
    # body pass (seal/retrieval.py): n-grams of 10
    dict(num_beams=15, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=10, max_length=10, length_penalty=0.0),
    dict(num_beams=15, diverse_bs_groups=5, diverse_bs_penalty=0.5, min_length=10, max_length=10, length_penalty=0.0),
    # title pass: own eos id, decoding forced to start at a document end
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=9, length_penalty=1.0,
         eos_token_id=777, force_decoding_from=[2]),
]


@pytest.mark.parametrize("kw", GRID + OPTIONS)
def test_diverse_generate_vs_oracle_tiny(kw, tiny):
    from group_oracle import fm_index_generate_groups_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny
    rng = np.random.default_rng(41)
    ids, am = make_inputs(rng, Q=8, S=12, vocab=2000)
    info = {}
    exp = fm_index_generate_groups_oracle(model, ora, ids, am, info=info, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst, n = compare_untied(got, exp, info["tie_sensitive"], ora, force=kw.get("force_decoding_from"),
                              skip=1 if kw.get("forced_bos_token_id") is not None else 0)
    print(f"{kw}: worst |dscore| = {worst:.3e}; {n}/{len(got)} queries compared")
    assert n >= len(got) // 2 + 1


def _golden():
    with open(os.path.join(HERE, "golden", "decode_groups_golden.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", range(len(_golden()["cases"])))
def test_diverse_generate_vs_reference_code_fixture(case):
    """decode_groups_golden.json: what the reference's own seal/beam_search.py returned for these inputs."""
    import torch
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    g = _golden()
    c = g["cases"][case]
    seqs = [d.tolist() for d in make_corpus(**g["corpus"])]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    kw = c["kw"]
    got = fm_index_generate(make_bart(**g["model"]), idx, torch.tensor(c["input_ids"]), torch.tensor(c["attention_mask"]),
                            keep_history=True, **kw)
    exp = [[(s, t, None) for s, t in q] for q in c["hyps"]]
    worst, n = compare_untied(got, exp, c["tie_sensitive"], ora, force=kw.get("force_decoding_from"),
                              skip=1 if kw.get("forced_bos_token_id") is not None else 0)
    print(f"reference-code fixture {kw}: worst |dscore| = {worst:.3e}; {n}/{len(got)} queries compared")
    assert n >= len(got) // 2 + 1


def test_penalty_zero_groups_are_copies(tiny):
    """Without a penalty the groups never see each other: every group's records equal group 0's, step by step."""
    from seal_b200.beam_search import generate_records
    docs, ora, idx, model = tiny
    rng = np.random.default_rng(43)
    ids, am = make_inputs(rng, Q=6, S=12, vocab=2000)
    B, G, T = 6, 3, 7
    rec = generate_records(model, idx, ids, am, 0, T, 0.0, B, num_beam_groups=G, diversity_penalty=0.0)
    gs, K = B // G, 2 * B // G
    for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
        a = rec[k]
        for s in range(T - 1):
            base = s * 2 * B
            for g in range(1, G):
                assert np.array_equal(a[:, base + g * K:base + (g + 1) * K], a[:, base:base + K]), (k, s, g)
        fb = (T - 1) * 2 * B
        for g in range(1, G):
            assert np.array_equal(a[:, fb + g * gs:fb + (g + 1) * gs], a[:, fb:fb + gs]), (k, "finalize", g)
    assert np.isfinite(rec["scores"]).any()


def test_generate_null_groups_is_one_group(tiny):
    """sealdec_generate with groups NULL and with {1, 0}: bit-identical record buffers."""
    import ctypes as C
    from seal_b200._lib import GroupParams, check, lib
    from seal_b200.beam_search import _engine_for, _make_params, _occurring_mask
    docs, ora, idx, model = tiny
    eng = _engine_for(model)
    rng = np.random.default_rng(44)
    ids, am = make_inputs(rng, Q=5, S=12, vocab=2000)
    ids = np.ascontiguousarray(ids.numpy()); am = np.ascontiguousarray(am.numpy())
    Q, S = ids.shape
    T = 8
    p = _make_params(eng.config, 6, 2, T, 0.0, eng.config.eos_token_id, None, False, False, 0, None)
    H = int(lib.sealdec_hyps_per_query(C.byref(p)))
    if idx._device is None:
        idx.to_device(eng.device)
    occ = _occurring_mask(idx, int(eng.config.vocab_size))

    def run(groups):
        out = [np.zeros((Q, H), np.float32), np.zeros((Q, H), np.int32), np.zeros((Q, H, T), np.int32),
               np.zeros((Q, H), np.uint8), np.zeros((Q, H), np.uint64), np.zeros((Q, H), np.uint64)]
        args = [eng._h, idx._dev(), occ.ctypes.data, C.byref(p), ids.ctypes.data, am.ctypes.data, Q, S] + [o.ctypes.data for o in out]
        check(lib.sealdec_generate(*args, groups))
        return out

    for a, b in zip(run(None), run(C.byref(GroupParams(1, 0.0)))):
        assert a.tobytes() == b.tobytes()
    with pytest.raises(Exception):
        check(lib.sealdec_generate(eng._h, idx._dev(), occ.ctypes.data, C.byref(p), ids.ctypes.data, am.ctypes.data,
                                   Q, S, *([None] * 6), C.byref(GroupParams(4, 0.0))))


def test_graph_replay_and_key_q20_beam15(tiny):
    """Q = 20, beam 15, G = 3 through the host-buffer API: the third call replays the captured CUDA graph and returns
    the eager call's records bit for bit; changing the penalty or G builds a new key (no stale graph)."""
    from seal_b200._lib import lib
    from seal_b200.beam_search import SealBartEngine, generate_records
    docs, ora, idx, model = tiny
    eng = SealBartEngine.from_hf(model, device=0)
    rng = np.random.default_rng(45)
    ids, am = make_inputs(rng, Q=20, S=12, vocab=2000)
    kw = dict(min_length=0, max_length=8, length_penalty=0.0, num_beams=15)
    used, recs = [], []
    for _ in range(3):
        recs.append(generate_records(eng, idx, ids, am, num_beam_groups=3, diversity_penalty=0.5, **kw))
        used.append(int(lib.sealbart_get_stat(eng._h, b"last_used_graph")))
    assert used[0] == 0 and used[2] == 1, used
    for r in recs[1:]:
        for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
            assert np.array_equal(r[k], recs[0][k]), k
    for grp, pen in ((3, 0.0), (5, 0.5)):
        other = generate_records(eng, idx, ids, am, num_beam_groups=grp, diversity_penalty=pen, **kw)
        assert int(lib.sealbart_get_stat(eng._h, b"last_used_graph")) == 0
        assert not np.array_equal(other["tokens"], recs[0]["tokens"]), (grp, pen)


def test_diverse_bart_large_batch20_beam15():
    """The SEALSearcher --diverse_bs_groups 3 --diverse_bs_penalty 0.5 operating point: bart-large (seeded random
    weights), batch 20, beam 15, body n-grams of 10, on the 200 k-token phrase corpus; oracle on the same GPU."""
    import torch
    from group_oracle import fm_index_generate_groups_oracle
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus, make_queries
    docs = make_corpus(n_docs=2000, doc_len=100, n_phrases=4000, seed=21)
    seqs = [d.tolist() for d in docs]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    model = make_bart(seed=0)
    ids, am = make_queries(20, seed=77)
    ids = torch.tensor(ids); am = torch.tensor(am)
    kw = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0, diverse_bs_groups=3, diverse_bs_penalty=0.5)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    info = {}
    exp = fm_index_generate_groups_oracle(model.to("cuda"), ora, ids.cuda(), am.cuda(), info=info, **kw)
    worst, n = compare_untied(got, exp, info["tie_sensitive"], ora)
    print(f"diverse batch20/beam15/G3: worst |dscore| = {worst:.3e}; {n}/20 queries compared")
    assert n >= 11
