"""fm_index_generate(topk=k) without a GPU: the oracle's top-k warp (tests/topk_oracle.py) reproduces what the
reference's own seal/beam_search.py returned (tests/golden/decode_topk_golden.json), and the drop-in treats every kind
of `topk` value the way the reference does, before any device work."""
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _golden():
    with open(os.path.join(HERE, "golden", "decode_topk_golden.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", range(len(_golden()["cases"])))
def test_topk_oracle_reproduces_reference_fixture(case):
    from topk_oracle import fm_index_generate_topk_oracle
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.synthetic import make_corpus
    g = _golden()
    c = g["cases"][case]
    ora = OracleIndex([d.tolist() for d in make_corpus(**g["corpus"])])
    model = make_bart(**g["model"])
    got = fm_index_generate_topk_oracle(model, ora, torch.tensor(c["input_ids"]), torch.tensor(c["attention_mask"]),
                                        **c["kw"])
    assert len(got) == len(c["hyps"])
    for q, (ours, ref) in enumerate(zip(got, c["hyps"])):
        assert [t for _, t, _ in ours] == [t for _, t in ref], f"query {q}: hypothesis lists differ"
        for (sa, _, _), (sb, _) in zip(ours, ref):
            assert sa == sb or abs(sa - sb) < 1e-5, (q, sa, sb)


def test_topk_warp_arithmetic():
    """k_eff = min(max(k, 1), V); ties at tau kept; -0.0 == +0.0; -inf entries count as values"""
    from topk_oracle import topk_warp
    x = torch.tensor([[3.0, 1.0, 3.0, 2.0, 2.0, -0.0, 0.0, float("-inf")]])
    ninf = float("-inf")
    assert topk_warp(x, 1).tolist() == [[3.0, ninf, 3.0, ninf, ninf, ninf, ninf, ninf]]
    assert topk_warp(x, 3).tolist() == [[3.0, ninf, 3.0, 2.0, 2.0, ninf, ninf, ninf]]
    assert topk_warp(x, 6).tolist() == [[3.0, 1.0, 3.0, 2.0, 2.0, -0.0, 0.0, ninf]]      # tau = 0: both zeros kept
    assert topk_warp(x, 8).tolist() == x.tolist()                                        # tau = -inf
    assert topk_warp(x, 100).tolist() == x.tolist()


@pytest.mark.parametrize("topk, exc", [
    (2.5, ValueError),                       # TopKLogitsWarper's constructor
    (np.int64(3), ValueError),               # not a Python int
    (-1, UnboundLocalError),                 # the reference never binds topk_warper
    (-7, UnboundLocalError),
])
def test_topk_arguments_rejected_before_device_work(topk, exc):
    """model / index / inputs are None: the checks must fire before anything touches them"""
    from seal_b200.beam_search import fm_index_generate
    for keep_history in (True, False):
        with pytest.raises(exc) as e:
            fm_index_generate(None, None, None, None, num_beams=4, keep_history=keep_history, topk=topk)
        if exc is ValueError:
            assert str(e.value) == f"`top_k` has to be a strictly positive integer, but is {topk}"


@pytest.mark.parametrize("topk, expect", [(0, 0), (False, 0), (None, 0), (0.0, 0), (True, 1), (1, 1), (10, 10),
                                          (50265, 50265)])
def test_topk_values_accepted(topk, expect):
    from seal_b200.beam_search import _check_topk
    assert _check_topk(topk, 1) == expect


@pytest.mark.parametrize("topk", [5, 0, None, 2.5, -3, np.int64(4), True])
def test_topk_ignored_with_diverse_groups(topk, monkeypatch):
    """group_beam_search never sees topk: with diverse_bs_groups > 1 the parameters carry top_k = 0, whatever topk is"""
    import seal_b200.beam_search as bs
    seen = {}

    def fake_generate_records(*a, **kw):
        seen.update(kw)
        raise RuntimeError("stop before device work")

    monkeypatch.setattr(bs, "generate_records", fake_generate_records)
    with pytest.raises(RuntimeError, match="stop before device work"):
        bs.fm_index_generate(None, None, None, None, num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=0.5,
                             keep_history=True, topk=topk)
    assert seen["top_k"] == 0 and seen["num_beam_groups"] == 2


def test_sample_still_not_implemented():
    from seal_b200.beam_search import fm_index_generate
    with pytest.raises(NotImplementedError):
        fm_index_generate(None, None, None, None, num_beams=4, keep_history=True, sample=True, topk=5)


def test_params_carry_top_k():
    """DecParams: top_k after shift, zero-filled when a caller passes the 17 older fields only"""
    import ctypes as C
    from types import SimpleNamespace
    from seal_b200._lib import DecParams
    from seal_b200.beam_search import _make_params
    assert C.sizeof(DecParams) == 80
    assert DecParams(*range(15), None, 10).top_k == 0
    cfg = SimpleNamespace(pad_token_id=1, decoder_start_token_id=2, eos_token_id=2, forced_eos_token_id=2)
    assert _make_params(cfg, 4, 0, 10, 0.0, 2, None, False, False, 0, None).top_k == 0
    assert _make_params(cfg, 4, 0, 10, 0.0, 2, None, False, False, 0, None, 17).top_k == 17
