"""Diverse beam groups (fm_index_generate's diverse_bs_groups / diverse_bs_penalty) without a GPU: the oracle
restatement of transformers 4.13's group_beam_search (tests/group_oracle.py) reproduces what the reference's own
seal/beam_search.py returned (tests/golden/decode_groups_golden.json), and the drop-in rejects bad arguments the way
the reference does, before any device work."""
import json
import os

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _golden():
    with open(os.path.join(HERE, "golden", "decode_groups_golden.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", range(len(_golden()["cases"])))
def test_group_oracle_reproduces_reference_fixture(case):
    from group_oracle import fm_index_generate_groups_oracle
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.synthetic import make_corpus
    g = _golden()
    c = g["cases"][case]
    ora = OracleIndex([d.tolist() for d in make_corpus(**g["corpus"])])
    model = make_bart(**g["model"])
    info = {}
    got = fm_index_generate_groups_oracle(model, ora, torch.tensor(c["input_ids"]), torch.tensor(c["attention_mask"]),
                                          info=info, **c["kw"])
    assert info["tie_sensitive"] == c["tie_sensitive"]
    assert len(got) == len(c["hyps"])
    for q, (ours, ref) in enumerate(zip(got, c["hyps"])):
        assert [t for _, t, _ in ours] == [t for _, t in ref], f"query {q}: hypothesis lists differ"
        for (sa, _, _), (sb, _) in zip(ours, ref):
            assert abs(sa - sb) < 1e-5, (q, sa, sb)


@pytest.mark.parametrize("kw, exc", [
    (dict(num_beams=4, diverse_bs_groups=3), ValueError),                               # 4 % 3 != 0
    (dict(num_beams=4, diverse_bs_groups=5), ValueError),                               # more groups than beams
    (dict(num_beams=4, diverse_bs_groups=8, diverse_bs_penalty=0.5), ValueError),       # Hamming constructor
    (dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=1), ValueError),         # penalty not a float
    (dict(num_beams=4, diverse_bs_groups=2.0), ValueError),                             # groups not an int
    (dict(num_beams=4, diverse_bs_groups=2, keep_history=False), NotImplementedError),  # stock grouped scorer
    (dict(num_beams=4, diverse_bs_groups=2, sample=True), NotImplementedError),
])
def test_diverse_arguments_rejected_before_device_work(kw, exc):
    """model / index / inputs are None: the checks must fire before anything touches them."""
    from seal_b200.beam_search import fm_index_generate
    kw = dict(kw)
    kw.setdefault("keep_history", True)
    with pytest.raises(exc):
        fm_index_generate(None, None, None, None, **kw)


def test_group_oracle_penalty_zero_groups_are_copies():
    """With no penalty the groups never see each other: every group decodes what group 0 decodes."""
    from group_oracle import group_beam_search_oracle
    V, B, G = 50, 6, 3
    gen = torch.Generator().manual_seed(0)
    table = torch.randn(4096, V, generator=gen)

    def step_logits(ids):
        h = (ids * torch.arange(1, ids.shape[1] + 1)).sum(1) % table.shape[0]
        return table[h]

    recs = group_beam_search_oracle(step_logits, 2, None, B, G, 0.0, 0, 5, 0.0, eos_token_id=2, pad_token_id=1,
                                    decoder_start_token_id=2, model_eos_token_id=2, forced_eos_token_id=None,
                                    disable_fm_index=True)
    for q in recs:
        q = [(s, t) for s, t, _ in q]
        gs, K = B // G, 2 * B // G
        steps = (len(q) - B) // (2 * B)
        for s in range(steps):
            blk = q[s * 2 * B:(s + 1) * 2 * B]
            for g in range(1, G):
                assert blk[g * K:(g + 1) * K] == blk[:K]
        fin = q[steps * 2 * B:]
        for g in range(1, G):
            assert fin[g * gs:(g + 1) * gs] == fin[:gs]
