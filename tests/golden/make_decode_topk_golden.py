"""Pins the top-k decode oracle (tests/topk_oracle.py) against the REFERENCE'S OWN decode code and stores the reference's
outputs as fixtures (tests/golden/decode_topk_golden.json).  Runs on the CPU:

    python tests/golden/make_decode_topk_golden.py            # writes the fixture
    python tests/golden/make_decode_topk_golden.py --fuzz N   # N random cases, nothing stored

/root/reference/seal/beam_search.py is imported UNMODIFIED through make_decode_golden's shims (that file is used as
it is): its fm_index_generate(topk=k) builds `TopKLogitsWarper(k)` -- the installed transformers class, whose arithmetic
4.13 shares -- and constrained_beam_search applies it to the raw logits before log_softmax (:163-164, :249-253).
keep_history=False hands the loop transformers 4.13's stock `BeamSearchScorer`, which is not installed: those cases use
`BeamSearchScorer413`, the interface of 4.13's class around oracle.decode_oracle.HFBeamSearchScorer413 (the restatement
the drop-in's replay is checked against; parity with 4.13 itself stays unpinned there, DESIGN.md section 2).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle.fm_oracle import OracleIndex  # noqa: E402
from oracle.decode_oracle import HFBeamSearchScorer413, make_bart  # noqa: E402
from seal_b200.synthetic import make_corpus  # noqa: E402
from topk_oracle import fm_index_generate_topk_oracle  # noqa: E402
from make_decode_golden import Bart413Adapter, load_reference_beam_search, make_inputs, CORPUS, MODEL  # noqa: E402


class BeamSearchScorer413(HFBeamSearchScorer413):
    """transformers 4.13 `BeamSearchScorer`'s interface (constructor keywords, process / finalize returning dicts of
    tensors, hypotheses as tensors) over the oracle's restatement."""

    def __init__(self, batch_size, num_beams, device=None, length_penalty=1.0, do_early_stopping=False,
                 num_beam_hyps_to_keep=1, num_beam_groups=1):
        assert num_beam_groups == 1
        super().__init__(batch_size, num_beams, length_penalty, do_early_stopping, num_beam_hyps_to_keep)

    def process(self, input_ids, next_scores, next_tokens, next_indices, pad_token_id=None, eos_token_id=None):
        sc, tk, ix = super().process(input_ids, next_scores, next_tokens, next_indices, pad_token_id, eos_token_id)
        return {"next_beam_scores": torch.tensor(sc, dtype=torch.float), "next_beam_tokens": torch.tensor(tk, dtype=torch.long),
                "next_beam_indices": torch.tensor(ix, dtype=torch.long)}

    def finalize(self, input_ids, final_beam_scores, final_beam_tokens, final_beam_indices, pad_token_id=None,
                 eos_token_id=None, max_length=None):
        seq, scores = super().finalize(input_ids, final_beam_scores, max_length, pad_token_id, eos_token_id)
        for h in self._beam_hyps:
            h.beams = [(s, torch.tensor(t, dtype=torch.long)) for s, t in h.beams]
        return {"sequences": seq, "sequence_scores": scores}


def load_reference():
    ref = load_reference_beam_search()
    ref.BeamSearchScorer = BeamSearchScorer413
    return ref


V = MODEL["vocab"]
BODY = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0)
TITLE = dict(num_beams=5, min_length=0, max_length=15, length_penalty=0.0, eos_token_id=777, force_decoding_from=[2])
CASES = ([dict(BODY, topk=k, keep_history=True) for k in (1, 2 * 15 - 1, 10, 100, V - 3)]
         + [dict(TITLE, topk=k, keep_history=True) for k in (1, 2 * 5 - 1, 10, 100, V - 3)]
         + [dict(BODY, topk=10, keep_history=False), dict(TITLE, topk=9, keep_history=False),
            dict(TITLE, topk=1, keep_history=False),
            dict(num_beams=4, min_length=0, max_length=6, length_penalty=0.0, disable_fm_index=True, topk=10,
                 keep_history=True),
            dict(num_beams=4, min_length=0, max_length=6, length_penalty=0.0, disable_fm_index=True, topk=2,
                 keep_history=False),
            dict(num_beams=3, min_length=0, max_length=6, length_penalty=0.0, forced_bos_token_id=0, topk=5,
                 keep_history=True),
            dict(num_beams=4, min_length=0, max_length=7, length_penalty=0.0, stop_at_count=3, always_allow_eos=True,
                 topk=7, keep_history=True)])


def same(got_ref, got_ora):
    """Same hypotheses in the same order, worst |dscore|; None if the lists differ."""
    worst = 0.0
    if len(got_ref) != len(got_ora):
        return None
    for a, b in zip(got_ref, got_ora):
        if [tuple(t) for _, t in a] != [tuple(t) for _, t, _ in b]:
            return None
        for (sa, _), (sb, _, _) in zip(a, b):
            worst = max(worst, abs(sa - sb)) if sa != sb else worst
    return worst


def main():
    ref = load_reference()
    docs = make_corpus(**CORPUS)
    ora = OracleIndex([d.tolist() for d in docs], backend="ref")
    model = make_bart(**MODEL)
    adapter = Bart413Adapter(model)
    out = {"corpus": CORPUS, "model": MODEL, "cases": []}
    worst_all = 0.0
    for ci, kw in enumerate(CASES):
        rng = np.random.default_rng(300 + ci)
        ids, am = make_inputs(rng, Q=4, S=12, vocab=CORPUS["vocab"])
        got_ref = ref.fm_index_generate(adapter, ora, ids, am, **kw)
        info = {}
        got_ora = fm_index_generate_topk_oracle(model, ora, ids, am, info=info, **kw)
        worst = same(got_ref, got_ora)
        assert worst is not None, f"case {ci}: hypothesis lists differ"
        worst_all = max(worst_all, worst)
        n_inf = sum(1 for a in got_ora for _, _, c in a if c == float("-inf"))
        print(f"case {ci} {kw}: {sum(len(a) for a in got_ref)} hypotheses identical in order, worst |dscore| {worst:.2e}, "
              f"records from -inf constrained picks {n_inf}, min k-gap per query {['%.2e' % g for g in info['min_gap']]}")
        out["cases"].append({"kw": kw, "seed": 300 + ci, "input_ids": ids.tolist(), "attention_mask": am.tolist(),
                             "hyps": [[[float(s), [int(x) for x in t]] for s, t in a] for a in got_ref]})
    assert worst_all < 1e-5
    with open(os.path.join(HERE, "decode_topk_golden.json"), "w") as f:
        json.dump(out, f)
    print("wrote decode_topk_golden.json", os.path.getsize(os.path.join(HERE, "decode_topk_golden.json")), "bytes")


def fuzz(n_cases):
    """Randomised cross-check (nothing stored): the reference's fm_index_generate(topk=...) vs the oracle on random
    parameter combinations -- same hypotheses in the same order, |dscore| < 1e-5, or the same exception type."""
    ref = load_reference()
    docs = make_corpus(**CORPUS)
    ora = OracleIndex([d.tolist() for d in docs], backend="ref")
    model = make_bart(**MODEL)
    adapter = Bart413Adapter(model)
    rng = np.random.default_rng(2718)
    bad = raised = 0
    for case in range(n_cases):
        max_length = int(rng.integers(3, 11))
        B = int(rng.integers(1, 9))
        kw = dict(num_beams=B, max_length=max_length, min_length=int(rng.integers(0, max_length + 1)),
                  length_penalty=float(rng.choice([0.0, 0.5, 1.0])), keep_history=bool(rng.random() < 0.7),
                  topk=int(rng.choice([1, 2, 2 * B - 1, 2 * B, 10, 100, V - 4, V - 3, V, V + 5])))
        if rng.random() < 0.3: kw["always_allow_eos"] = True
        if rng.random() < 0.3: kw["stop_at_count"] = int(rng.choice([1, 2, 5]))
        if rng.random() < 0.25:
            d = int(rng.integers(0, docs.shape[0])); a = int(rng.integers(0, docs.shape[1] - 3))
            kw["force_decoding_from"] = [int(t) for t in docs[d, a:a + int(rng.integers(1, 3))]]
        if rng.random() < 0.2: kw["forced_bos_token_id"] = 0
        if rng.random() < 0.15: kw["disable_fm_index"] = True
        if rng.random() < 0.2: kw["eos_token_id"] = int(rng.integers(4, CORPUS["vocab"]))
        ids, am = make_inputs(rng, Q=int(rng.integers(1, 4)), S=int(rng.integers(4, 13)), vocab=CORPUS["vocab"])
        try:
            a = ref.fm_index_generate(adapter, ora, ids, am, **kw)
        except Exception as e:
            raised += 1
            try:
                fm_index_generate_topk_oracle(model, ora, ids, am, **kw)
                print("case", case, kw, "reference raised", type(e).__name__, e, "but the oracle did not"); bad += 1
            except Exception as e2:
                if type(e2) is not type(e):
                    print("case", case, kw, "different exceptions", type(e).__name__, type(e2).__name__); bad += 1
            continue
        worst = same(a, fm_index_generate_topk_oracle(model, ora, ids, am, **kw))
        if worst is None or worst >= 1e-5:
            bad += 1
            print("case", case, "MISMATCH", kw)
    print(f"fuzz: {n_cases} cases ({raised} where both raise), {bad} mismatches")
    return bad


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--fuzz":
        sys.exit(1 if fuzz(int(sys.argv[2])) else 0)
    main()
