"""Pins the diverse-beam-group decode oracle (tests/group_oracle.py) against the REFERENCE'S OWN decode code and stores
the reference's outputs as fixtures (tests/golden/decode_groups_golden.json).  Run in the build container only:

    python tests/golden/make_decode_groups_golden.py            # writes the fixture
    python tests/golden/make_decode_groups_golden.py --fuzz N   # N random cases, nothing stored

/root/reference/seal/beam_search.py is imported UNMODIFIED (make_decode_golden.load_reference_beam_search): its
fm_index_generate builds the processor list, appends HammingDiversityLogitsProcessor and IndexBasedLogitsProcessor
(num_beams // groups) to it, builds BeamSearchScorerWithMemory(num_beam_groups=G) and calls
`model.group_beam_search` (seal/beam_search.py:447-532) -- all as shipped.  transformers 4.13 is not installed, so
two of its pieces are supplied, restated from its published algorithm (the only assumptions left):

  * `HammingDiversityLogitsProcessor` (constructor checks and __call__), installed on `transformers` before the
    reference module is loaded;
  * `group_beam_search`, a method of `GroupBart413Adapter` (make_decode_golden.Bart413Adapter plus this method).
    transformers 5.5's LogitsProcessorList still forwards `current_tokens` / `beam_group_idx` to processors that
    take them (the 4.13 protocol), so the reference's list is used as it is.
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
from oracle.decode_oracle import make_bart  # noqa: E402
from seal_b200.synthetic import make_corpus  # noqa: E402
from group_oracle import fm_index_generate_groups_oracle, proc_hamming_413  # noqa: E402
from make_decode_golden import Bart413Adapter, load_reference_beam_search, make_inputs, CORPUS, MODEL  # noqa: E402


class HammingDiversityLogitsProcessor413:
    """transformers 4.13 HammingDiversityLogitsProcessor (generation_logits_process.py), restated."""

    def __init__(self, diversity_penalty: float, num_beams: int, num_beam_groups: int):
        if not isinstance(diversity_penalty, float) or (not diversity_penalty > 0.0):
            raise ValueError("`diversity_penalty` should be a float strictly larger than 0.")
        self._diversity_penalty = diversity_penalty
        if not isinstance(num_beams, int) or num_beams < 2:
            raise ValueError("`num_beams` should be an integer strictly larger than 1.")
        self._num_beams = num_beams
        if not isinstance(num_beam_groups, int) or num_beam_groups < 2:
            raise ValueError("`num_beam_groups` should be an integer strictly larger than 1.")
        if num_beam_groups > num_beams:
            raise ValueError("`beam_groups` has to be smaller or equal to `num_beams`.")
        self._num_beam_groups = num_beam_groups

    def __call__(self, input_ids, scores, current_tokens, beam_group_idx):
        return proc_hamming_413(current_tokens, scores, beam_group_idx, self._diversity_penalty, self._num_beams,
                                self._num_beam_groups)


class GroupBart413Adapter(Bart413Adapter):
    def group_beam_search(self, input_ids, beam_scorer, logits_processor=None, stopping_criteria=None,
                          pad_token_id=None, eos_token_id=None, output_scores=None, **model_kwargs):
        """transformers 4.13 GenerationMixin.group_beam_search, restated (no synced GPUs, no output dicts: the
        reference calls it with return_dict_in_generate False and reads the scorer's memory)."""
        batch_size = len(beam_scorer._beam_hyps)
        num_beams = beam_scorer.num_beams
        num_beam_groups = beam_scorer.num_beam_groups
        num_sub_beams = num_beams // num_beam_groups
        batch_beam_size, cur_len = input_ids.shape
        assert num_beams * batch_size == batch_beam_size
        beam_scores = torch.full((batch_size, num_beams), -1e9, dtype=torch.float)
        # the first beam of each group starts at 0, so that the beams of a group do not all pick the same tokens
        beam_scores[:, ::num_sub_beams] = 0
        beam_scores = beam_scores.view((batch_size * num_beams,))
        while True:
            current_tokens = torch.zeros(batch_size * num_beams, dtype=input_ids.dtype)
            reordering_indices = torch.zeros(batch_size * num_beams, dtype=torch.long)
            model_inputs = self.prepare_inputs_for_generation(input_ids, **model_kwargs)
            outputs = self(**model_inputs, return_dict=True)
            for beam_group_idx in range(num_beam_groups):
                group_start_idx = beam_group_idx * num_sub_beams
                group_end_idx = min(group_start_idx + num_sub_beams, num_beams)
                group_size = group_end_idx - group_start_idx
                batch_group_indices = []
                for batch_idx in range(batch_size):
                    batch_group_indices.extend([batch_idx * num_beams + idx for idx in range(group_start_idx, group_end_idx)])
                group_input_ids = input_ids[batch_group_indices]
                next_token_logits = outputs.logits[batch_group_indices, -1, :]
                next_token_logits = self.adjust_logits_during_generation(next_token_logits, cur_len=cur_len)
                next_token_scores = torch.nn.functional.log_softmax(next_token_logits, dim=-1)
                vocab_size = next_token_scores.shape[-1]
                next_token_scores = logits_processor(group_input_ids, next_token_scores, current_tokens=current_tokens,
                                                     beam_group_idx=beam_group_idx)
                next_token_scores = next_token_scores + beam_scores[batch_group_indices].unsqueeze(-1).expand_as(next_token_scores)
                next_token_scores = next_token_scores.view(batch_size, group_size * vocab_size)
                next_token_scores, next_tokens = torch.topk(next_token_scores, 2 * group_size, dim=1, largest=True, sorted=True)
                next_indices = torch.div(next_tokens, vocab_size, rounding_mode="floor")
                next_tokens = next_tokens % vocab_size
                beam_outputs = beam_scorer.process(group_input_ids, next_token_scores, next_tokens, next_indices,
                                                   pad_token_id=pad_token_id, eos_token_id=eos_token_id)
                beam_scores[batch_group_indices] = beam_outputs["next_beam_scores"]
                beam_next_tokens = beam_outputs["next_beam_tokens"]
                beam_idx = beam_outputs["next_beam_indices"]
                input_ids[batch_group_indices] = group_input_ids[beam_idx]
                group_input_ids = torch.cat([group_input_ids[beam_idx, :], beam_next_tokens.unsqueeze(-1)], dim=-1)
                current_tokens[batch_group_indices] = group_input_ids[:, -1]
                reordering_indices[batch_group_indices] = (
                    num_beams * torch.div(beam_idx, group_size, rounding_mode="floor") + group_start_idx + (beam_idx % group_size))
            input_ids = torch.cat([input_ids, current_tokens.unsqueeze(-1)], dim=-1)
            model_kwargs = self._update_model_kwargs_for_generation(outputs, model_kwargs, is_encoder_decoder=True)
            assert model_kwargs["past"] is None                      # full re-forward: nothing to reorder
            cur_len = cur_len + 1
            if beam_scorer.is_done or stopping_criteria(input_ids, None):
                break
        sequence_outputs = beam_scorer.finalize(input_ids, beam_scores, next_tokens, next_indices, pad_token_id=pad_token_id,
                                                eos_token_id=eos_token_id, max_length=stopping_criteria.max_length)
        return sequence_outputs["sequences"]


def load_reference():
    import transformers
    transformers.HammingDiversityLogitsProcessor = HammingDiversityLogitsProcessor413
    return load_reference_beam_search()


CASES = [
    dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0),
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.0, min_length=2, max_length=6, length_penalty=1.0),
    dict(num_beams=3, diverse_bs_groups=3, diverse_bs_penalty=2.0, min_length=0, max_length=6, length_penalty=0.0),
    dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0,
         always_allow_eos=True),
    dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=0.5, min_length=0, max_length=7, length_penalty=0.0,
         stop_at_count=3),
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=6, length_penalty=0.0,
         forced_bos_token_id=0),
    dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=2.0, min_length=0, max_length=6, length_penalty=0.0,
         disable_fm_index=True),
    dict(num_beams=15, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=10, max_length=10, length_penalty=0.0),
    dict(num_beams=15, diverse_bs_groups=5, diverse_bs_penalty=0.5, min_length=10, max_length=10, length_penalty=0.0),
    dict(num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5, min_length=0, max_length=9, length_penalty=0.0,
         eos_token_id=777, force_decoding_from=[2]),
    dict(num_beams=4, diverse_bs_groups=2, diverse_bs_penalty=0.5, min_length=3, max_length=7, length_penalty=1.0,
         force_decoding_from=[996, 523]),
]


def same(got_ref, got_ora):
    """Same hypotheses in the same order, worst |dscore|; None if the lists differ."""
    worst = 0.0
    if len(got_ref) != len(got_ora):
        return None
    for a, b in zip(got_ref, got_ora):
        if [tuple(t) for _, t in a] != [tuple(t) for _, t, _ in b]:
            return None
        for (sa, _), (sb, _, _) in zip(a, b):
            worst = max(worst, abs(sa - sb))
    return worst


def main():
    ref = load_reference()
    docs = make_corpus(**CORPUS)
    ora = OracleIndex([d.tolist() for d in docs], backend="ref")
    model = make_bart(**MODEL)
    adapter = GroupBart413Adapter(model)
    out = {"corpus": CORPUS, "model": MODEL, "cases": []}
    worst_all = 0.0
    for ci, kw in enumerate(CASES):
        rng = np.random.default_rng(200 + ci)
        ids, am = make_inputs(rng, Q=4, S=12, vocab=CORPUS["vocab"])
        got_ref = ref.fm_index_generate(adapter, ora, ids, am, keep_history=True, **kw)
        info = {}
        got_ora = fm_index_generate_groups_oracle(model, ora, ids, am, info=info, **kw)
        worst = same(got_ref, got_ora)
        assert worst is not None, f"case {ci}: hypothesis lists differ"
        worst_all = max(worst_all, worst)
        print(f"case {ci} {kw}: {sum(len(a) for a in got_ref)} hypotheses identical in order, worst |dscore| {worst:.2e}, "
              f"tie-sensitive queries {info['tie_sensitive']}")
        out["cases"].append({"kw": kw, "seed": 200 + ci, "input_ids": ids.tolist(), "attention_mask": am.tolist(),
                             "tie_sensitive": info["tie_sensitive"],
                             "hyps": [[[float(s), [int(x) for x in t]] for s, t in a] for a in got_ref]})
    assert worst_all < 1e-5
    with open(os.path.join(HERE, "decode_groups_golden.json"), "w") as f:
        json.dump(out, f)
    print("wrote decode_groups_golden.json", os.path.getsize(os.path.join(HERE, "decode_groups_golden.json")), "bytes")


def fuzz(n_cases):
    """Randomised cross-check (nothing stored): the reference's fm_index_generate vs the oracle restatement on random
    parameter combinations -- same hypotheses in the same order, |dscore| < 1e-5, or the same exception type."""
    ref = load_reference()
    docs = make_corpus(**CORPUS)
    ora = OracleIndex([d.tolist() for d in docs], backend="ref")
    model = make_bart(**MODEL)
    adapter = GroupBart413Adapter(model)
    rng = np.random.default_rng(4242)
    bad = raised = 0
    for case in range(n_cases):
        max_length = int(rng.integers(3, 11))
        G = int(rng.choice([2, 3, 4]))
        kw = dict(num_beams=G * int(rng.integers(1, 4)), diverse_bs_groups=G,
                  diverse_bs_penalty=float(rng.choice([0.0, 0.25, 0.5, 2.0])), max_length=max_length,
                  min_length=int(rng.integers(0, max_length + 1)), length_penalty=float(rng.choice([0.0, 0.5, 1.0])))
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
            a = ref.fm_index_generate(adapter, ora, ids, am, keep_history=True, **kw)
        except Exception as e:
            raised += 1
            try:
                fm_index_generate_groups_oracle(model, ora, ids, am, **kw)
                print("case", case, kw, "reference raised", type(e).__name__, e, "but the oracle did not"); bad += 1
            except Exception as e2:
                if type(e2) is not type(e):
                    print("case", case, kw, "different exceptions", type(e).__name__, type(e2).__name__); bad += 1
            continue
        worst = same(a, fm_index_generate_groups_oracle(model, ora, ids, am, **kw))
        if worst is None or worst >= 1e-5:
            bad += 1
            print("case", case, "MISMATCH", kw)
    print(f"fuzz: {n_cases} cases ({raised} where both raise), {bad} mismatches")
    return bad


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--fuzz":
        sys.exit(1 if fuzz(int(sys.argv[2])) else 0)
    main()
