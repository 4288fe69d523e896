"""TEST INFRASTRUCTURE ONLY -- diverse beam groups for the decode oracle (oracle/decode_oracle.py).

fm_index_generate with diverse_bs_groups > 1 (seal/beam_search.py:447-469, :491-503, :523-532 of the reference) hands
the decode to transformers 4.13's `group_beam_search` with a `HammingDiversityLogitsProcessor`.  Neither exists in the
installed transformers 5.5 and 4.13 is not vendored, so both are restated here from 4.13's published algorithm (the way
DESIGN.md section 2 restates the stock BeamSearchScorer): PARITY UNPINNED against 4.13 itself.  Everything else --
processors, index mask, scorer, hypothesis container -- is the pinned oracle's own code.
tests/golden/make_decode_groups_golden.py runs the reference's fm_index_generate / IndexBasedLogitsProcessor /
BeamSearchScorerWithMemory unmodified around the same restatement and stores tests/golden/decode_groups_golden.json.
"""
import os
import sys
from typing import Callable, List, Optional, Sequence

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.decode_oracle import (NEG_INF, HFBartCachedStepper, HFBartStepper, HypsWithMemory,  # noqa: E402
                                  IndexBasedLogitsProcessorOracle, proc_forced_bos, proc_forced_eos, proc_inf_nan,
                                  proc_min_length)


def proc_hamming_413(current_tokens, scores, beam_group_idx, diversity_penalty, num_beams, num_beam_groups):
    """transformers 4.13 `HammingDiversityLogitsProcessor.__call__` (seal/beam_search.py:447-454 appends it), restated
    from 4.13 (module docstring).  `scores` holds the group's rows [batch * group_size, V]; in place."""
    num_sub_beams = num_beams // num_beam_groups
    batch_size = current_tokens.shape[0] // num_beams
    group_start_idx = beam_group_idx * num_sub_beams
    group_end_idx = min(group_start_idx + num_sub_beams, num_beams)
    group_size = group_end_idx - group_start_idx
    vocab_size = scores.shape[-1]
    if group_start_idx == 0:
        return scores
    for batch_idx in range(batch_size):
        previous_group_tokens = current_tokens[batch_idx * num_beams: batch_idx * num_beams + group_start_idx]
        token_frequency = torch.bincount(previous_group_tokens, minlength=vocab_size).to(scores.device)
        scores[batch_idx * group_size: (batch_idx + 1) * group_size] -= diversity_penalty * token_frequency
    return scores


def group_beam_search_oracle(
        step_logits: Callable[[torch.Tensor], torch.Tensor],
        batch_size: int,
        index,
        num_beams: int,
        num_beam_groups: int,
        diversity_penalty: float,
        min_length: int,
        max_length: int,
        length_penalty: float = 1.0,
        eos_token_id: int = 2,
        pad_token_id: int = 1,
        decoder_start_token_id: int = 2,
        model_eos_token_id: int = 2,
        forced_eos_token_id: Optional[int] = 2,
        forced_bos_token_id: Optional[int] = None,
        force_decoding_from: Optional[List[int]] = None,
        stop_at_count: int = 0,
        always_allow_eos: bool = False,
        disable_fm_index: bool = False,
        processors: Sequence[str] = ("min_length", "forced_bos", "forced_eos", "inf_nan"),
        reorder: Optional[Callable[[torch.Tensor], None]] = None,
        info: Optional[dict] = None):
    """fm_index_generate with diverse_bs_groups > 1 and keep_history=True (:447-469, :491-503, :523-532):
    transformers 4.13's `group_beam_search` (restated, see proc_hamming_413) driving BeamSearchScorerWithMemory with
    group_size = num_beams // num_beam_groups (:580, :625-690).  Processors in the reference's list order: the HF ones,
    then Hamming (if diversity_penalty > 0), then the index mask built for num_beams // num_beam_groups beams.

    Returns what constrained_beam_search_oracle returns; the third item of a record is its (constrained) score.
    `info["tie_sensitive"]` (if `info` is a dict): per query, whether the token of a -inf (tie-filled) beam entered the
    Hamming penalty of a finite score in a later group.  Which of several -inf candidates torch.topk returns is
    unspecified, so such a query's later groups may legitimately differ between implementations."""
    G = num_beam_groups
    gs = num_beams // G
    cdp = None
    if not disable_fm_index:
        cdp = IndexBasedLogitsProcessorOracle(index, gs, pad_token_id=pad_token_id,
                                              eos_token_id=eos_token_id or model_eos_token_id,
                                              force_decoding_from=force_decoding_from, stop_at_count=stop_at_count,
                                              always_allow_eos=always_allow_eos,
                                              forced_bos_token_id=forced_bos_token_id)
    hyps = [HypsWithMemory(length_penalty, max_length) for _ in range(batch_size)]
    tie = [False] * batch_size
    R = batch_size * num_beams
    input_ids = torch.full((R, 1), decoder_start_token_id, dtype=torch.long)
    beam_scores = torch.full((batch_size, num_beams), -1e9, dtype=torch.float)
    beam_scores[:, ::gs] = 0
    beam_scores = beam_scores.view(-1)
    while True:
        logits = step_logits(input_ids).float()
        current_tokens = torch.zeros(R, dtype=torch.long)
        filled = torch.zeros(R, dtype=torch.bool)             # the new beam is a -inf tie-fill
        reordering_indices = torch.zeros(R, dtype=torch.long)
        cur_len = input_ids.shape[-1]
        for g in range(G):
            g0 = g * gs
            idx = [b * num_beams + i for b in range(batch_size) for i in range(g0, g0 + gs)]
            group_ids = input_ids[idx]
            scores = torch.log_softmax(logits[idx], dim=-1)
            for p in processors:
                if p == "min_length" and min_length is not None and min_length > -1:
                    scores = proc_min_length(group_ids, scores, min_length, model_eos_token_id)
                elif p == "forced_bos" and forced_bos_token_id is not None:
                    scores = proc_forced_bos(group_ids, scores, forced_bos_token_id)
                elif p == "forced_eos" and forced_eos_token_id is not None:
                    scores = proc_forced_eos(group_ids, scores, max_length, forced_eos_token_id)
                elif p == "inf_nan":
                    scores = proc_inf_nan(group_ids, scores)
            if diversity_penalty > 0.0:
                scores = proc_hamming_413(current_tokens, scores, g, diversity_penalty, num_beams, G)
            if cdp is not None:
                scores = cdp(group_ids, scores)
            scores = scores + beam_scores[idx].unsqueeze(-1).expand_as(scores)
            V = scores.shape[-1]
            if diversity_penalty > 0.0 and g > 0:
                for b in range(batch_size):
                    prev = filled[b * num_beams: b * num_beams + g0]
                    toks = current_tokens[b * num_beams: b * num_beams + g0][prev]
                    if len(toks) and torch.isfinite(scores[b * gs:(b + 1) * gs][:, toks]).any():
                        tie[b] = True
            scores = scores.view(batch_size, gs * V)
            top_s, top_i = torch.topk(scores, 2 * gs, dim=1, largest=True, sorted=True)
            next_indices = torch.div(top_i, V, rounding_mode="floor")
            next_tokens = top_i % V
            # BeamSearchScorerWithMemory.process with group_size = gs (:625-690)
            nb_scores = torch.zeros((batch_size, gs)); nb_tokens = torch.zeros((batch_size, gs), dtype=torch.long)
            nb_idx = torch.zeros((batch_size, gs), dtype=torch.long)
            for b in range(batch_size):
                beam_idx = 0
                broken = False
                for tok, sc, bi in zip(next_tokens[b].tolist(), top_s[b].tolist(), next_indices[b].tolist()):
                    bbi = b * gs + bi
                    hyps[b].add(group_ids[bbi].tolist() + [tok], sc, sc)
                    if broken or (eos_token_id is not None and tok == eos_token_id):
                        pass
                    else:
                        nb_scores[b, beam_idx] = sc; nb_tokens[b, beam_idx] = tok; nb_idx[b, beam_idx] = bbi
                        beam_idx += 1
                    if beam_idx == gs:
                        broken = True
                if beam_idx < gs:
                    raise ValueError(f"At most {gs} tokens can be equal to `eos_token_id: {eos_token_id}`.")
            beam_idx_flat = nb_idx.view(-1)
            beam_scores[idx] = nb_scores.view(-1)
            input_ids[idx] = group_ids[beam_idx_flat]
            current_tokens[idx] = nb_tokens.view(-1)
            filled[idx] = nb_scores.view(-1) == NEG_INF
            reordering_indices[idx] = num_beams * torch.div(beam_idx_flat, gs, rounding_mode="floor") + g0 + beam_idx_flat % gs
        input_ids = torch.cat([input_ids, current_tokens.unsqueeze(-1)], dim=-1)
        if reorder is not None:
            reorder(reordering_indices)
        if cur_len + 0 >= max_length or input_ids.shape[-1] >= max_length:
            break
    for b in range(batch_size):                                                   # finalize :705-725
        for beam_id in range(num_beams):
            bbi = b * num_beams + beam_id
            hyps[b].add(input_ids[bbi].tolist(), beam_scores[bbi].item(), float("nan"))
    if info is not None:
        info["tie_sensitive"] = tie
    return [[(s * (len(t) ** length_penalty), t, c) for (s, t, c) in h.beams if s > NEG_INF] for h in hyps]


def fm_index_generate_groups_oracle(model, index, input_ids, attention_mask, min_length=3, max_length=25,
                                    length_penalty=1.0, num_beams=3, diverse_bs_groups=2, diverse_bs_penalty=0.0,
                                    eos_token_id=None, force_decoding_from=None, always_allow_eos=False,
                                    disable_fm_index=False, stop_at_count=0,
                                    processors=("min_length", "forced_bos", "forced_eos", "inf_nan"), use_cache=False,
                                    info=None, **kw):
    """seal/beam_search.py:391-557 with diverse_bs_groups > 1 and keep_history=True on an HF BART model (the arguments
    of oracle.decode_oracle.fm_index_generate_oracle); with use_cache=True the decoder KV cache is permuted by 4.13's
    `reordering_indices` after every step."""
    cfg = model.config
    stepper = (HFBartCachedStepper if use_cache else HFBartStepper)(model, input_ids, attention_mask, num_beams)
    forced_bos = kw.pop("forced_bos_token_id", cfg.forced_bos_token_id)           # :415-418
    return group_beam_search_oracle(
        stepper, input_ids.shape[0], index, num_beams, diverse_bs_groups, diverse_bs_penalty, min_length, max_length,
        length_penalty, eos_token_id=eos_token_id if eos_token_id is not None else cfg.eos_token_id,
        pad_token_id=cfg.pad_token_id, decoder_start_token_id=cfg.decoder_start_token_id,
        model_eos_token_id=cfg.eos_token_id, forced_eos_token_id=cfg.forced_eos_token_id,
        forced_bos_token_id=forced_bos, force_decoding_from=force_decoding_from, stop_at_count=stop_at_count,
        always_allow_eos=always_allow_eos, disable_fm_index=disable_fm_index, processors=processors,
        reorder=stepper.reorder if use_cache else None, info=info)
