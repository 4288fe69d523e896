"""TEST INFRASTRUCTURE ONLY -- the top-k logits warp for the decode oracle (oracle/decode_oracle.py).

fm_index_generate(topk=k) (seal/beam_search.py:163-164, :249-253 of the reference) builds transformers'
`TopKLogitsWarper(k)` and applies it to each step's raw logits, after final_logits_bias and before log_softmax; the
processors, the index mask, the top-2B and the gather of the unconstrained scores follow unchanged.  The warp is restated
here from its arithmetic (the same in transformers 4.13 and 5.5):

    k_eff = min(max(k, 1), V);  tau = the k_eff-th largest value of the fp32 row;  x < tau  ->  -inf

(ties at tau kept, -0.0 == +0.0, -inf entries count as values).  Because it only rewrites the logits, the oracle is the
pinned constrained_beam_search_oracle driven by a stepper that warps what the model returns.
tests/golden/make_decode_topk_golden.py runs the reference's own fm_index_generate(topk=...) beside it and stores
tests/golden/decode_topk_golden.json.
"""
import contextlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.decode_oracle import (NEG_INF, HFBartCachedStepper, HFBartStepper,  # noqa: E402
                                  constrained_beam_search_oracle)


def topk_warp(logits, k):
    """TopKLogitsWarper(k)(input_ids, logits), restated (module docstring)"""
    k_eff = min(max(int(k), 1), logits.shape[-1])
    tau = torch.topk(logits, k_eff)[0][..., -1, None]
    return logits.masked_fill(logits < tau, NEG_INF)


class TopKStepper:
    """step_logits wrapper: the model's logits through topk_warp.  `gaps` (if a list) receives, per call, the per-row
    difference between the k-th and the (k+1)-th largest logit -- how far the row is from changing its kept set."""

    def __init__(self, stepper, k, gaps=None):
        self.stepper, self.k, self.gaps = stepper, k, gaps
        if hasattr(stepper, "reorder"):
            self.reorder = stepper.reorder

    def __call__(self, decoder_input_ids):
        x = self.stepper(decoder_input_ids).float()
        if self.gaps is not None and self.k < x.shape[-1]:
            top = torch.topk(x, self.k + 1)[0]
            with torch.no_grad():
                g = (top[:, self.k - 1] - top[:, self.k]).double()
            self.gaps.append(torch.nan_to_num(g, nan=float("inf")))
        return topk_warp(x, self.k)


@contextlib.contextmanager
def flat_index_ties():
    """torch.topk with equal values in ascending flat-index order -- the rule the CUDA kernels document for the order
    torch leaves unspecified -- for the duration of the block"""
    topk = torch.topk

    def stable_topk(x, k, dim=-1, largest=True, sorted=True):
        assert largest and sorted
        v, i = torch.sort(x, dim=dim, descending=True, stable=True)
        return v.narrow(dim, 0, k), i.narrow(dim, 0, k)

    torch.topk = stable_topk
    try:
        yield
    finally:
        torch.topk = topk


def fm_index_generate_topk_oracle(model, index, input_ids, attention_mask, min_length=3, max_length=25,
                                  length_penalty=1.0, num_beams=3, eos_token_id=None, force_decoding_from=None,
                                  always_allow_eos=False, disable_fm_index=False, stop_at_count=0, topk=0,
                                  processors=("min_length", "forced_bos", "forced_eos", "inf_nan"), use_cache=False,
                                  keep_history=True, transformers_output=False, info=None, flat_ties=False, **kw):
    """seal/beam_search.py:391-557 on an HF BART model with the arguments of
    oracle.decode_oracle.fm_index_generate_oracle plus `topk` (> 0: the warp on every step; 0: none).
    flat_ties=True orders equal scores by flat index in every top-k (flat_index_ties), as the CUDA kernels do.
    `info` (if a dict) receives two per-query lists:
      * "min_gap": the smallest gap between the k-th and (k+1)-th largest logit over the query's rows at every step
        (inf when topk is 0 or >= V);
      * "tie_sensitive": whether at some step a group of equal finite constrained scores in the top-2B either holds
        the last entry (it may continue below the cut) or holds both a candidate that became a beam and a non-EOS one
        that did not.  torch.topk leaves the order among equal values unspecified, so such a query's beams depend on
        it.  With a small k this is common at the first step: beams 1.. are copies of beam 0 at -1e9, and once beam 0
        has fewer than 2B finite candidates their tied candidates enter the list."""
    cfg = model.config
    stepper = (HFBartCachedStepper if use_cache else HFBartStepper)(model, input_ids, attention_mask, num_beams)
    gaps = [] if info is not None else None
    trace = [] if info is not None else None
    if topk > 0:
        stepper = TopKStepper(stepper, int(topk), gaps)
    forced_bos = kw.pop("forced_bos_token_id", cfg.forced_bos_token_id)           # :415-418
    with flat_index_ties() if flat_ties else contextlib.nullcontext():
        out = constrained_beam_search_oracle(
            stepper, input_ids.shape[0], index, num_beams, min_length, max_length, length_penalty,
            eos_token_id=eos_token_id if eos_token_id is not None else cfg.eos_token_id,
            pad_token_id=cfg.pad_token_id, decoder_start_token_id=cfg.decoder_start_token_id,
            model_eos_token_id=cfg.eos_token_id, forced_eos_token_id=cfg.forced_eos_token_id,
            forced_bos_token_id=forced_bos, force_decoding_from=force_decoding_from, stop_at_count=stop_at_count,
            always_allow_eos=always_allow_eos, disable_fm_index=disable_fm_index, processors=processors,
            reorder=getattr(stepper, "reorder", None) if use_cache else None, trace=trace, keep_history=keep_history,
            transformers_output=transformers_output)
    if info is not None:
        Q = input_ids.shape[0]
        min_gap = [float("inf")] * Q
        for g in gaps or []:
            per_q = g.view(Q, -1).min(dim=1).values.tolist()
            min_gap = [min(a, b) for a, b in zip(min_gap, per_q)]
        info["min_gap"] = min_gap
        eos = eos_token_id if eos_token_id is not None else cfg.eos_token_id
        info["tie_sensitive"] = [any(_tie_sensitive(t["top_constrained"][q].tolist(), t["top_tokens"][q].tolist(),
                                                    num_beams, eos) for t in trace if "top_constrained" in t)
                                 for q in range(Q)]
    return out


def _tie_sensitive(scores, tokens, num_beams, eos):
    """see fm_index_generate_topk_oracle's `info`"""
    beam, nb = [], 0
    for tok in tokens:
        became = tok != eos and nb < num_beams
        nb += became
        beam.append(None if tok == eos else became)
    last = len(scores) - 1
    for i, s in enumerate(scores):
        if s == NEG_INF:
            continue
        group = [j for j, t in enumerate(scores) if t == s]
        if len(group) > 1 and (last in group or len({beam[j] for j in group} - {None}) > 1):
            return True
    return False
