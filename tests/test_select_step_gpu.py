"""GPU: one decode step's selection (topk_rows_kernel + select_merge_kernel) and the lm_head statistics epilogue
(HeadEpi) against a float64 step reference.

The step runs through sealdec_debug_select_step, which takes the same kernel dispatch as a generate
(launch_select_step) on inputs chosen here; every output and scratch buffer starts as NaN / all-ones bits.

Reference (HF's own arithmetic, seal/beam_search.py:244-332 and BeamSearchScorerWithMemory.process :614-703): p64 is
the float64 log-softmax of the fp32 logits passed through the processors (oracle.decode_oracle's proc_*), rounded to
fp32; the candidate score is the fp32 sum fl32(p32 + beam_score), as HF's `processed + beam_scores`.  At the first step
beams 1.. carry -1e9, so their candidates tie exactly in fp32 (ulp(1e9) = 64) and the reference sees those ties too.

Bounds (derived from the kernels' summation order, not measured; u = 2^-24):
  * row_max equals the fp32 row maximum bit for bit (a max is exact).
  * |row_logsum - logsumexp64| <= E_ls = rel_se / (1 - rel_se) + ulp(|L|), logf being good to 1 ulp, with
        rel_se * S = u * sum_i e_i |d_i|  +  (4u + 5u * n_resc) * S  +  gamma(n_add) * S  +  n * 2^-148,
    d_i = x_i - max, e_i = exp(d_i), S = sum e_i.  The first term is the rounding of every exponent argument: a term
    passes through expf(x - mx_t) and the rescales expf(mx_t - mx_t') ... expf(mx_T - max), each argument rounded to
    half an ulp of its magnitude, and the magnitudes add up to |d_i| because the running maxima only grow.  expf is
    good to 2 ulp (4u relative), each rescale costs 4u + a rounded product (u); n_resc rescales reach a term:
    ceil(V / (16 THREADS)) four-float4 batches + the tail iterations + the block merge when streaming, or the tiles
    of a thread + 1 with head statistics.  n_add is the longest addition chain: 4 (16-value tree) + batches +
    4 * tail iterations + 5 (warp) + THREADS / 32 (block, sequential), or with head statistics 19 (the epilogue:
    a pair add, 16 sequential adds, 2 shuffle adds) + tiles per thread + 5 + THREADS / 32.  The last term covers expf
    results in the subnormal range.
  * every candidate or recorded score s: |s - s_ref| <= delta = E_ls + ulp(|x - max|) + ulp(|p|) + ulp(|s|)
    (the kernel rounds x - max, then - logsum, then + beam_score; the reference rounds p64 and the sum).  Diverse-group
    candidates whose penalty is applied add 2 ulp(|s|) for the two more roundings.

Selection checks, per candidate list and per query (or group):
  * exact, on the kernel's own scores: p_k = fl32(fl32(x - row_max) - row_logsum) through the processors, s_k =
    fl32(p_k + beam_score) is what the kernels compute (no operation there can be contracted), so each list must be
    exactly the top-2B of s_k over its rows ordered by (score descending, flat index ascending), and the records
    exactly the merge of the lists -- ties, the staging-buffer overflow and its sub-rounds, the first step's
    pruning and the fill-ins included;
  * membership against the float64 reference: the k-th kernel entry scores, in the reference, at least the
    reference's k-th minus 2 delta, and nothing the kernel left out scores more than its last entry plus 2 delta;
  * exact against the reference where no two reference scores next to each other among the top 2B + 1 are within
    2 delta (or tie exactly on identical inputs), and in the constructed exact-tie cases;
  * fill-ins: the lowest flat indices that are not finite allowed candidates, with the unconstrained score
    (G = 1, within delta of the reference) or -inf (G > 1), valid 0;
  * BeamSearchScorerWithMemory.process exactly: new beams, parents, tokens, the ancestry layout, pw, EOS handling and
    the error flag; record and new-beam lo / hi against the oracle LF step (a backward step on the parent's
    (lo, hi - 1)).

Not built: the `count_before > 0` merge of the overflow path (decode_kernels.cuh, topk_rows_kernel).  A generate
cannot reach it: at the first step every row of a query has the same mask, and a row that stages more than BUF/2 is
merged before the next row starts; at later steps a CTA has one row.
"""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32MAX = float(np.finfo(np.float32).max)
EOS, PAD, START, SHIFT = 2, 1, 2, 10
GN = 128
REPORT = []


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    yield
    for line in REPORT:
        print(line)


@pytest.fixture(scope="module")
def index(small_corpus):
    """one small real index (device FM index + oracle) and prefixes of real documents as parent states"""
    from oracle.fm_oracle import OracleIndex
    from seal_b200.index import FMIndex
    seqs = [d.tolist() for d in small_corpus]
    idx = FMIndex(); idx.initialize(seqs, in_memory=True); idx.to_device(0)
    ora = OracleIndex(seqs)
    return idx, ora, seqs


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


def gamma(n):
    return n * U / (1.0 - n * U)


def make_params(B, T, min_length=-1, forced_eos=-1, forced_bos=-1, stop_at_count=0, always_allow_eos=0,
                disable_fm_index=0):
    from seal_b200._lib import DecParams
    return DecParams(B, min_length, T, 1.0, EOS, PAD, START, EOS, forced_eos, forced_bos, stop_at_count,
                     always_allow_eos, disable_fm_index, 1, 0, None, SHIFT)


def run_step(fm_h, s):
    """sealdec_debug_select_step on the case dict `s`; returns every output"""
    from seal_b200._lib import GroupParams, lib, check
    p, Q, V, cur = s["p"], s["Q"], s["V"], s["cur_len"]
    B, T = p.num_beams, p.max_length
    R, K = Q * B, 2 * B
    o = dict(row_max=np.empty(R, np.float32), row_logsum=np.empty(R, np.float32), row_rule=np.empty(R, np.uint8),
             cand_val=np.empty((R, K), np.float32), cand_idx=np.empty((R, K), np.int32), cand_cnt=np.empty(R, np.int32),
             lists=np.zeros(1, np.int32), bs_out=np.empty(R, np.float32), tok_out=np.empty((R, T), np.int32),
             anc_out=np.empty((R, T), np.int32), lo_out=np.empty(R, np.uint64), hi_out=np.empty(R, np.uint64),
             pw_out=np.empty(R, np.uint64), rec_score=np.empty((Q, K), np.float32), rec_len=np.empty((Q, K), np.int32),
             rec_tok=np.empty((Q, K, T), np.int32), rec_valid=np.empty((Q, K), np.uint8),
             rec_lo=np.empty((Q, K), np.uint64), rec_hi=np.empty((Q, K), np.uint64), err=np.zeros(1, np.int32))
    ptr = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data
    keep = [np.ascontiguousarray(s[k]) if s.get(k) is not None else None
            for k in ("logits", "head_stats", "masks", "occ", "bs", "tokens", "anc", "lo", "hi", "pw")]
    grp = GroupParams(s["G"], s["penalty"])
    check(lib.sealdec_debug_select_step(
        fm_h if not p.disable_fm_index else None, C.byref(p), C.byref(grp), Q, V, cur, int(s["shared"]),
        int(s["ignored"]), *[ptr(a) for a in keep],
        *[o[k].ctypes.data for k in ("row_max", "row_logsum", "row_rule", "cand_val", "cand_idx", "cand_cnt", "lists",
                                     "bs_out", "tok_out", "anc_out", "lo_out", "hi_out", "pw_out", "rec_score",
                                     "rec_len", "rec_tok", "rec_valid", "rec_lo", "rec_hi", "err")]))
    return o


# ---- the float64 step reference --------------------------------------------------------------------------------------
def processors(p, cur_len, P):
    """HF 4.13 processors in the order of oracle.decode_oracle (MinLength, ForcedBOS, ForcedEOS, InfNanRemove) on the
    [R][V] log-probabilities P (float64 or float32, in place)"""
    if p.min_length > -1 and cur_len < p.min_length:
        P[:, p.model_eos_token_id] = -np.inf
    if p.forced_bos_token_id >= 0 and cur_len == 1:
        keep = np.full_like(P, -np.inf); keep[:, p.forced_bos_token_id] = 0; P[...] = keep
    if p.forced_eos_token_id >= 0 and cur_len == p.max_length - 1:
        keep = np.full_like(P, -np.inf); keep[:, p.forced_eos_token_id] = 0; P[...] = keep
    P[np.isnan(P)] = 0.0
    P[P == np.inf] = F32MAX
    return P


def allowed_and_rules(s):
    p, Q, V, cur = s["p"], s["Q"], s["V"], s["cur_len"]
    B = p.num_beams; R = Q * B
    fb_step = p.forced_bos_token_id >= 0 and cur == 1
    eff_len = cur - (1 if p.forced_bos_token_id >= 0 else 0)
    rules = np.zeros(R, np.uint8)
    if p.disable_fm_index:
        return np.ones((R, V), bool), rules
    A = np.zeros((R, V), bool)
    if fb_step:
        A[:, p.forced_bos_token_id] = True
        return A, rules
    bits = lambda words: np.unpackbits(words.view(np.uint8), bitorder="little")[:V].astype(bool)
    for r in range(R):
        if eff_len > 1:
            last = int(s["tokens"][r, cur - 1])
            ended = last in (p.eos_token_id, p.pad_token_id)
            count = 0 if ended else int(s["pw"][r])
            if p.stop_at_count > 0 and count <= p.stop_at_count:
                rules[r] = 1
            elif ended:
                rules[r] = 2
        if rules[r] == 1:
            A[r, p.eos_token_id] = True
        elif rules[r] == 2:
            A[r, p.pad_token_id] = True
        else:
            A[r] = bits(s["occ"] if eff_len == 1 else s["masks"][r])
        if p.always_allow_eos:
            A[r, p.eos_token_id] = True
    return A, rules


def step_sizes(s):
    """(THREADS, rescales, additions) of the statistics path the step takes"""
    V = s["V"]
    threads = 512 if s["cur_len"] == 1 else 256
    if s.get("head_stats") is not None:
        per = -(-(-(-V // GN)) // threads)
        return threads, per + 1, 19 + per + 5 + threads // 32
    batches = V // (16 * threads)
    tail = -(-(V - batches * 16 * threads) // (4 * threads))
    return threads, batches + tail + 1, 4 + batches + 4 * tail + 5 + threads // 32


def reference(s):
    """float64 row statistics, p32, reference scores and per-candidate bound"""
    p, Q, V, cur = s["p"], s["Q"], s["V"], s["cur_len"]
    B = p.num_beams; R = Q * B
    lrow = (np.arange(R) // B) if s["shared"] else np.arange(R)
    _, n_resc, n_add = step_sizes(s)
    with np.errstate(all="ignore"):
        if s["ignored"]:
            X = np.zeros((R, V)); m = np.zeros(R); L = np.zeros(R); E = np.zeros(R); D = np.zeros((R, V))
            P = np.zeros((R, V))
        else:
            X = s["logits"][lrow].astype(np.float64)
            m = X.max(1)
            D = X - m[:, None]
            e = np.exp(D)
            S = e.sum(1)
            L = np.log(S)
            fin = np.where(np.isfinite(D), D, 0.0)
            rel = (U * (e * np.abs(fin)).sum(1) + (4 * U + 5 * U * n_resc) * S + gamma(n_add) * S + V * 2.0 ** -148) / S
            E = rel / (1 - rel) + ulp(L)
            E = np.where(np.isfinite(L) & np.isfinite(m), E, 0.0)
            P = D - L[:, None]
        P = processors(p, cur, P)
        P32 = P.astype(np.float32)
        bs = s["bs"].astype(np.float32)
        Sref = P32 + bs[:, None]
        delta = E[:, None] + np.where(np.isfinite(D), ulp(D), 0) + ulp(P32) + ulp(Sref)
    return dict(m=m, L=L, E=E, P32=P32, S=Sref, delta=delta, X=X)


def kernel_scores(s, o, stat_rows):
    """the kernels' own scores from their row statistics: fl32(fl32(x - row_max) - row_logsum), processors, + bs"""
    p, Q, V, cur = s["p"], s["Q"], s["V"], s["cur_len"]
    B = p.num_beams; R = Q * B
    lrow = (np.arange(R) // B) if s["shared"] else np.arange(R)
    with np.errstate(all="ignore"):
        if s["ignored"]:
            Pk = np.zeros((R, V), np.float32)
        else:
            X = s["logits"][lrow].astype(np.float32)
            Pk = (X - o["row_max"][stat_rows][:, None]) - o["row_logsum"][stat_rows][:, None]
        Pk = processors(p, cur, Pk)
        return Pk, Pk + s["bs"].astype(np.float32)[:, None]


def top_k(scores, flats, k):
    order = np.lexsort((flats, -scores.astype(np.float64)))[:k]
    return scores[order], flats[order]


def lf(ora, tok, lo, hi):
    l, r = ora.backward_search_step(int(tok) + SHIFT, int(lo), int(hi) - 1)
    return l, r + 1


def check_step(s, o, ora, label, exact_ties=False):
    p, Q, V, cur = s["p"], s["Q"], s["V"], s["cur_len"]
    B, T = p.num_beams, p.max_length
    R, K = Q * B, 2 * B
    G, pen = s["G"], s["penalty"]
    gs, Kg = B // G, 2 * (B // G)
    fm_on = not p.disable_fm_index
    fb_step = p.forced_bos_token_id >= 0 and cur == 1
    bs = s["bs"].astype(np.float32)
    A, rules = allowed_and_rules(s)
    ref = reference(s)
    lists = int(o["lists"][0])
    exp_lists = (2 if gs > 1 else 1) if (cur == 1 and G > 1) else 1 if cur == 1 else B
    assert lists == exp_lists, (label, lists)
    worst = {"logsum": 0.0, "score": 0.0}

    # ---- row statistics; which rows the kernel computed -------------------------------------------------------------
    if cur == 1:
        if G > 1:
            rows_listed = np.array([q * B + j for q in range(Q) for j in range(lists)])
        else:
            rows_listed = np.arange(R)
        stat_rows = np.repeat(np.arange(Q) * B, B)              # every row of a query reads the same logits row
    else:
        rows_listed = np.arange(R)
        stat_rows = np.arange(R)
    computed = np.zeros(R, bool); computed[rows_listed] = True
    written = o["row_rule"] != 0xFF                         # the rule byte starts as 0xFF
    assert not (written & ~computed).any(), (label, "statistics written for a row no list covers")
    if cur > 1:
        assert written.all(), (label, "a row's statistics were not written")
    for r in np.nonzero(written)[0]:
        if not s["ignored"]:
            mref = np.nanmax(s["logits"][r // B if s["shared"] else r]) if np.isnan(ref["m"][r]) else ref["m"][r]
            assert o["row_max"][r] == np.float32(mref) or (np.isneginf(mref) and np.isneginf(o["row_max"][r])), \
                (label, r, o["row_max"][r], mref)
            if np.isfinite(ref["L"][r]) and np.isfinite(ref["m"][r]):
                err = abs(float(o["row_logsum"][r]) - ref["L"][r])
                assert err <= ref["E"][r], (label, r, err, ref["E"][r])
                worst["logsum"] = max(worst["logsum"], err / ref["E"][r])
        else:
            assert o["row_max"][r] == 0 and o["row_logsum"][r] == 0
        assert o["row_rule"][r] == rules[r], (label, r, o["row_rule"][r], rules[r])
    if cur == 1:                                    # rows that share logits and mask share their statistics
        for r in np.nonzero(written)[0]:
            q0 = (r // B) * B
            assert o["row_max"][r] == o["row_max"][q0] and (
                o["row_logsum"][r] == o["row_logsum"][q0] or np.isnan(o["row_logsum"][q0])), (label, r)

    lrow = (np.arange(R) // B) if s["shared"] else np.arange(R)
    keys = {}
    sig = np.array([keys.setdefault((b"" if s["ignored"] else s["logits"][lrow[r]].tobytes(), bs[r].tobytes()), len(keys))
                    for r in range(R)])                     # rows with bit-identical inputs
    Pk, Sk = kernel_scores(s, o, stat_rows)
    cand = A & (Sk > -np.inf)
    assert np.array_equal(cand, A & (ref["S"] > -np.inf)), (label, "finite candidates differ from the reference")
    with np.errstate(invalid="ignore"):
        dev = np.where(cand, np.abs(Sk.astype(np.float64) - ref["S"]), 0.0)
        ratio = np.where(cand, dev / np.maximum(ref["delta"], 1e-300), 0.0)
    worst["score"] = float(ratio.max(initial=0.0))
    assert worst["score"] <= 1.0, (label, "score outside delta", np.unravel_index(np.argmax(ratio), ratio.shape))

    # ---- candidate lists: exactly the top-K of the kernel's own scores over the list's rows -------------------------
    def list_rows(q, l):
        if cur == 1 and G == 1:
            return list(range(q * B, q * B + B))
        return [q * B + l]

    for q in range(Q):
        for l in range(lists):
            rows = list_rows(q, l)
            sc = np.concatenate([Sk[r][cand[r]] for r in rows])
            fl = np.concatenate([(r - q * B) * V + np.nonzero(cand[r])[0] for r in rows]).astype(np.int64)
            ev, ei = top_k(sc, fl, K)
            gi = q * lists + l
            n = o["cand_cnt"][gi]
            assert n == len(ev), (label, q, l, n, len(ev))
            assert np.array_equal(o["cand_idx"][gi, :n], ei), (label, "list", q, l, o["cand_idx"][gi, :n], ei)
            assert np.array_equal(o["cand_val"][gi, :n].view(np.uint32), ev.view(np.uint32)), (label, "list values", q, l)
            if cur == 1 and G == 1 and n == K:      # a row the kernel skipped could not have entered the list
                for r in rows:
                    if not written[r]:
                        assert bs[r] < ev[-1], (label, "pruned row", r)

    # ---- the merge, group by group, the fill-ins and process --------------------------------------------------------
    n_exact = 0
    new_tok = np.full((Q, B), -1)
    err = 0
    for q in range(Q):
        for g in range(G):
            b0 = g * gs
            rows = list(range(q * B + b0, q * B + b0 + gs))
            counts = {}
            if pen > 0:
                for t in new_tok[q, :b0]:
                    if t >= 0:
                        counts[int(t)] = counts.get(int(t), 0) + 1
            sc_k, sc_r, dl, fl, tw = [], [], [], [], []
            for r in rows:
                v = np.nonzero(cand[r])[0]
                sk = Sk[r][v].copy(); sr = ref["S"][r][v].copy(); d = ref["delta"][r][v].copy()
                cnt = np.zeros(len(v), np.int64)
                for i, t in enumerate(v if counts else ()):
                    c = counts.get(int(t), 0)
                    if c:
                        pp = np.float32(pen) * np.float32(c)
                        sk[i] = np.float32(np.float32(Pk[r][t] - pp) + bs[r])
                        sr[i] = np.float32(np.float32(ref["P32"][r][t] - pp) + bs[r])
                        d[i] += 2 * ulp(sr[i])
                        cnt[i] = c
                # candidates with bit-identical kernel inputs (logit, row statistics, beam score, penalty) tie in
                # the kernel exactly when they tie in the reference, and so do candidates whose whole interval
                # p32 +- (delta - ulp(s)) rounds, with the beam score, to the same fp32 value (-1e9 + p)
                dp = d - ulp(sr)
                with np.errstate(invalid="ignore"):
                    base = ref["P32"][r][v].astype(np.float64) + float(bs[r])
                    stable = ((base - dp).astype(np.float32) == (base + dp).astype(np.float32)) & (cnt == 0)
                tw.append(np.stack([ref["X"][r][v], np.full(len(v), float(sig[r])), cnt.astype(np.float64),
                                    stable.astype(np.float64)], 1))
                sc_k.append(sk); sc_r.append(sr); dl.append(d); fl.append((r - q * B) * V + v)
            sc_k, sc_r, dl, fl, tw = map(np.concatenate, (sc_k, sc_r, dl, fl, tw))
            fl = fl.astype(np.int64)
            order = np.lexsort((fl, -sc_k.astype(np.float64)))
            kv, ki = sc_k[order][:Kg], fl[order][:Kg]
            want = len(ki)
            hs = o["rec_score"][q, 2 * b0:2 * b0 + Kg]
            htok = o["rec_tok"][q, 2 * b0:2 * b0 + Kg]
            hval = o["rec_valid"][q, 2 * b0:2 * b0 + Kg]
            # merged list: exact given the kernel's scores
            assert np.array_equal(hs[:want].view(np.uint32), kv.view(np.uint32)), (label, "records", q, g, hs[:want], kv)
            assert (hval[:want] == 1).all() and (hval[want:] == 0).all(), (label, "valid", q, g)
            # against the float64 reference: membership within 2 delta, exact where unambiguous
            rorder = np.lexsort((fl, -sc_r.astype(np.float64)))
            rv, ri, rd = sc_r[rorder], fl[rorder], dl[rorder]
            pos = {int(f): i for i, f in enumerate(fl)}
            for k in range(want):
                i = pos[int(ki[k])]
                assert sc_r[i] >= rv[k] - dl[i] - rd[k], (label, "membership", q, g, k)
            if want:
                last = pos[int(ki[-1])]
                left = np.ones(len(fl), bool); left[[pos[int(f)] for f in ki]] = False
                assert not (left & (sc_r > sc_k[last] + dl + dl[last])).any(), (label, "left out", q, g)
            top = min(Kg + 1, len(rv))
            rt = tw[rorder]
            gaps_ok = all(rv[i] - rv[i + 1] > rd[i] + rd[i + 1] or
                          (rv[i] == rv[i + 1] and (np.array_equal(rt[i, :3], rt[i + 1, :3]) or rt[i, 3] * rt[i + 1, 3] > 0))
                          for i in range(top - 1))
            if gaps_ok:
                assert np.array_equal(ri[:want], ki), (label, "not the reference's list", q, g, ri[:want], ki)
                n_exact += 1
            # fill-ins: the lowest flat indices that are not finite allowed candidates
            fill = []
            f = b0 * V
            while len(fill) < Kg - want and f < (b0 + gs) * V:
                r, v = q * B + f // V, f % V
                if not cand[r, v]:
                    fill.append(f)
                f += 1
            merged = list(ki) + fill
            assert len(merged) == Kg
            for k, f in enumerate(merged):
                r, v = q * B + f // V, f % V
                assert htok[k, cur] == v and np.array_equal(htok[k, :cur], s["tokens"][r, :cur]), (label, "tokens", q, k)
                assert (htok[k, cur + 1:] == PAD).all() and o["rec_len"][q, 2 * b0 + k] == cur + 1
                if k >= want:
                    if G == 1:
                        assert hs[k] == Sk[r, v] or (np.isnan(hs[k]) and np.isnan(Sk[r, v])), (label, "fill-in", q, k)
                        if np.isfinite(ref["S"][r, v]):
                            assert abs(float(hs[k]) - ref["S"][r, v]) <= ref["delta"][r, v], (label, "fill-in", q, k)
                        else:
                            assert hs[k] == ref["S"][r, v]
                    else:
                        assert hs[k] == -np.inf, (label, "grouped fill-in", q, k)
                # record LF
                el, eh = 0, 0
                if fm_on and k < want and not fb_step:
                    el, eh = lf(ora, v, s["lo"][r], s["hi"][r])
                assert (o["rec_lo"][q, 2 * b0 + k], o["rec_hi"][q, 2 * b0 + k]) == (el, eh), (label, "record lo/hi", q, k)
            # process: the first gs non-EOS picks become the group's beams
            nb = 0
            for k, f in enumerate(merged):
                if nb == gs:
                    break
                v = f % V
                if v == p.eos_token_id:
                    continue
                pr = q * B + f // V
                nr = q * B + b0 + nb
                new_tok[q, b0 + nb] = v
                assert o["bs_out"][nr].view(np.uint32) == np.float32(hs[k]).view(np.uint32), (label, "beam score", nr)
                assert np.array_equal(o["tok_out"][nr, :cur], s["tokens"][pr, :cur]) and o["tok_out"][nr, cur] == v
                assert (o["tok_out"][nr, cur + 1:] == PAD).all()
                assert np.array_equal(o["anc_out"][nr, :cur - 1], s["anc"][pr, :cur - 1]) and o["anc_out"][nr, cur - 1] == pr
                assert (o["anc_out"][nr, cur:] == -1).all(), (label, "ancestry written past cur_len", nr)
                if fb_step:
                    el, eh, epw = s["lo"][pr], s["hi"][pr], s["pw"][pr]
                else:
                    el, eh = lf(ora, v, s["lo"][pr], s["hi"][pr]) if fm_on else (0, 0)
                    epw = s["hi"][pr] - s["lo"][pr]
                assert (o["lo_out"][nr], o["hi_out"][nr], o["pw_out"][nr]) == (el, eh, epw), (label, "beam lo/hi/pw", nr)
                nb += 1
            for j in range(nb, gs):
                nr = q * B + b0 + j
                err = 1
                assert o["bs_out"][nr] == 0 and (o["lo_out"][nr], o["hi_out"][nr], o["pw_out"][nr]) == (0, 0, 0)
                assert (o["tok_out"][nr] == -1).all()
    assert o["err"][0] == err, (label, "error flag", o["err"][0], err)
    if exact_ties:
        assert n_exact == Q * G, (label, "the constructed ties were not checked exactly", n_exact)
    REPORT.append(f"{label}: worst |logsum err|/E_ls {worst['logsum']:.3f}, worst |s - s_ref|/delta "
                  f"{worst['score']:.3f}, lists equal to the reference exactly: {n_exact}/{Q * G}")
    return worst


# ---- case construction -----------------------------------------------------------------------------------------------
def words_of(A):
    V = A.shape[-1]
    W = (V + 31) // 32
    pad = np.zeros(A.shape[:-1] + (W * 32,), bool); pad[..., :V] = A
    return np.packbits(pad, axis=-1, bitorder="little").view(np.uint32).reshape(A.shape[:-1] + (W,))


def walks(seqs, rng, R, n):
    """R prefixes of n tokens of real documents: tokens rows [START] + prefix, SA ranges of the prefix and pw"""
    return [seqs[int(rng.integers(len(seqs)))][int(o):int(o) + n] for o in rng.integers(0, 20, size=R)]


def base_case(index, rng, B, V, Q, cur_len=3, T=10, G=1, penalty=0.0, **pkw):
    """a later step (cur_len >= 2) with parent states from real walks"""
    _, ora, seqs = index
    R = Q * B
    p = make_params(B, T, **pkw)
    tokens = np.full((R, T), PAD, np.int32)
    lo = np.zeros(R, np.uint64); hi = np.zeros(R, np.uint64); pw = np.zeros(R, np.uint64)
    for r, w in enumerate(walks(seqs, rng, R, cur_len - 1)):
        tokens[r, 0] = START; tokens[r, 1:cur_len] = w
        lo[r], hi[r] = ora.get_range(w)
        pl, ph = ora.get_range(w[:-1])
        pw[r] = ph - pl
    anc = np.tile(np.arange(R, dtype=np.int32)[:, None], (1, T))
    anc[:, :cur_len - 1] = rng.integers(0, R, size=(R, cur_len - 1))
    bs = (-rng.uniform(0.5, 8.0, size=R)).astype(np.float32)
    return dict(p=p, Q=Q, V=V, cur_len=cur_len, G=G, penalty=penalty, shared=False, ignored=False, head_stats=None,
                logits=None, masks=None, occ=None, bs=bs, tokens=tokens, anc=anc, lo=lo, hi=hi, pw=pw)


def random_masks(rng, R, V, counts):
    A = np.zeros((R, V), bool)
    for r in range(R):
        n = min(counts[r % len(counts)], V)
        A[r, rng.choice(V, size=n, replace=False)] = True
    M = words_of(A)
    if V & 31:                                       # bits past V in the last word must be ignored
        M[::2, -1] |= np.uint32(0xFFFFFFFF) << np.uint32(V & 31)
    return M


def logits_rows(rng, R, V, kinds):
    X = (rng.standard_normal((R, V)) * 3.0).astype(np.float32)
    for r in range(R):
        kind = kinds[r % len(kinds)]
        if kind == "coarse":                         # many exact ties inside the row, at every rank
            X[r] = np.round(X[r] * 2) / 2
        elif kind == "minus50":
            X[r] -= 50.0
        elif kind == "plus50":
            X[r] += 50.0
        elif kind == "constant":
            X[r] = 1.5
    return X


def run_and_check(index, s, label, exact_ties=False):
    idx = index[0]
    o = run_step(idx._dev(), s)
    return check_step(s, o, index[1], label, exact_ties)


LATER_B = [1, 2, 15, 16, 32]
LATER_V = [50265, 50272, 4099, 130]


@pytest.mark.parametrize("V", LATER_V)
@pytest.mark.parametrize("B", LATER_B)
def test_later_step_vs_float64(index, B, V):
    """one CTA per row (256 threads, BUF 4096): allowed tokens per row 0, 1, 2B-1, 2B, 2B+1, 2048, 2049, 4096, 4097 and
    all of V; logits smooth, on a coarse grid (ties at every rank) and shifted by -50 / +50"""
    rng = np.random.default_rng(B * 100003 + V)
    K = 2 * B
    counts = [0, 1, K - 1, K, K + 1, 2048, 2049, 4096, 4097, V]
    Q = max(2, -(-len(counts) // B))
    s = base_case(index, rng, B, V, Q)
    R = Q * B
    s["masks"] = random_masks(rng, R, V, counts)
    s["logits"] = logits_rows(rng, R, V, ["smooth", "minus50", "coarse", "plus50"])
    run_and_check(index, s, f"later B={B} V={V}")


def test_later_step_tie_cases(index):
    """a constant row with every token allowed (the top-2B are the 2B lowest ids, across the sub-round merges), values
    duplicated at the K-th boundary, and two beams with the same logits and the same score"""
    rng = np.random.default_rng(11)
    B, V = 15, 50265
    K = 2 * B
    s = base_case(index, rng, B, V, Q=2)
    R = 2 * B
    X = logits_rows(rng, R, V, ["smooth"])
    A = np.zeros((R, V), bool)
    bs = np.full(R, -400.0, np.float32)
    A[0] = True; X[0] = 0.25; bs[0] = -1.0                   # constant, all allowed
    A[1] = True; X[1] = -3.0; X[1, 5000:5000 + K + 7] = 4.0  # K + 7 tied leaders: the K-th boundary falls inside
    bs[1] = -1.5
    A[2, rng.choice(V, 3000, replace=False)] = True
    X[2, A[2]] = np.round(X[2, A[2]])                         # integer logits: long runs of ties
    A[B] = A[B + 1] = rng.random(V) < 0.3                     # second query, beams 0 and 1: identical rows and scores
    X[B + 1] = X[B]; bs[B] = bs[B + 1] = -0.5
    A[B + 2] = True; X[B + 2] = -60.0                         # a constant row below 0
    s["masks"] = words_of(A); s["logits"] = X; s["bs"] = bs
    run_and_check(index, s, "ties later", exact_ties=True)


@pytest.mark.parametrize("n_occ", [8192, 8193, "index", 5])
@pytest.mark.parametrize("B", [4, 15])
def test_first_step_vs_float64(index, B, n_occ):
    """512 threads, BUF 8192, logits shared by a query's beams, one CTA per query, beams 1.. at -1e9.  n_occ = 5 (< 2B):
    rows 1.. are not pruned, and their candidates tie exactly at -1e9 and must come out in flat-index order."""
    idx, ora, _ = index
    rng = np.random.default_rng(B * 7 + (n_occ if isinstance(n_occ, int) else 1))
    V, Q, T = 50265, 3, 10
    s = base_case(index, rng, B, V, Q, cur_len=1, T=T)
    R = Q * B
    s["tokens"][:] = PAD; s["tokens"][:, 0] = START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["anc"] = np.tile(np.arange(R, dtype=np.int32)[:, None], (1, T))
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    A = np.zeros(V, bool)
    if n_occ == "index":
        A[[t for t in idx.occurring_distinct if 0 <= t < V]] = True
    else:
        A[rng.choice(V, n_occ, replace=False)] = True
    s["occ"] = words_of(A)
    s["shared"] = True
    X = (rng.standard_normal((Q, V)) * 2.0).astype(np.float32)
    X[1] -= 50.0
    if n_occ == 5:                                            # keep p > -31: fl32(p - 1e9) = -1e9 exactly
        X = np.clip(X, -4, 4) - (50.0 * (np.arange(Q) == 1))[:, None].astype(np.float32)
    s["logits"] = X
    run_and_check(index, s, f"first B={B} occ={n_occ}", exact_ties=n_occ == 5)


def test_first_step_mask_is_not_a_row_mask(index):
    """logits_shared = 0 at cur_len 1 (the compact first step turned off): one logits row per beam"""
    idx, ora, _ = index
    rng = np.random.default_rng(3)
    B, V, Q, T = 8, 4099, 2, 6
    s = base_case(index, rng, B, V, Q, cur_len=1, T=T)
    R = Q * B
    s["tokens"][:] = PAD; s["tokens"][:, 0] = START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    s["occ"] = words_of(rng.random(V) < 0.5)
    s["logits"] = np.repeat((rng.standard_normal((Q, V)) * 2).astype(np.float32), B, axis=0)
    run_and_check(index, s, "first unshared")


PROC_CASES = {
    "min_length": dict(pkw=dict(min_length=5)),
    "forced_eos_dense": dict(pkw=dict(forced_eos=EOS), cur_len=9),
    "forced_eos_dead_step": dict(pkw=dict(forced_eos=EOS), cur_len=9, ignored=True),
    "stop_at_count": dict(pkw=dict(stop_at_count=40)),
    "always_allow_eos": dict(pkw=dict(always_allow_eos=1)),
    "disable_fm_index": dict(pkw=dict(disable_fm_index=1)),
    "ended_rows": dict(pkw=dict()),
    "invalid_values": dict(pkw=dict()),
    "score_minus_1e9": dict(pkw=dict(), bs=-1e9),
    "score_minus_300": dict(pkw=dict(), bs=-300.0),
}


@pytest.mark.parametrize("name", list(PROC_CASES))
def test_processors_and_rules(index, name):
    cfg = PROC_CASES[name]
    rng = np.random.default_rng(len(name))
    B, V, Q = 4, 4099, 3
    s = base_case(index, rng, B, V, Q, cur_len=cfg.get("cur_len", 3), **cfg["pkw"])
    R = Q * B
    s["masks"] = random_masks(rng, R, V, [3, 20, 200, 1, 0, 9])
    s["logits"] = logits_rows(rng, R, V, ["smooth", "minus50"])
    if cfg.get("ignored"):
        s["ignored"] = True; s["logits"] = None
    if "bs" in cfg:
        s["bs"] = (cfg["bs"] - rng.uniform(0, 3, size=R)).astype(np.float32) if cfg["bs"] > -1e3 else \
            np.full(R, cfg["bs"], np.float32)
    if name == "stop_at_count":
        s["pw"][::2] = rng.integers(1, 41, size=len(s["pw"][::2]))
    if name in ("ended_rows", "stop_at_count"):
        s["tokens"][1, s["cur_len"] - 1] = EOS
        s["tokens"][5, s["cur_len"] - 1] = PAD
        s["tokens"][6, s["cur_len"] - 1] = EOS
    if name == "invalid_values":
        s["logits"][0, 17] = np.nan
        s["logits"][4, 1000] = np.inf
        s["logits"][8] = -np.inf
        s["logits"][9, :] = -np.inf; s["logits"][9, 3] = 0.0
    if name == "always_allow_eos":
        s["masks"][:, 0] &= ~np.uint32(1 << EOS)
    run_and_check(index, s, f"proc {name}")


def test_forced_bos_first_step(index):
    """ForcedBOS at cur_len 1: one allowed token per row, fill-ins with -inf, the parent range carried over"""
    idx, ora, _ = index
    rng = np.random.default_rng(5)
    B, V, Q, T = 4, 4099, 2, 8
    s = base_case(index, rng, B, V, Q, cur_len=1, T=T, forced_bos=0)
    R = Q * B
    s["tokens"][:] = PAD; s["tokens"][:, 0] = START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    s["occ"] = words_of(rng.random(V) < 0.5)
    s["shared"] = True
    s["logits"] = (rng.standard_normal((Q, V)) * 2).astype(np.float32)
    run_and_check(index, s, "forced BOS")


@pytest.mark.parametrize("cur_len", [1, 3])
@pytest.mark.parametrize("G,B", [(3, 15), (3, 3)])
def test_diverse_groups_vs_float64(index, cur_len, G, B):
    """G = 3 with penalty 0.5: group by group, penalised candidates recomputed; the first step lists rows 0 and 1 only
    (lists = 2, or 1 when gs = 1)"""
    idx, ora, _ = index
    rng = np.random.default_rng(cur_len * 10 + B)
    V, Q, T = 4099, 2, 8
    s = base_case(index, rng, B, V, Q, cur_len=cur_len, T=T, G=G, penalty=0.5)
    R = Q * B
    gs = B // G
    if cur_len == 1:
        s["tokens"][:] = PAD; s["tokens"][:, 0] = START
        s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
        s["bs"] = np.where(np.arange(R) % gs == 0, 0.0, -1e9).astype(np.float32)
        s["occ"] = words_of(rng.random(V) < 0.3)
        s["shared"] = True
        X = (rng.standard_normal((Q, V)) * 2).astype(np.float32)
        X[:, :40] = 6.0 + np.round(X[:, :40])                 # a few strong, tied tokens every group wants
        s["logits"] = X
    else:
        M = rng.random((R, V)) < 0.02
        M[:, :40] = True
        s["masks"] = words_of(M)
        X = (rng.standard_normal((R, V)) * 2).astype(np.float32)
        X[:, :40] = 6.0 + np.round(X[:, :40])
        s["logits"] = X
    run_and_check(index, s, f"groups G={G} B={B} cur_len={cur_len}")


def test_rejects_configurations_generate_never_runs(index):
    from seal_b200._lib import SealB200Error
    rng = np.random.default_rng(9)
    s = base_case(index, rng, 4, 4099, 2)
    s["masks"] = random_masks(rng, 8, 4099, [5])
    s["logits"] = logits_rows(rng, 8, 4099, ["smooth"])
    run_step(index[0]._dev(), s)                              # valid
    bad = [dict(cur_len=10), dict(cur_len=0), dict(shared=True), dict(ignored=True),
           dict(head_stats=np.zeros((8, 33, 2), np.float32), G=2), dict(G=3)]
    for b in bad:
        t = dict(s); t.update(b)
        with pytest.raises(SealB200Error):
            run_step(index[0]._dev(), t)
    t = dict(s); t["p"] = make_params(33, 10)
    with pytest.raises(SealB200Error):
        run_step(index[0]._dev(), t)


# ---- the lm_head statistics epilogue -----------------------------------------------------------------------------------
def run_head(A, W, b, mask, eos=EOS, pad=PAD):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    mp = -(-M // GN) * GN
    tiles = -(-N // GN)
    Cm = np.empty((mp, N), np.float32); st = np.empty((mp, tiles, 2), np.float32); fused = np.zeros(1, np.int32)
    check(lib.sealdec_debug_head(M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                 np.ascontiguousarray(mask).ctypes.data, eos, pad, Cm.ctypes.data, st.ctypes.data,
                                 fused.ctypes.data))
    return Cm, st, bool(fused[0])


def run_dense(A, W, b):
    from seal_b200._lib import lib, check
    M, K = A.shape; N = W.shape[0]
    out = np.empty((M, N), np.float32)
    us = C.c_double(0)
    check(lib.sealdec_debug_gemm_ex(3, M, N, K, A.ctypes.data, W.ctypes.data, b.ctypes.data if b is not None else None,
                                    out.ctypes.data, 0, 0, C.byref(us), -1, 1))
    return out


def head_inputs(rng, M, N, K, kind):
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float32)
    W = (rng.standard_normal((N, K)) * (0.5 / math.sqrt(K))).astype(np.float32)
    if kind == "spread":          # a spread of hundreds: whole tiles far below the row's maximum
        b = (-400.0 * ((np.arange(N) // GN) % 3 == 1) + rng.standard_normal(N)).astype(np.float32)
    elif kind == "negative":      # every logit < 0: a padding column counted as 0 would be the tile's maximum
        b = np.full(N, -50.0, np.float32)
        A[::3] = 0.0              # constant rows
    else:
        b = None
    mask = words_of(rng.integers(0, 100, size=(M, N), dtype=np.uint8) == 0)
    return A, W, b, mask


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# 2 100 rows at K = 1 024 take the banded tile order; (1, 128, 1 024) and (129, 129, 1 024) the split-K path
HEAD_SHAPES = [(1, 50265, 64), (129, 50265, 64), (300, 129, 64), (300, 128, 64), (2100, 50265, 1024),
               (1, 128, 1024), (129, 129, 1024)]
HEAD_CASES = [(M, N, K, kind) for (M, N, K) in HEAD_SHAPES for kind in ("spread", "negative")] + [(129, 50265, 64, "nobias")]


@pytest.mark.parametrize("M,N,K,kind", HEAD_CASES)
def test_head_epilogue_vs_float64(M, N, K, kind):
    """read set, stored values, tile max and tile sum exp(x - max) of the statistics epilogue against the dense GEMM
    and float64.  Stored values equal the dense GEMM bit for bit (the same expression, acc * w_unscale + bias, in the
    same kernel body).  The tile sum: per lane a pair add and 16 sequential adds, two shuffle adds -- 19 roundings in
    one chain -- and expf (2 ulp) of an argument rounded to half an ulp of |d|:
        |se - S64| <= u sum e_i |d_i| + 4u S + gamma(19) S + 128 * 2^-148."""
    rng = np.random.default_rng(M + N + K)
    A, W, b, mask = head_inputs(rng, M, N, K, kind)
    Cm, st, fused = run_head(A, W, b, mask)
    dense = run_dense(A, W, b)
    tiles = -(-N // GN)
    kblocks = K // 64
    split = tiles * -(-M // GN) * 2 <= sm_count() and kblocks >= 4
    assert fused == (not split), (fused, split)
    assert np.isnan(Cm[M:]).all() and (st[M:].view(np.uint32) == 0xFFFFFFFF).all(), "rows >= M written"
    if not fused:                 # split-K: the dense store, no statistics
        assert np.array_equal(Cm[:M].view(np.uint32), dense.view(np.uint32))
        assert (st.view(np.uint32) == 0xFFFFFFFF).all()
        REPORT.append(f"head {M}x{N}x{K} {kind}: split-K, dense store")
        return
    bits = np.unpackbits(mask.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
    read = bits.copy(); read[:, :GN] = True; read[:, EOS] = True; read[:, PAD] = True
    stored = ~np.isnan(Cm[:M])
    assert np.array_equal(stored, read), ("stored set is not the read set", np.argwhere(stored != read)[:5])
    assert np.array_equal(Cm[:M][read].view(np.uint32), dense[read].view(np.uint32)), "stored values differ"
    worst = 0.0
    for t in range(tiles):
        x = dense[:, t * GN:(t + 1) * GN].astype(np.float64)
        mx = x.max(1)
        assert np.array_equal(st[:M, t, 0], mx.astype(np.float32)), ("tile max", t)
        d = x - mx[:, None]
        e = np.exp(d)
        S = e.sum(1)
        bound = U * (e * np.abs(d)).sum(1) + 4 * U * S + gamma(19) * S + GN * 2.0 ** -148
        err = np.abs(st[:M, t, 1].astype(np.float64) - S)
        assert (err <= bound).all(), ("tile sum", t, np.argmax(err / bound))
        worst = max(worst, float((err / bound).max()))
    REPORT.append(f"head {M}x{N}x{K} {kind}: worst |tile sum err| / bound {worst:.3f}")


@pytest.mark.parametrize("V", [50265, 4099])
def test_select_step_on_head_statistics(index, V):
    """head_tiles > 0: the statistics and the NaN-poisoned logits of sealdec_debug_head feed the step; the float64
    reference is built on the dense fp32 logits of the same GEMM"""
    rng = np.random.default_rng(V)
    B, Q, Kd = 15, 2, 64
    s = base_case(index, rng, B, V, Q)
    R = Q * B
    M = rng.random((R, V)) < 0.02
    M[0] = False; M[0, :3] = True                             # fewer than 2B finite candidates: fill-ins from tile 0
    s["masks"] = words_of(M)
    A = (rng.standard_normal((R, Kd)) * 0.5).astype(np.float32)
    W = (rng.standard_normal((V, Kd)) * 0.3).astype(np.float32)
    b = (rng.standard_normal(V) - 50.0 * (np.arange(V) % 7 == 0)).astype(np.float32)
    A[5] = 0.0                                                # a row of bias only
    Cm, st, fused = run_head(A, W, b, s["masks"])
    assert fused
    s["logits"] = Cm[:R]
    s["head_stats"] = st[:R]
    o = run_step(index[0]._dev(), s)
    s_ref = dict(s); s_ref["logits"] = run_dense(A, W, b)
    check_step(s_ref, o, index[1], f"head stats V={V}")
