"""GPU: the top-k logits warp (fm_index_generate's topk, include/sealdec.h sealdec_params_t.top_k).

* topk_threshold_kernel through sealdec_debug_topk_threshold against numpy on crafted rows.  tau and the row max must
  match bit for bit (the kernel returns -0.0 as +0.0, equal as floats).  The log-sum-exp over x >= tau is summed per
  thread over ceil(V / 512) strided keys, then by the warp's 5-level shuffle tree, then over the 16 warps in order, so
  with u = 2^-24, d_i = x_i - max, e_i = exp(d_i), S = sum of the kept e_i and n_add = ceil(V / 512) + 5 + 16:
      |logsum - log S| <= rel / (1 - rel) + ulp(log S),
      rel * S = u * sum e_i |d_i|  (x - max rounded)  +  4u * S  (expf, 2 ulp)  +  gamma(n_add) * S  +  V * 2^-148,
  logf being good to 1 ulp.  There is no rescaling: the max is known before the sum.
* One decode step through sealdec_debug_select_step with top_k > 0, checked by test_select_step_gpu.check_step against
  the float64 step reference on the warped logits (x < tau replaced by -inf: what TopKLogitsWarper hands log_softmax),
  with the bound above in place of the streaming one.  Forcing steps must be unaffected; head statistics are refused.
* Whole generates against tests/topk_oracle.py (tiny model and bart-large) and the reference-code fixture, compared as
  test_decode_gpu.compare_generate does.  A query whose oracle trace has a row where the k-th and the (k+1)-th largest
  logit lie within 1e-4 of each other is boundary-ambiguous (the GPU's logits may keep the other one) and left out.
  With k < 2B the first step's list often ends in candidates that tie exactly (beams 1.. are copies of beam 0 at
  -1e9), and torch.topk leaves their order unspecified: the oracle runs with flat_ties=True (equal scores in flat-index
  order, the kernels' rule), and against the reference's own fixture such tie-sensitive queries are left out too.
* Exact equalities: top_k >= V and diverse groups are the top_k = 0 decode; query slices, CUDA-graph replay, the
  launch count and the dense lm_head.
"""
import json
import os

import numpy as np
import pytest

import test_select_step_gpu as tss
from test_decode_gpu import compare_generate, make_inputs, tiny_setup
from test_select_step_gpu import index  # noqa: F401  (fixture)
from test_query_slices_gpu import assert_identical, setup  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24
GAP = 1e-4


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


@pytest.fixture(scope="module")
def tiny():
    return tiny_setup()


# ---- the threshold kernel --------------------------------------------------------------------------------------------
def run_threshold(X, V, ld, k):
    from seal_b200._lib import check, lib
    R = X.shape[0]
    buf = np.full((R, ld), np.nan, np.float32)                 # columns V .. ld-1 must not be read
    buf[:, :V] = X
    thr = np.empty(R, np.float32); mx = np.empty(R, np.float32); ls = np.empty(R, np.float32)
    check(lib.sealdec_debug_topk_threshold(R, V, ld, buf.ctypes.data, k, thr.ctypes.data, mx.ctypes.data, ls.ctypes.data))
    return thr, mx, ls


def crafted_rows(rng, V, k):
    rows = {}
    rows["smooth"] = rng.standard_normal(V) * 3.0
    rows["ties"] = np.round(rng.standard_normal(V) * 4.0) / 2.0            # long runs of exact ties at every rank
    rows["constant"] = np.full(V, 0.75)
    x = rng.standard_normal(V) * 2.0
    x[rng.choice(V, 3, replace=False)] = -np.inf                           # the three -inf bias entries
    rows["neg_inf"] = x
    x = rng.standard_normal(V) * 2.0
    x[rng.random(V) < 0.3] = -np.inf
    rows["many_neg_inf"] = x
    n_pos = min(max(k - 5, 0), V - 10)                                     # tau lands on the zeros for k <= V
    x = -1.0 - np.abs(rng.standard_normal(V))
    perm = rng.permutation(V)
    x[perm[:n_pos]] = 1.0 + np.abs(rng.standard_normal(n_pos))
    z = perm[n_pos:n_pos + 10]
    x[z] = 0.0
    x[z[::2]] = -0.0
    rows["signed_zeros"] = x
    rows["large"] = rng.choice([-1.0, 1.0], V) * rng.uniform(1e37, 3.4e38, V)
    rows["all_neg_inf_but_one"] = np.full(V, -np.inf); rows["all_neg_inf_but_one"][V // 3] = -7.5
    names = list(rows)
    return names, np.stack([rows[n] for n in names]).astype(np.float32)


def numpy_threshold(X, k):
    V = X.shape[1]
    k_eff = min(max(k, 1), V)
    tau = -np.sort(-X.astype(np.float64), axis=1)[:, k_eff - 1]
    mx = X.astype(np.float64).max(1)
    n_add = -(-V // 512) + 5 + 16
    gamma = n_add * U / (1 - n_add * U)
    with np.errstate(all="ignore"):
        d = X.astype(np.float64) - mx[:, None]
        e = np.where(X.astype(np.float64) >= tau[:, None], np.exp(d), 0.0)
        S = e.sum(1)
        L = np.log(S)
        fin = np.where(np.isfinite(d), np.abs(d), 0.0)
        rel = (U * (e * fin).sum(1) + 4 * U * S + gamma * S + V * 2.0 ** -148) / S
        E = rel / (1 - rel) + np.spacing(np.abs(L.astype(np.float32))).astype(np.float64)
    return tau, mx, L, E


def same_float(a, b):
    """bit-identical, except that a kernel +0.0 stands for either zero"""
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | ((a == 0) & (b == 0) & ~np.signbit(a))


SHAPES = [(2000, 2000), (50265, 50265), (4099, 4099), (4099, 4104), (50265, 50268)]


@pytest.mark.parametrize("V,ld", SHAPES)
def test_threshold_kernel_vs_numpy(V, ld):
    rng = np.random.default_rng(V + ld)
    worst = 0.0
    for k in (1, 2, V - 4, V - 3, V - 2, V, V + 7):
        names, X = crafted_rows(rng, V, k)
        thr, mx, ls = run_threshold(X, V, ld, k)
        tau, mref, L, E = numpy_threshold(X, k)
        for i, n in enumerate(names):
            assert same_float(thr[i], tau[i]), (V, ld, k, n, thr[i], tau[i])
            assert same_float(mx[i], mref[i]), (V, ld, k, n, mx[i], mref[i])
            err = abs(float(ls[i]) - L[i])
            assert err <= E[i], (V, ld, k, n, float(ls[i]), L[i], E[i])
            worst = max(worst, err / E[i])
        if k >= V - 3:                                                     # -inf entries count: nothing finite removed
            row = X[names.index("neg_inf")]
            assert thr[names.index("neg_inf")] == row[np.isfinite(row)].min() if k == V - 3 else \
                np.isneginf(thr[names.index("neg_inf")])
        if k <= 10:
            assert thr[names.index("signed_zeros")] == 0
    print(f"threshold V={V} ld={ld}: worst |logsum err| / bound = {worst:.3f}")


def test_threshold_rejects_bad_arguments():
    from seal_b200._lib import SealB200Error, check, lib
    X = np.zeros((2, 60000), np.float32)
    out = [np.empty(2, np.float32) for _ in range(3)]
    for R, V, ld, k in ((2, 53249, 60000, 5), (2, 100, 99, 5), (2, 100, 100, 0), (0, 100, 100, 5)):
        with pytest.raises(SealB200Error):
            check(lib.sealdec_debug_topk_threshold(R, V, ld, X.ctypes.data, k, *[o.ctypes.data for o in out]))


# ---- one decode step -------------------------------------------------------------------------------------------------
def warped(s, k):
    """the case with TopKLogitsWarper(k) applied to its logits rows"""
    X = s["logits"]
    k_eff = min(k, X.shape[1])
    tau = -np.sort(-X, axis=1)[:, k_eff - 1]
    t = dict(s)
    t["logits"] = np.where(X < tau[:, None], np.float32(-np.inf), X).astype(np.float32)
    return t


def with_top_k(s, k):
    t = dict(s)
    p = type(s["p"]).from_buffer_copy(s["p"])
    p.top_k = k
    t["p"] = p
    return t


@pytest.fixture
def threshold_bound(monkeypatch):
    """check_step's log-sum-exp bound for the threshold kernel's summation order (module docstring)"""
    monkeypatch.setattr(tss, "step_sizes", lambda s: (512, 0, -(-s["V"] // 512) + 5 + 16))


def run_topk_step(index, s, k, label):
    o = tss.run_step(index[0]._dev(), with_top_k(s, k))
    return tss.check_step(warped(s, k), o, index[1], label)


@pytest.mark.parametrize("k", [1, 3, 29, 500])
@pytest.mark.parametrize("V", [50265, 4099])
def test_later_step_topk(index, threshold_bound, V, k):
    """later step, one CTA per row: allowed tokens per row 0 .. V, logits smooth, on a coarse grid (ties at tau), shifted.
    Small k: most allowed tokens fall below tau, so lists run short and fill-ins score -inf."""
    rng = np.random.default_rng(V * 7 + k)
    B = 15
    counts = [0, 1, 29, 30, 31, 2048, 4097, V]
    s = tss.base_case(index, rng, B, V, 2)
    R = 2 * B
    s["masks"] = tss.random_masks(rng, R, V, counts)
    s["logits"] = tss.logits_rows(rng, R, V, ["smooth", "minus50", "coarse", "plus50"])
    run_topk_step(index, s, k, f"topk later V={V} k={k}")


@pytest.mark.parametrize("k", [1, 7, 1000])
@pytest.mark.parametrize("B", [4, 15])
def test_first_step_topk(index, threshold_bound, B, k):
    """first step: logits shared by a query's beams (one threshold row per query), beams 1.. at -1e9"""
    idx, ora, _ = index
    rng = np.random.default_rng(B * 13 + k)
    V, Q, T = 50265, 3, 10
    s = tss.base_case(index, rng, B, V, Q, cur_len=1, T=T)
    R = Q * B
    s["tokens"][:] = tss.PAD; s["tokens"][:, 0] = tss.START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["anc"] = np.tile(np.arange(R, dtype=np.int32)[:, None], (1, T))
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    s["occ"] = tss.words_of(rng.random(V) < 0.4)
    s["shared"] = True
    X = (rng.standard_normal((Q, V)) * 2.0).astype(np.float32)
    X[1] -= 50.0
    s["logits"] = X
    run_topk_step(index, s, k, f"topk first B={B} k={k}")


@pytest.mark.parametrize("name", ["stop_at_count", "ended_rows", "always_allow_eos", "min_length", "disable_fm_index"])
def test_rules_and_processors_topk(index, threshold_bound, name):
    """rule-1 (count <= stop_at_count: EOS only) and rule-2 (ended: pad only) rows, whose one allowed token usually lies
    below tau and then enters as a -inf pick; processors after the warp"""
    cfg = tss.PROC_CASES[name]
    rng = np.random.default_rng(len(name) + 100)
    B, V, Q = 4, 4099, 3
    s = tss.base_case(index, rng, B, V, Q, cur_len=3, **cfg["pkw"])
    R = Q * B
    s["masks"] = tss.random_masks(rng, R, V, [3, 20, 200, 1, 0, 9])
    s["logits"] = tss.logits_rows(rng, R, V, ["smooth", "minus50"])
    if name == "stop_at_count":
        s["pw"][::2] = rng.integers(1, 41, size=len(s["pw"][::2]))
    if name in ("ended_rows", "stop_at_count"):
        for r, t in ((1, tss.EOS), (5, tss.PAD), (6, tss.EOS)):
            s["tokens"][r, 2] = t
    if name == "always_allow_eos":
        s["masks"][:, 0] &= ~np.uint32(1 << tss.EOS)
    for k in (2, 50):
        run_topk_step(index, s, k, f"topk proc {name} k={k}")


def test_forcing_steps_unaffected(index):
    """forced BOS (cur_len 1) and the forced-EOS step whose logits are ignored: top_k changes no output"""
    idx, ora, _ = index
    rng = np.random.default_rng(17)
    B, V, Q, T = 4, 4099, 2, 8
    s = tss.base_case(index, rng, B, V, Q, cur_len=1, T=T, forced_bos=0)
    R = Q * B
    s["tokens"][:] = tss.PAD; s["tokens"][:, 0] = tss.START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    s["occ"] = tss.words_of(rng.random(V) < 0.5)
    s["shared"] = True
    s["logits"] = (rng.standard_normal((Q, V)) * 2).astype(np.float32)
    d = tss.base_case(index, rng, B, V, 3, cur_len=9, forced_eos=tss.EOS)
    d["masks"] = tss.random_masks(rng, 12, V, [3, 20])
    d["ignored"] = True
    for case in (s, d):
        ref = tss.run_step(idx._dev(), case)
        for k in (1, 5):
            got = tss.run_step(idx._dev(), with_top_k(case, k))
            for key in ref:
                assert ref[key].tobytes() == got[key].tobytes(), key


def test_rejects_topk_configurations(index):
    from seal_b200._lib import SealB200Error
    rng = np.random.default_rng(19)
    s = tss.base_case(index, rng, 4, 4099, 2)
    s["masks"] = tss.random_masks(rng, 8, 4099, [5])
    s["logits"] = tss.logits_rows(rng, 8, 4099, ["smooth"])
    tss.run_step(index[0]._dev(), with_top_k(s, 5))                     # valid
    bad = [(dict(head_stats=np.zeros((8, 33, 2), np.float32)), 5), (dict(G=2), 5), ({}, -1)]
    for b, k in bad:
        t = with_top_k(s, k); t.update(b)
        with pytest.raises(SealB200Error):
            tss.run_step(index[0]._dev(), t)


# ---- whole generates -------------------------------------------------------------------------------------------------
def _golden():
    with open(os.path.join(HERE, "golden", "decode_topk_golden.json")) as f:
        return json.load(f)


def compare_unambiguous(got, exp, info, ora, kw, ties=False):
    keep = [q for q in range(len(got)) if info["min_gap"][q] >= GAP and not (ties and info["tie_sensitive"][q])]
    compare_generate([got[q] for q in keep], [exp[q] for q in keep], ora, force=kw.get("force_decoding_from"),
                     skip=1 if kw.get("forced_bos_token_id") is not None else 0)
    return len(keep)


def test_generate_vs_oracle_tiny(tiny):
    """every configuration of the fixture on 8 other queries; at least half of all queries compared (83 of 136 pass the
    boundary filter on the oracle's CPU logits)"""
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny
    total = compared = 0
    for ci, kw in enumerate(_golden()["cases"]):
        kw = kw["kw"]
        rng = np.random.default_rng(500 + ci)
        ids, am = make_inputs(rng, Q=8, S=12, vocab=2000)
        info = {}
        exp = fm_index_generate_topk_oracle(model, ora, ids, am, info=info, flat_ties=True, **kw)
        got = fm_index_generate(model, idx, ids, am, **kw)
        n = compare_unambiguous(got, exp, info, ora, kw)
        print(f"tiny {kw}: {n}/8 queries compared, excluded (k-gap < {GAP}): "
              f"{[q for q in range(8) if info['min_gap'][q] < GAP]}")
        total += 8; compared += n
    assert compared >= total // 2, (compared, total)


def test_generate_vs_reference_code_fixture():
    """decode_topk_golden.json: what the reference's own seal/beam_search.py returned for these inputs; boundary-ambiguous
    and tie-sensitive queries left out, at least a third of all compared (28 of 68 pass both filters on the CPU)"""
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    g = _golden()
    seqs = [d.tolist() for d in make_corpus(**g["corpus"])]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    model = make_bart(**g["model"])
    total = compared = 0
    for c in g["cases"]:
        kw = c["kw"]
        ids, am = torch.tensor(c["input_ids"]), torch.tensor(c["attention_mask"])
        info = {}
        fm_index_generate_topk_oracle(model, ora, ids, am, info=info, **kw)     # for the boundary gaps only
        got = fm_index_generate(model, idx, ids, am, **kw)
        exp = [[(s, t, None) for s, t in q] for q in c["hyps"]]
        n = compare_unambiguous(got, exp, info, ora, kw, ties=True)
        print(f"reference-code fixture {kw}: {n}/{len(got)} queries compared")
        total += len(got); compared += n
    assert compared >= total // 3, (compared, total)


def test_generate_bart_large_batch20_beam15():
    """SEALSearcher's body pass with --topk: bart-large (seeded random weights), batch 20, beam 15, n-grams of 10, on
    the 200 k-token phrase corpus; oracle on the same GPU"""
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
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
    compared = 0
    for k in (1, 29):
        kw = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0, topk=k)
        got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
        info = {}
        exp = fm_index_generate_topk_oracle(model.to("cuda"), ora, ids.cuda(), am.cuda(), info=info, flat_ties=True, **kw)
        n = compare_unambiguous(got, exp, info, ora, kw)
        print(f"bart-large batch20/beam15 topk={k}: {n}/20 queries compared")
        compared += n
    assert compared >= 10, compared


# ---- exact equalities ------------------------------------------------------------------------------------------------
RECORD_KEYS = ("scores", "lens", "tokens", "valid", "lo", "hi")


def test_top_k_at_least_vocab_is_no_warp(tiny):
    from seal_b200.beam_search import generate_records
    docs, ora, idx, model = tiny
    ids, am = make_inputs(np.random.default_rng(61), Q=6, S=12, vocab=2000)
    kw = dict(min_length=0, max_length=8, length_penalty=0.0, num_beams=5)
    ref = generate_records(model, idx, ids, am, **kw)
    for k in (2000, 2007):
        assert_identical(ref, generate_records(model, idx, ids, am, top_k=k, **kw))
    assert not np.array_equal(ref["tokens"], generate_records(model, idx, ids, am, top_k=3, **kw)["tokens"])


def test_diverse_groups_ignore_topk(tiny):
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny
    ids, am = make_inputs(np.random.default_rng(62), Q=6, S=12, vocab=2000)
    kw = dict(min_length=0, max_length=7, length_penalty=0.0, num_beams=6, diverse_bs_groups=3, diverse_bs_penalty=0.5,
              keep_history=True)
    assert fm_index_generate(model, idx, ids, am, topk=5, **kw) == fm_index_generate(model, idx, ids, am, topk=0, **kw)


def test_query_slices_bit_identical_with_topk(setup):
    """300 queries x beam 15 (the sliced path) with top_k = 10: slices on and off give the same records; the lm_head
    stays dense (no statistics-epilogue steps) while the top_k = 0 decode of the same batch uses the epilogue"""
    from test_query_slices_gpu import BASE, PATH_QUERY_SLICES, make_inputs as slice_inputs, run
    idx, eng = setup
    ids, am = slice_inputs(np.random.default_rng(63), 300, 16, 2000)
    whole, paths0 = run(eng, idx, ids, am, 0, top_k=10, **BASE)
    assert eng.stat("fused_head_steps") == 0
    sliced, paths1 = run(eng, idx, ids, am, 1, top_k=10, **BASE)
    assert eng.stat("fused_head_steps") == 0
    assert not paths0 & PATH_QUERY_SLICES and paths1 & PATH_QUERY_SLICES
    assert_identical(whole, sliced)
    run(eng, idx, ids, am, 1, **BASE)
    fused0 = eng.stat("fused_head_steps")
    print(f"fused_head_steps: top_k=0 {fused0}, top_k=10 0")
    assert fused0 > 0


def test_graph_replay_and_launch_count(tiny):
    """the same buffers with top_k 0, then 10, then 0 again: every call (eager, captured, replayed) returns the eager
    run's records; the top-k decode launches one threshold kernel per step whose logits are read"""
    from seal_b200.beam_search import SealBartEngine, generate_records
    docs, ora, idx, model = tiny
    eng = SealBartEngine.from_hf(model, device=0)
    ids, am = make_inputs(np.random.default_rng(64), Q=20, S=12, vocab=2000)
    T = 8
    kw = dict(min_length=0, max_length=T, length_penalty=0.0, num_beams=15)
    eager, launches = {}, {}
    eng.set_option("cuda_graph", 0)
    for k in (0, 10):
        eager[k] = generate_records(eng, idx, ids, am, top_k=k, **kw)
        launches[k] = eng.last_launch_count()
        assert eng.stat("last_used_graph") == 0
    # forced_eos_token_id = 2 in the config: the last step's logits are ignored; no forced BOS
    assert launches[10] - launches[0] == T - 2, launches
    eng.set_option("cuda_graph", 1)
    used = []
    for k in (0, 0, 0, 10, 10, 10, 0):
        assert_identical(eager[k], generate_records(eng, idx, ids, am, top_k=k, **kw))
        used.append(eng.stat("last_used_graph"))
    assert used == [0, 1, 1, 0, 1, 1, 1], used
    eng.set_option("cuda_graph", -1)
