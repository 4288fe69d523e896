"""GPU: the top-k logits warp on vocabularies above 53 248 entries (mT5's 250 112), where the threshold of a logits row
runs on one cluster of ceil(V / 53 248) CTAs (topk_threshold_cluster_kernel, decode_kernels.cuh).

* The cluster kernel through sealdec_debug_topk_threshold_cluster against numpy on test_topk_gpu's crafted rows, from
  one CTA (V <= 53 248) to the 8-CTA limit (V = 425 984), with the float4 and the scalar staging path (ld = V odd, or
  ld a multiple of 4).  tau and the max must match bit for bit.  The log-sum-exp is summed in a fixed order: per CTA
  as the one-CTA kernel sums a row (ceil(chunk / 512) strided keys per thread, the warp's 5-level tree, the 16 warps in
  order), then the n CTA sums in rank order, so test_topk_gpu's bound holds with
      n_add = ceil(chunk / 512) + 5 + 16 + (n - 1),   chunk = ceil(V / n) rounded up to a multiple of 4.
  At n = 1 the order is the one-CTA kernel's, and the outputs must equal it bit for bit.
* One decode step at V = 250 112 through test_select_step_gpu's run_step / check_step with top_k set, against the
  float64 step reference on warped logits, with the bound above in place of the streaming one.
* Whole generates at V = 250 112 against tests/topk_oracle.py: a seeded tiny T5 (d_model 128, gated-gelu, untied
  lm_head) with the mT5 vocabulary and SEAL's T5 token conventions, on an index whose symbols reach past 2^16 (an
  18-level wavelet tree); both scorers and transformers_output.  Boundary-ambiguous queries (the k-th and (k+1)-th
  largest logit of some row within 1e-4) and tie-sensitive ones are left out, as in test_topk_gpu.py.  One BART model
  with V = 60 000 at k = 10.  The stat "topk_cluster_steps" shows which threshold kernel ran.
* CUDA-graph replay and the two-query-slice path at V = 250 112 with top_k = 10 give the eager call's records.
"""
import numpy as np
import pytest

import test_select_step_gpu as tss
from t5_models import PAD, make_t5, t5_sources, title_corpus
from test_query_slices_gpu import assert_identical
from test_topk_gpu import GAP, U, crafted_rows, numpy_threshold, same_float, warped, with_top_k

pytestmark = pytest.mark.gpu

V_MT5 = 250112
MAX_CTA_VOCAB = 53248
MAX_CLUSTER_VOCAB = 8 * MAX_CTA_VOCAB
TOL = 1e-4                      # |dscore| of a recorded hypothesis, the project's decode bound


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    assert not torch.backends.cuda.matmul.allow_tf32


def cluster_shape(V):
    n = -(-V // MAX_CTA_VOCAB)
    return n, (-(-V // n) + 3) // 4 * 4


def cluster_n_add(V):
    n, chunk = cluster_shape(V)
    return -(-chunk // 512) + 5 + 16 + (n - 1)


# ---- the threshold kernel --------------------------------------------------------------------------------------------
def run_threshold(fn, X, V, ld, k):
    from seal_b200._lib import check
    R = X.shape[0]
    buf = np.full((R, ld), np.nan, np.float32)                 # columns V .. ld-1 must not be read
    buf[:, :V] = X
    thr = np.empty(R, np.float32); mx = np.empty(R, np.float32); ls = np.empty(R, np.float32)
    check(fn(R, V, ld, buf.ctypes.data, k, thr.ctypes.data, mx.ctypes.data, ls.ctypes.data))
    return thr, mx, ls


def cluster_bound(X, k):
    """numpy_threshold's (tau, max, log S) with its log-sum-exp bound at the cluster kernel's n_add"""
    tau, mx, L, _ = numpy_threshold(X, k)
    V = X.shape[1]
    n_add = cluster_n_add(V)
    gamma = n_add * U / (1 - n_add * U)
    with np.errstate(all="ignore"):
        X64 = X.astype(np.float64)
        d = X64 - mx[:, None]
        e = np.where(X64 >= tau[:, None], np.exp(d), 0.0)
        S = e.sum(1)
        fin = np.where(np.isfinite(d), np.abs(d), 0.0)
        rel = (U * (e * fin).sum(1) + 4 * U * S + gamma * S + V * 2.0 ** -148) / S
        E = rel / (1 - rel) + np.spacing(np.abs(L.astype(np.float32))).astype(np.float64)
    return tau, mx, L, E


CLUSTER_V = [2000, 50265, 53249, 106496, 106497, V_MT5, MAX_CLUSTER_VOCAB]


@pytest.mark.parametrize("ld_kind", ["ld_eq_V", "ld_aligned"])
@pytest.mark.parametrize("V", CLUSTER_V)
def test_cluster_threshold_vs_numpy(V, ld_kind):
    from seal_b200._lib import lib
    ld = V if ld_kind == "ld_eq_V" else (V + 3) // 4 * 4 + 4
    rng = np.random.default_rng(V * 3 + ld)
    worst = 0.0
    for k in (1, 2, V - 4, V - 3, V - 2, V - 1, V, V + 7):
        names, X = crafted_rows(rng, V, k)
        thr, mx, ls = run_threshold(lib.sealdec_debug_topk_threshold_cluster, X, V, ld, k)
        tau, mref, L, E = cluster_bound(X, k)
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
        if V <= MAX_CTA_VOCAB:                                             # one CTA: the one-CTA kernel's order
            one = run_threshold(lib.sealdec_debug_topk_threshold, X, V, ld, k)
            for a, b in zip(one, (thr, mx, ls)):
                assert a.tobytes() == b.tobytes(), (V, ld, k)
    print(f"cluster threshold V={V} ld={ld} (n={cluster_shape(V)[0]}): worst |logsum err| / bound = {worst:.3f}")


def test_cluster_threshold_rejects_bad_arguments():
    from seal_b200._lib import SealB200Error, check, lib
    X = np.zeros((2, MAX_CLUSTER_VOCAB + 8), np.float32)
    out = [np.empty(2, np.float32) for _ in range(3)]
    for R, V, ld, k in ((2, MAX_CLUSTER_VOCAB + 1, MAX_CLUSTER_VOCAB + 8, 5), (2, 100, 99, 5), (2, 100, 100, 0),
                        (0, 100, 100, 5), (2, 0, 100, 5)):
        with pytest.raises(SealB200Error):
            check(lib.sealdec_debug_topk_threshold_cluster(R, V, ld, X.ctypes.data, k, *[o.ctypes.data for o in out]))


# ---- one decode step at V = 250 112 ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def index():
    """an index over the mT5 id space (symbols past 2^16) and prefixes of its documents, as test_select_step_gpu's"""
    from oracle.fm_oracle import OracleIndex
    from seal_b200._lib import lib
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    seqs = [d.tolist() for d in make_corpus(n_docs=2000, doc_len=40, n_phrases=5000, seed=7, vocab=V_MT5)]
    idx = FMIndex(); idx.initialize(seqs, in_memory=True); idx.to_device(0)
    assert int(lib.sealfm_max_level(idx._handle())) >= 17
    return idx, OracleIndex(seqs), seqs


@pytest.fixture
def cluster_bound_step(monkeypatch):
    """check_step's log-sum-exp bound for the cluster kernel's summation order (module docstring)"""
    monkeypatch.setattr(tss, "step_sizes", lambda s: (512, 0, cluster_n_add(s["V"])))


def run_topk_step(index, s, k, label):
    o = tss.run_step(index[0]._dev(), with_top_k(s, k))
    return tss.check_step(warped(s, k), o, index[1], label)


@pytest.mark.parametrize("k", [1, 29, 1000])
def test_later_step_topk_mt5(index, cluster_bound_step, k):
    """later step, one CTA per row in the select kernel: allowed tokens per row 0 .. V, smooth / shifted / coarse rows"""
    rng = np.random.default_rng(V_MT5 + k)
    B = 15
    s = tss.base_case(index, rng, B, V_MT5, 2)
    R = 2 * B
    s["masks"] = tss.random_masks(rng, R, V_MT5, [0, 1, 29, 30, 31, 2048, 70000, V_MT5])
    s["logits"] = tss.logits_rows(rng, R, V_MT5, ["smooth", "minus50", "coarse", "plus50"])
    run_topk_step(index, s, k, f"topk later V={V_MT5} k={k}")


@pytest.mark.parametrize("B,k", [(15, 1), (4, 7), (15, 1000)])
def test_first_step_topk_mt5(index, cluster_bound_step, B, k):
    """first step: logits shared by a query's beams (one threshold row per query), beams 1.. at -1e9"""
    idx, ora, _ = index
    rng = np.random.default_rng(B * 17 + k)
    Q, T = 3, 10
    s = tss.base_case(index, rng, B, V_MT5, Q, cur_len=1, T=T)
    R = Q * B
    s["tokens"][:] = tss.PAD; s["tokens"][:, 0] = tss.START
    s["lo"][:] = 0; s["hi"][:] = ora.size() + 1; s["pw"][:] = ora.size() + 1
    s["anc"] = np.tile(np.arange(R, dtype=np.int32)[:, None], (1, T))
    s["bs"] = np.where(np.arange(R) % B == 0, 0.0, -1e9).astype(np.float32)
    s["occ"] = tss.words_of(rng.random(V_MT5) < 0.4)
    s["shared"] = True
    X = (rng.standard_normal((Q, V_MT5)) * 2.0).astype(np.float32)
    X[1] -= 50.0
    s["logits"] = X
    run_topk_step(index, s, k, f"topk first V={V_MT5} B={B} k={k}")


@pytest.mark.parametrize("name", ["stop_at_count", "ended_rows", "always_allow_eos"])
def test_rules_topk_mt5(index, cluster_bound_step, name):
    """rule-1 (count <= stop_at_count: EOS only) and rule-2 (ended: pad only) rows, and always_allow_eos"""
    cfg = tss.PROC_CASES[name]
    rng = np.random.default_rng(len(name) + 200)
    B, Q = 4, 3
    s = tss.base_case(index, rng, B, V_MT5, Q, cur_len=3, **cfg["pkw"])
    R = Q * B
    s["masks"] = tss.random_masks(rng, R, V_MT5, [3, 20, 200, 1, 0, 9])
    s["logits"] = tss.logits_rows(rng, R, V_MT5, ["smooth", "minus50"])
    if name == "stop_at_count":
        s["pw"][::2] = rng.integers(1, 41, size=len(s["pw"][::2]))
    if name in ("ended_rows", "stop_at_count"):
        for r, t in ((1, tss.EOS), (5, tss.PAD), (6, tss.EOS)):
            s["tokens"][r, 2] = t
    if name == "always_allow_eos":
        s["masks"][:, 0] &= ~np.uint32(1 << tss.EOS)
    for k in (2, 50):
        run_topk_step(index, s, k, f"topk rules {name} V={V_MT5} k={k}")


# ---- whole generates -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mt5():
    """(oracle index, FM index, title EOS, {logit scale: (fp32 HF T5 on the CPU, engine)}) with the mT5 vocabulary.
    Scale 1 gives logits of standard deviation ~4 (tests/t5_models.py), scale 0.25 ~1.  Without the warp (top_k = 0)
    the log-softmax sums all 250 112 terms in fp32: at ~4 the fp32 oracle's own score is 2.6e-5 per step from a
    float64 rescoring, so a 10-step score reaches the 1e-4 bound on rounding alone; the top_k = 0 runs use ~1."""
    import torch
    from oracle.fm_oracle import OracleIndex
    from seal_b200._lib import lib
    from seal_b200.beam_search import SealBartEngine, SealT5Engine
    from seal_b200.index import FMIndex
    docs, teos = title_corpus(vocab=V_MT5)
    assert max(max(d) for d in docs) >= 1 << 16
    idx = FMIndex(); idx.initialize(docs, in_memory=True)
    assert int(lib.sealfm_max_level(idx._handle())) >= 17
    models = {}
    for scale in (1.0, 0.25):
        cpu = make_t5("tiny_gated", vocab=V_MT5)
        with torch.no_grad():
            cpu.decoder.final_layer_norm.weight.mul_(scale)
        eng = SealBartEngine.from_hf(cpu, device=0, gemm_mode=3)
        assert isinstance(eng, SealT5Engine)
        models[scale] = (cpu, eng)
    return OracleIndex(docs), idx, teos, models


def compare_generate(ours, oracle_out, ora, keep_q, force=None):
    """as test_t5_gpu.compare_generate, on the queries keep_q marks"""
    force = list(force or [])
    keep = lambda t: ora.get_count(force + list(t[1:])) > 0
    worst = 0.0
    for q, (a, b) in enumerate(zip(ours, oracle_out)):
        if not keep_q[q]:
            continue
        fa = sorted([(tuple(t), s) for s, t in a if keep(t)])
        fb = sorted([(tuple(t), s) for s, t, _ in b if keep(t)])
        assert [x[0] for x in fa] == [x[0] for x in fb], f"query {q}: hypothesis sets differ"
        for (ta, sa), (tb, sb) in zip(fa, fb):
            worst = max(worst, abs(sa - sb))
            assert abs(sa - sb) <= TOL, (q, ta, sa, sb)
    return worst


def unambiguous(info):
    return [g >= GAP and not t for g, t in zip(info["min_gap"], info["tie_sensitive"])]


def strip_pad(row):
    row = list(row)
    while len(row) > 1 and row[-1] == PAD:
        row.pop()
    return row


@pytest.mark.parametrize("k", [0, 1, 10, 100])
def test_generate_mt5_vs_oracle(mt5, k):
    """body n-grams (both scorers, and the stock scorer's transformers_output) and titles (forced title BOS, the title
    EOS); the cluster threshold runs on every step whose logits are read iff k > 0"""
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
    from seal_b200.beam_search import fm_index_generate
    ora, idx, teos, models = mt5
    cpu, eng = models[1.0 if k > 0 else 0.25]
    rng = np.random.default_rng(40 + k)
    Q = 8
    ids, am = (torch.from_numpy(a) for a in t5_sources(rng, Q, 14, V_MT5))
    body = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0, topk=k)
    title = dict(num_beams=5, min_length=1, max_length=15, length_penalty=0.0, force_decoding_from=[1],
                 eos_token_id=teos, topk=k)
    total = compared = 0
    for label, kw, keep_history in (("body", body, True), ("body stock scorer", body, False),
                                    ("title", title, True)):
        info = {}
        exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, info=info, flat_ties=True, keep_history=keep_history, **kw)
        got = fm_index_generate(eng, idx, ids, am, keep_history=keep_history, **kw)
        steps = eng.stat("topk_cluster_steps")
        assert (steps > 0) == (k > 0), (label, steps)
        keep_q = unambiguous(info)
        worst = compare_generate(got, exp, ora, keep_q, force=kw.get("force_decoding_from"))
        n = sum(keep_q)
        print(f"mT5 V={V_MT5} topk={k} {label}: {n}/{Q} queries compared, {Q - n} excluded "
              f"(k-gap < {GAP} or tie-sensitive), worst |dscore| {worst:.2e}, topk_cluster_steps {steps}")
        total += Q; compared += n
    info = {}
    seq_exp = fm_index_generate_topk_oracle(cpu, ora, ids, am, info=info, flat_ties=True, keep_history=False,
                                            transformers_output=True, **body)
    seq_got = fm_index_generate(eng, idx, ids, am, keep_history=False, transformers_output=True, **body).cpu()
    keep_q = unambiguous(info)
    for q in range(Q):
        if keep_q[q]:
            assert strip_pad(seq_got[q].tolist()) == strip_pad(seq_exp[q].tolist()), q
    print(f"mT5 V={V_MT5} topk={k} transformers_output: {sum(keep_q)}/{Q} sequences compared")
    assert compared >= total // 3, (compared, total)


def test_generate_bart_60000_vs_oracle():
    """a BART model with a vocabulary past 53 248 (two-CTA clusters) at k = 10; a 50 265-id model does not take the
    cluster kernel"""
    import torch
    from topk_oracle import fm_index_generate_topk_oracle
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import SealBartEngine, fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    from test_decode_gpu import make_inputs
    compared = 0
    for V, Q in ((60000, 16), (50265, 4)):
        seqs = [d.tolist() for d in make_corpus(n_docs=300, doc_len=30, n_phrases=600, seed=3, vocab=V)]
        ora = OracleIndex(seqs)
        idx = FMIndex(); idx.initialize(seqs, in_memory=True)
        model = make_bart(seed=0, layers=2, vocab=V, d_model=128)
        eng = SealBartEngine.from_hf(model, device=0)
        ids, am = make_inputs(np.random.default_rng(V), Q=Q, S=12, vocab=V)
        kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0, topk=10)
        got = fm_index_generate(eng, idx, ids, am, keep_history=True, **kw)
        steps = eng.stat("topk_cluster_steps")
        if V <= MAX_CTA_VOCAB:
            assert steps == 0, steps
            continue
        assert steps > 0, steps
        info = {}
        exp = fm_index_generate_topk_oracle(model, ora, ids, am, info=info, flat_ties=True, **kw)
        keep_q = unambiguous(info)
        worst = compare_generate(got, exp, ora, keep_q)
        compared = sum(keep_q)
        print(f"BART V={V} topk=10: {compared}/{Q} queries compared, {Q - compared} excluded, worst |dscore| "
              f"{worst:.2e}, topk_cluster_steps {steps}")
    assert compared >= 4, compared                  # the 2-layer d_model 128 BART's k-th logit gaps are often < 1e-4


# ---- CUDA-graph replay and query slices ------------------------------------------------------------------------------
def test_graph_replay_bit_identical_mt5(mt5):
    """20 queries x beam 15 with top_k = 10: the eager call, then three identical calls with CUDA graphs on (eager,
    captured, replayed), on the engine's own stream; every call returns the eager records and counts the same steps"""
    from seal_b200.beam_search import generate_records
    ora, idx, teos, models = mt5
    cpu, eng = models[1.0]
    ids, am = t5_sources(np.random.default_rng(70), 20, 14, V_MT5)
    kw = dict(num_beams=15, min_length=8, max_length=8, length_penalty=0.0, top_k=10)
    eng.set_option("cuda_graph", 0)
    try:
        eager = generate_records(eng, idx, ids, am, **kw)
        steps = eng.stat("topk_cluster_steps")
        assert steps == 7, steps                                    # no forced BOS / EOS: every step reads logits
        assert eng.stat("last_used_graph") == 0
        eng.set_option("cuda_graph", 1)
        used = []
        for _ in range(3):
            assert_identical(eager, generate_records(eng, idx, ids, am, **kw))
            used.append(eng.stat("last_used_graph"))
            assert eng.stat("topk_cluster_steps") == steps
        assert used == [0, 1, 1], used
    finally:
        eng.set_option("cuda_graph", -1)


def test_query_slices_bit_identical_mt5():
    """280 queries x beam 15 (more than 2 048 rows per slice; d_model 512, so no GEMM of a slice splits K) with
    top_k = 10: slices on and off give the same records"""
    from seal_b200._lib import check, lib
    from seal_b200.beam_search import SealBartEngine, generate_records
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    from test_query_slices_gpu import PATH_QUERY_SLICES
    seqs = [d.tolist() for d in make_corpus(n_docs=300, doc_len=30, n_phrases=600, seed=5, vocab=V_MT5)]
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    eng = SealBartEngine.from_hf(make_t5("medium", vocab=V_MT5), device=0, gemm_mode=3)
    ids, am = t5_sources(np.random.default_rng(9), 280, 12, V_MT5)
    kw = dict(num_beams=15, min_length=4, max_length=4, length_penalty=0.0, top_k=10)
    recs = []
    for sl in (0, 1):
        check(lib.sealbart_set_option(eng._h, b"query_slices", sl))
        try:
            recs.append(generate_records(eng, idx, ids, am, **kw))
        finally:
            check(lib.sealbart_set_option(eng._h, b"query_slices", -1))
        assert bool(eng.stat("last_paths") & PATH_QUERY_SLICES) == bool(sl)
        assert eng.stat("topk_cluster_steps") == 3
    assert_identical(recs[0], recs[1])
