"""GPU parity of the decode path (include/sealdec.h) against the CPU/torch restatement of
seal/beam_search.py (oracle/decode_oracle.py) driving transformers' BART in eager fp32.
Integer outputs (tokens, SA ranges, masks) bit-exact; beam scores within 1e-4 (BASELINE.json)."""
import math
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"


def tiny_setup(vocab=2000, n_docs=300, doc_len=30, layers=2, d_model=128, seed=3):
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    docs = make_corpus(n_docs=n_docs, doc_len=doc_len, n_phrases=2 * n_docs, seed=seed, vocab=vocab)
    seqs = [d.tolist() for d in docs]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    model = make_bart(seed=0, layers=layers, vocab=vocab, d_model=d_model)
    return docs, ora, idx, model


def make_inputs(rng, Q, S, vocab):
    import torch
    ids = torch.tensor(rng.integers(4, vocab, size=(Q, S)), dtype=torch.long)
    am = torch.ones_like(ids)
    ids[:, 0] = 0
    for q in range(Q):
        l = int(rng.integers(max(3, S // 2), S + 1))
        ids[q, l - 1] = 2
        ids[q, l:] = 1
        am[q, l:] = 0
    return ids, am


def compare_generate(ours, oracle_out, ora, tol=TOL, force=None, skip=0):
    """ours: [[(score, tokens)]], oracle_out: [[(score, tokens, constrained)]].  Compares, per query,
    the hypotheses that survive the caller's filter (tokens found in the index, SURVEY.md §H4): the
    FM-index query of a hypothesis is force_decoding_from + tokens[1 + skip:] (skip = 1 under a forced
    BOS, which the reference drops before querying, seal/beam_search.py:71,96-101)."""
    assert len(ours) == len(oracle_out)
    worst = 0.0
    force = list(force or [])
    keep = lambda t: ora.get_count(force + list(t[1 + skip:])) > 0
    for q, (a, b) in enumerate(zip(ours, oracle_out)):
        fa = sorted([(tuple(t), s) for s, t in a if keep(t)])
        fb = sorted([(tuple(t), s) for s, t, _ in b if keep(t)])
        assert [x[0] for x in fa] == [x[0] for x in fb], (
            f"query {q}: hypothesis token sets differ\nours-only: {sorted(set(x[0] for x in fa) - set(x[0] for x in fb))[:5]}"
            f"\noracle-only: {sorted(set(x[0] for x in fb) - set(x[0] for x in fa))[:5]}")
        for (ta, sa), (tb, sb) in zip(fa, fb):
            worst = max(worst, abs(sa - sb))
            assert abs(sa - sb) <= tol, (q, ta, sa, sb)
    return worst


def test_bart_step_logits_vs_hf_tiny():
    import torch
    from oracle.decode_oracle import HFBartStepper
    from seal_b200.beam_search import SealBartEngine
    docs, ora, idx, model = tiny_setup()
    eng = SealBartEngine.from_hf(model, device=0)
    rng = np.random.default_rng(1)
    ids, am = make_inputs(rng, Q=3, S=11, vocab=2000)
    B = 4
    for t in (1, 2, 5):
        dec = torch.tensor(rng.integers(4, 2000, size=(3 * B, t)), dtype=torch.long); dec[:, 0] = 2
        ref = HFBartStepper(model, ids, am, B)(dec).numpy()
        got = eng.debug_step_logits(ids.numpy(), am.numpy(), B, dec.numpy())
        fin = np.isfinite(ref)
        assert np.array_equal(np.isfinite(got), fin)
        err = np.abs(got[fin] - ref[fin]).max()
        print(f"tiny t={t}: max |dlogit| = {err:.3e}")
        assert err < 2e-5, (t, err)


def test_bart_step_logits_vs_hf_bart_large():
    """BartConfig() == bart-large, seeded random weights; teacher-forced logits at t=1 and t=4."""
    import torch
    from oracle.decode_oracle import make_bart, HFBartStepper
    from seal_b200.beam_search import SealBartEngine
    model = make_bart(seed=0)
    eng = SealBartEngine.from_hf(model, device=0)
    rng = np.random.default_rng(2)
    ids, am = make_inputs(rng, Q=2, S=9, vocab=50265)
    B = 3
    for t in (1, 4):
        dec = torch.tensor(rng.integers(4, 50265, size=(2 * B, t)), dtype=torch.long); dec[:, 0] = 2
        ref = HFBartStepper(model, ids, am, B)(dec).numpy()
        got = eng.debug_step_logits(ids.numpy(), am.numpy(), B, dec.numpy())
        fin = np.isfinite(ref)
        assert np.array_equal(np.isfinite(got), fin)
        err = np.abs(got[fin] - ref[fin]).max()
        lp_ref = torch.log_softmax(torch.tensor(ref), -1).numpy(); lp_got = torch.log_softmax(torch.tensor(got), -1).numpy()
        lerr = np.abs(lp_got[fin] - lp_ref[fin]).max()
        print(f"bart-large t={t}: max |dlogit| = {err:.3e}, max |dlogprob| = {lerr:.3e}")
        # fp32 SIMT GEMM: ~7e-6; 3xFP16 tensor-core GEMM with 256-K TMEM chunks: ~1.3e-5; 3xTF32
        # (SEALB200_GEMM=1,2): ~2e-5.  The contract is 1e-4 on summed beam scores, enforced by the
        # generate tests below.
        assert lerr < 4e-5, (t, err, lerr)


@pytest.mark.parametrize("kw", [
    dict(num_beams=5, min_length=8, max_length=8, length_penalty=0.0),
    dict(num_beams=3, min_length=2, max_length=6, length_penalty=1.0),
    dict(num_beams=4, min_length=0, max_length=7, length_penalty=0.0, always_allow_eos=True),
    dict(num_beams=4, min_length=0, max_length=7, length_penalty=0.0, stop_at_count=3),
    dict(num_beams=5, min_length=3, max_length=7, length_penalty=0.0, force_decoding_from="doc"),
    dict(num_beams=3, min_length=0, max_length=6, length_penalty=0.0, forced_bos_token_id=0),
    dict(num_beams=4, min_length=0, max_length=6, length_penalty=0.0, disable_fm_index=True),
    dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0),
    # title-style pass (seal/retrieval.py:162-176): own eos id, decoding forced to start at a document end
    dict(num_beams=5, min_length=0, max_length=9, length_penalty=0.0, eos_token_id=777, force_decoding_from=[2]),
])
def test_fm_index_generate_vs_oracle_tiny(kw):
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny_setup()
    kw = dict(kw)
    if kw.get("force_decoding_from") == "doc":
        kw["force_decoding_from"] = docs[5].tolist()[3:5]
    rng = np.random.default_rng(4)
    ids, am = make_inputs(rng, Q=6, S=12, vocab=2000)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"),
                             skip=1 if kw.get("forced_bos_token_id") is not None else 0)
    print(f"{kw}: worst |dscore| = {worst:.3e}; hyps/query = {[len(x) for x in got]}")
    if not kw.get("disable_fm_index"):
        assert max(len(x) for x in got) > kw["num_beams"]


@pytest.mark.parametrize("case", range(9))
def test_fm_index_generate_vs_reference_code_fixture(case):
    """tests/golden/decode_golden.json holds what the reference's OWN seal/beam_search.py returned (run
    unmodified in the build container by tests/golden/make_decode_golden.py) for these inputs."""
    import json
    import torch
    from oracle.decode_oracle import make_bart
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import fm_index_generate
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus
    with open(os.path.join(os.path.dirname(__file__), "golden", "decode_golden.json")) as f:
        g = json.load(f)
    c = g["cases"][case]
    docs = make_corpus(**g["corpus"])
    seqs = [d.tolist() for d in docs]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    model = make_bart(**g["model"])
    kw = c["kw"]
    got = fm_index_generate(model, idx, torch.tensor(c["input_ids"]), torch.tensor(c["attention_mask"]), keep_history=True, **kw)
    exp = [[(s, t, None) for s, t in q] for q in c["hyps"]]
    worst = compare_generate(got, exp, ora, force=kw.get("force_decoding_from"),
                             skip=1 if kw.get("forced_bos_token_id") is not None else 0)
    print(f"reference-code fixture {kw}: worst |dscore| = {worst:.3e}")


@pytest.mark.parametrize("gemm_mode", [3, 5])
def test_fm_index_generate_many_rows_tiny(gemm_mode, monkeypatch):
    """40 queries x 8 beams = 320 live rows: more than one 128-row GEMM tile, so the persistent GEMM (gemm_mode 3,
    the default) and the 2-CTA cluster GEMM (gemm_mode 5) run inside the decode loop (odd number of row tiles: the
    last cluster has an empty second CTA)."""
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200.beam_search import fm_index_generate
    monkeypatch.setenv("SEALB200_GEMM", str(gemm_mode))
    docs, ora, idx, model = tiny_setup()
    rng = np.random.default_rng(21)
    ids, am = make_inputs(rng, Q=40, S=14, vocab=2000)
    kw = dict(num_beams=8, min_length=3, max_length=8, length_penalty=0.0)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst = compare_generate(got, exp, ora)
    print(f"many rows: worst |dscore| = {worst:.3e}; hyps/query = {len(got[0])}")


def test_fm_index_generate_long_wide_shapes():
    """Shapes beyond the benchmark's: source longer than one 32-key chunk (S = 45), more beams than one
    16-row attention sweep (20), more decoder positions than the 12-key self-attention fast path (16)."""
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny_setup(n_docs=600, doc_len=40)
    rng = np.random.default_rng(9)
    ids, am = make_inputs(rng, Q=3, S=45, vocab=2000)
    kw = dict(num_beams=20, min_length=0, max_length=16, length_penalty=0.5)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst = compare_generate(got, exp, ora)
    print(f"long/wide shapes: worst |dscore| = {worst:.3e}; hyps/query = {[len(x) for x in got]}")


def test_fm_index_generate_sample_corpus_bart_large():
    """BASELINE.json configs[0]: the README's 3-document sample (README.md:149-153) through a fixed
    toy word->id table, 1 query, beam 5, bart-large (seeded random weights)."""
    import torch
    from oracle.decode_oracle import make_bart, fm_index_generate_oracle
    from oracle.fm_oracle import OracleIndex
    from seal_b200.beam_search import fm_index_generate, generate_records
    from seal_b200.index import FMIndex
    corpus = ["Doc 1 @@ This is a sample document",
              "Doc 2 @@ And here you find the final one",
              "Doc 3 @@ This is another sample document"]
    words = sorted({w for line in corpus for w in line.split()})
    table = {w: 1000 + 7 * i for i, w in enumerate(words)}
    seqs = [[table[w] for w in line.split()] + [2] for line in corpus]
    ora = OracleIndex(seqs)
    idx = FMIndex(); idx.initialize(seqs, in_memory=True)
    assert idx.occurring_distinct == ora.occurring_distinct
    model = make_bart(seed=0)
    ids = torch.tensor([[0, 1000, 1007, 1014, 1021, 2]]); am = torch.ones_like(ids)
    kw = dict(num_beams=5, min_length=10, max_length=10, length_penalty=0.0)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst = compare_generate(got, exp, ora)
    print(f"sample corpus: worst |dscore| = {worst:.3e}, {len(got[0])} hyps")
    # SA ranges reported for valid hypotheses equal the oracle's get_range
    rec = generate_records(model, idx, ids, am, **kw)
    n = 0
    for h in range(rec["scores"].shape[1]):
        if rec["valid"][0, h] == 1:
            toks = rec["tokens"][0, h, : rec["lens"][0, h]].tolist()
            assert (int(rec["lo"][0, h]), int(rec["hi"][0, h])) == ora.get_range(toks[1:]), toks
            n += 1
    assert n > 0


def test_fm_index_generate_bart_large_batch20_beam15():
    """The reference's operating point (README.md:76-83): batch 20, beam 15, body n-grams of 10,
    on a 200 k-token phrase corpus; oracle = HF BART eager fp32 on the same GPU + CPU FM oracle."""
    import torch
    from oracle.decode_oracle import make_bart, fm_index_generate_oracle
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
    kw = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    model_gpu = model.to("cuda")
    exp = fm_index_generate_oracle(model_gpu, ora, ids.cuda(), am.cuda(), **kw)
    worst = compare_generate(got, exp, ora)
    print(f"batch20/beam15: worst |dscore| = {worst:.3e}; hyps/query min {min(len(x) for x in got)} max {max(len(x) for x in got)}")


@pytest.mark.parametrize("kw", [
    dict(),
    dict(always_allow_eos=True),
    dict(stop_at_count=2),
    dict(force_decoding_from="doc"),
    dict(forced_bos_token_id=0),
])
def test_index_based_logits_processor_vs_oracle(kw):
    """Stateless HF-protocol hook, seal/beam_search.py:62-140: exact mask equality (scores + {0,-inf})."""
    import torch
    from oracle.decode_oracle import IndexBasedLogitsProcessorOracle
    from seal_b200.beam_search import IndexBasedLogitsProcessor
    docs, ora, idx, _ = tiny_setup(layers=1)
    kw = dict(kw)
    if kw.get("force_decoding_from") == "doc":
        kw["force_decoding_from"] = docs[9].tolist()[2:4]
    V, B, nb = 2000, 4, 3
    rng = np.random.default_rng(8)
    po = IndexBasedLogitsProcessorOracle(ora, B, pad_token_id=1, eos_token_id=2, **kw)
    pg = IndexBasedLogitsProcessor(idx, B, pad_token_id=1, eos_token_id=2, **kw)
    for t in (1, 2, 3, 5):
        rows = []
        for r in range(nb * B):
            d = docs[int(rng.integers(0, len(docs)))].tolist()
            a = int(rng.integers(0, len(d) - 8))
            sent = [2] + d[a:a + t - 1]
            u = rng.random()
            if t > 1 and u < 0.15: sent[-1] = 2              # row that ended in eos
            elif t > 1 and u < 0.25: sent[-1] = 1            # ... in pad
            elif t > 1 and u < 0.35: sent[-1] = int(rng.integers(4, V))   # token that breaks the n-gram
            rows.append(sent)
        ids = torch.tensor(rows, dtype=torch.long)
        scores = torch.randn(nb * B, V)
        exp = po(ids.clone(), scores.clone())
        got = pg(ids.cuda(), scores.cuda()).cpu()
        assert torch.equal(torch.isinf(exp), torch.isinf(got)), (t, kw)
        fin = ~torch.isinf(exp)
        assert torch.equal(exp[fin], got[fin])


def test_headline_config_q1000_10M_index_vs_oracle_sample():
    """The benchmarked configuration itself (bench.py, BASELINE.json configs[1]): 1 000 queries x beam 15 in ONE batch
    on the 10 M-token index with BART-large -- M = 15 000-row GEMM tiles, the compact first step, the packed encoder.
    Checked: (a) every first-step record's [lo, hi) (30 000 ranges, the 15 000 new beams among them) against the
    compiled reference FM-index; (b) a seeded sample of 8 queries against the reference algorithm (oracle decode, HF
    BART eager fp32 on the same GPU): same hypotheses, |dscore| <= 1e-4, SA ranges == get_range."""
    import torch
    from oracle.decode_oracle import make_bart, fm_index_generate_oracle
    from oracle.fm_oracle import OracleIndex, RefFM, PortFM, ref_available
    from seal_b200.beam_search import SealBartEngine, generate_records, records_to_output
    from seal_b200.cpp_modules.fm_index import FMIndex as RawFM
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus, make_queries, corpus_symbols
    docs = make_corpus()
    sym = corpus_symbols(docs)
    index = FMIndex(); RawFM.initialize(index, sym)
    index.beginnings = list(range(0, docs.size + 1, docs.shape[1])); index._sync_beginnings(); index.to_device(0)
    index.occurring_distinct, index.occurring_counts = index.get_distinct_count(0, len(index))
    ora = OracleIndex(_raw=(RefFM if ref_available() else PortFM)(sym))
    ora.beginnings = list(index.beginnings)
    ora.occurring_distinct, ora.occurring_counts = ora.get_distinct_count(0, len(ora))
    assert index.occurring_distinct == ora.occurring_distinct
    model = make_bart(seed=0)
    eng = SealBartEngine.from_hf(model, device=0)
    ids, am = make_queries(1000, seed=4321)
    kw = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0)
    rec = generate_records(eng, index, ids, am, forced_bos_token_id=None, **kw)
    # (a) first-step records
    K = 30
    n = 0
    for q in range(1000):
        for h in range(K):
            if rec["valid"][q, h] == 1:
                toks = rec["tokens"][q, h, :rec["lens"][q, h]].tolist()
                assert (int(rec["lo"][q, h]), int(rec["hi"][q, h])) == ora.get_range(toks[1:]), (q, h, toks)
                n += 1
    assert n >= 15000
    # (b) sampled queries
    sample = sorted(np.random.default_rng(7).choice(1000, size=8, replace=False).tolist())
    model_gpu = model.to("cuda")
    exp = fm_index_generate_oracle(model_gpu, ora, torch.tensor(ids[sample]).cuda(), torch.tensor(am[sample]).cuda(), use_cache=True, **kw)
    got_all = records_to_output({k: v[sample] for k, v in rec.items() if v is not None}, 0.0)
    worst = compare_generate(got_all, exp, ora)
    for i, q in enumerate(sample):
        for h in range(rec["scores"].shape[1]):
            if rec["valid"][q, h] == 1:
                toks = rec["tokens"][q, h, :rec["lens"][q, h]].tolist()
                assert (int(rec["lo"][q, h]), int(rec["hi"][q, h])) == ora.get_range(toks[1:])
    print(f"headline config: {n} first-step ranges exact; sample {sample}: worst |dscore| = {worst:.3e}")


def test_device_records_graph_replay_and_host_api_agree():
    """generate_records_device (sealdec_generate_dx): the 1st call of a shape runs eagerly, the 2nd is captured into a
    CUDA graph, later ones replay it -- all must give the records of the host-buffer API bit for bit."""
    import torch
    from seal_b200._lib import lib
    from seal_b200.beam_search import SealBartEngine, generate_records, generate_records_device
    docs, ora, idx, model = tiny_setup()
    eng = SealBartEngine.from_hf(model, device=0)
    rng = np.random.default_rng(31)
    ids, am = make_inputs(rng, Q=5, S=12, vocab=2000)
    kw = dict(num_beams=4, min_length=6, max_length=6, length_penalty=0.0)
    host = generate_records(eng, idx, ids.numpy(), am.numpy(), **kw)
    ids_d = ids.cuda(); am_d = am.cuda()
    out = None
    used = []
    for it in range(4):
        out = generate_records_device(eng, idx, ids_d, am_d, out=out, src_tokens=int(am.sum()), **kw)
        torch.cuda.synchronize()
        used.append(int(lib.sealbart_get_stat(eng._h, b"last_used_graph")))
        got = out.host()
        assert not got["errors"].any()
        for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
            assert np.array_equal(got[k], host[k]), (it, k)
    assert used[-1] == 1 and used[0] == 0, used
    # a wrong source-token count is reported, not silently used
    lib.sealbart_set_option(eng._h, b"cuda_graph", 0)
    bad = generate_records_device(eng, idx, ids_d, am_d, src_tokens=int(am.sum()) - 1, **kw)
    assert bad.host()["errors"][2] == 1


def test_fp16_range_overflow_falls_back_to_tf32():
    """ADVICE r1: activations beyond the fp16 range of the default 3xFP16 GEMM mode.  The host-buffer API repeats the
    pass with the 3xTF32 kernels and still matches eager fp32; the device API raises error flag [1]."""
    import torch
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200._lib import lib
    from seal_b200.beam_search import SealBartEngine, fm_index_generate, generate_records_device
    docs, ora, idx, model = tiny_setup()
    with torch.no_grad():
        model.model.decoder.layers[0].fc1.weight.mul_(2e6)        # fc1 outputs ~ 5e5 > 65504
    eng = SealBartEngine.from_hf(model, device=0)
    rng = np.random.default_rng(5)
    ids, am = make_inputs(rng, Q=3, S=10, vocab=2000)
    kw = dict(num_beams=4, min_length=5, max_length=5, length_penalty=0.0)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(eng, idx, ids, am, keep_history=True, **kw)
    assert int(lib.sealbart_get_stat(eng._h, b"overflow_fallbacks")) >= 1
    worst = compare_generate(got, exp, ora, tol=2e-4)
    print(f"overflow fallback: worst |dscore| = {worst:.3e}")
    out = generate_records_device(eng, idx, ids.cuda(), am.cuda(), **kw)
    assert out.host()["errors"][1] == 1


@pytest.mark.parametrize("kw", [
    dict(num_beams=3, min_length=0, max_length=40, length_penalty=1.0, disable_fm_index=True),
    dict(num_beams=4, min_length=0, max_length=36, length_penalty=0.0),
])
def test_fm_index_generate_beyond_32_positions(kw):
    """max_length > 32 (README.md:209-216 decodes with max_length=100): the long self-attention kernel."""
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny_setup(n_docs=400, doc_len=60)
    rng = np.random.default_rng(17)
    ids, am = make_inputs(rng, Q=2, S=10, vocab=2000)
    exp = fm_index_generate_oracle(model, ora, ids, am, **kw)
    got = fm_index_generate(model, idx, ids, am, keep_history=True, **kw)
    worst = compare_generate(got, exp, ora, tol=2e-4)
    print(f"{kw}: worst |dscore| = {worst:.3e}")


@pytest.mark.parametrize("kw", [
    dict(num_beams=4, min_length=0, max_length=8, length_penalty=1.0, always_allow_eos=True),
    dict(num_beams=3, min_length=2, max_length=7, length_penalty=0.0, always_allow_eos=True),
    dict(num_beams=5, min_length=0, max_length=9, length_penalty=1.0, disable_fm_index=True),
])
def test_fm_index_generate_keep_history_false(kw):
    """The signature's default scorer path (seal/beam_search.py:406,505-515; README.md:209-216): transformers' stock
    BeamSearchScorer.  Oracle = the loop with the restated 4.13 scorer inside (parity unpinned for that class, see
    oracle/decode_oracle.py); product = same kernels + host replay of the scorer over the records."""
    import torch
    from oracle.decode_oracle import fm_index_generate_oracle
    from seal_b200.beam_search import fm_index_generate
    docs, ora, idx, model = tiny_setup()
    rng = np.random.default_rng(14)
    ids, am = make_inputs(rng, Q=5, S=12, vocab=2000)
    exp = fm_index_generate_oracle(model, ora, ids, am, keep_history=False, **kw)
    got = fm_index_generate(model, idx, ids, am, **kw)                     # keep_history defaults to False
    assert all(len(g) <= kw["num_beams"] for g in got)
    worst = compare_generate(got, exp, ora)
    print(f"keep_history=False {kw}: worst |dscore| = {worst:.3e}; hyps/query = {[len(x) for x in got]}")
    if kw.get("disable_fm_index"):
        seq_exp = fm_index_generate_oracle(model, ora, ids, am, keep_history=False, transformers_output=True, **kw)
        seq_got = fm_index_generate(model, idx, ids, am, transformers_output=True, **kw)
        assert torch.equal(seq_got.cpu(), seq_exp)


def test_batch20_graph_replay_bart_large_is_bit_stable():
    """The reference's operating point through the host-buffer API, three times: eager, captured, replayed (CUDA graph
    with programmatic dependent launches between the ~1 900 kernels) -- all three must return identical records."""
    from oracle.decode_oracle import make_bart
    from seal_b200._lib import lib
    from seal_b200.beam_search import SealBartEngine, generate_records
    from seal_b200.index import FMIndex
    from seal_b200.synthetic import make_corpus, make_queries
    docs = make_corpus(n_docs=2000, doc_len=100, n_phrases=4000, seed=21)
    idx = FMIndex(); idx.initialize([d.tolist() for d in docs], in_memory=True)
    eng = SealBartEngine.from_hf(make_bart(seed=0), device=0)
    ids, am = make_queries(20, seed=77)
    kw = dict(num_beams=15, min_length=10, max_length=10, length_penalty=0.0)
    recs = [generate_records(eng, idx, ids, am, **kw) for _ in range(4)]
    assert int(lib.sealbart_get_stat(eng._h, b"last_used_graph")) == 1
    for r in recs[1:]:
        for k in ("scores", "lens", "tokens", "valid", "lo", "hi"):
            assert np.array_equal(r[k], recs[0][k]), k
