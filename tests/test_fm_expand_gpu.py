"""FM-index expansion and LF kernels against a brute-force BWT reference, at the kernels' dispatch thresholds and at
wavelet-tree heights 1 ... 24.

Reference: the suffixes of text + [0] sorted by numpy prefix doubling give SA and BWT, and every query follows from
them -- the successor set of [lo, hi) is np.unique(bwt[lo:hi]), an LF step is C[c] plus the occurrences of c before
l and before r + 1 (a searchsorted over (symbol, position) keys), locate is SA[row], extract is a slice of the text,
a document id is a bisection over the beginnings.  Nothing here uses the product's builder.  Two things the plain BWT
does not define come from the oracle: the LF step with r = size() (the reference's first-step quirk, DESIGN.md
section 2; the compiled reference where it was built, else the C port) and the successors of a range ending at
size() + 1 (the C port: the reference sizes that output by sigma, which such a range can exceed).

Dispatch is a pure function of a range's width and of the number of distinct symbol prefixes at each tree level (its
frontier profile), so every case's profile is computed from the reference and test_cases_cover_every_dispatch_threshold
asserts that both sides of each threshold are exercised:
  * warp path (width < kWideRange = 2 048): BFS while the frontier holds <= 32 nodes, then 33 ... 64 depth-first roots
    (expand_dfs_smem), the switch near the root (spread symbols) and at the leaves (clustered symbols);
  * block path (width >= 2 048, block_expand_bfs): the next level goes to global scratch once a non-last level holds
    more than 512 nodes; a full alphabet fills the global frontier's 2^(L-1) entries (L = 12 and 16);
  * the wide-row work list with more wide rows than wide CTAs and more rows than the narrow grid has warps;
  * distinct_count_multi's chunking by range count, by pair words and by bitmap bytes, and the tile carry of
    order_pairs_kernel (symbols more than 256 bitmap words apart).
Only test_numpy_reference_matches_the_oracle runs without a GPU.
"""
import ctypes as C

import numpy as np
import pytest

HEIGHTS = (1, 2, 8, 15, 16, 17, 18, 19, 20, 21, 24)
WIDE = 2048                  # kWideRange (fm_expand.cuh)
SMEM_NODES = 512             # block_expand_bfs moves the next level to global scratch above this many nodes
POISON = 0x5A5A5A5A5A5A5A5A
SENT = np.uint64(0xDEADBEEFDEADBEEF)
U64MAX = (1 << 64) - 1
MARK, DIGITS = 12, list(range(14, 46, 2))          # separator and key digits of the designed texts (never payload)

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------------------------
# brute-force reference
# ------------------------------------------------------------------------------------------------------------------
def suffix_array(t):
    """SA of t (t[-1] = 0 is the unique smallest symbol) by prefix doubling."""
    t = np.asarray(t, dtype=np.int64)
    n = len(t)
    rank = np.unique(t, return_inverse=True)[1].astype(np.int64)
    k = 1
    while True:
        second = np.full(n, -1, dtype=np.int64)
        if k < n:
            second[:n - k] = rank[k:]
        sa = np.lexsort((second, rank))
        r1, r2 = rank[sa], second[sa]
        step = np.zeros(n, dtype=np.int64)
        step[1:] = (r1[1:] != r1[:-1]) | (r2[1:] != r2[:-1])
        rank = np.empty(n, dtype=np.int64)
        rank[sa] = np.cumsum(step)
        if rank[sa[-1]] == n - 1:
            return sa
        k *= 2


class BWTRef:
    def __init__(self, text, oracle=None):
        self.text = np.asarray(text, dtype=np.int64)
        t = np.append(self.text, 0)
        self.m = m = len(t)
        self.L = int(max(int(self.text.max()), 1)).bit_length()
        self.sa = suffix_array(t)
        self.bwt = t[(self.sa - 1) % m]
        self.sorted = np.sort(t)
        self.keys = np.sort(self.bwt * m + np.arange(m))
        self.alphabet = np.unique(t)
        self._oracle = oracle
        self._port = None
        self._succ = {}

    @property
    def oracle(self):
        if self._oracle is None:
            from oracle.fm_oracle import make_backend
            self._oracle = make_backend(self.text.astype(np.uint64))
        return self._oracle

    def C(self, c):
        return np.searchsorted(self.sorted, c, side="left")

    def occ(self, c, x):
        """occurrences of symbol c in bwt[:x] (c < 2^L, x <= m)"""
        c = np.asarray(c, dtype=np.int64); x = np.asarray(x, dtype=np.int64)
        return np.searchsorted(self.keys, c * self.m + x) - np.searchsorted(self.keys, c * self.m)

    def lf_one(self, c, l, r):
        """FMIndex::backward_search_step on the inclusive range [l, r]: (1, 0) for a symbol that does not occur, C[c]
        plus the occurrences of c before l and before r + 1 otherwise (uint64, wrap-around included)."""
        c, l, r = int(c), int(l), int(r)
        if r >= self.m:
            return self.oracle.backward_search_step(c, l, r)
        if c >= (1 << self.L) or (c != 0 and self.C(c + 1) == self.C(c)):
            return 1, 0
        base = int(self.C(c))
        return (base + int(self.occ(c, l))) & U64MAX, (base + int(self.occ(c, r + 1)) - 1) & U64MAX

    def successors(self, lo, hi):
        """(ascending symbols, counts) of BWT[lo, hi); hi <= size() + 1."""
        key = (lo, hi)
        if key not in self._succ:
            if hi <= lo:
                self._succ[key] = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
            elif hi <= self.m:
                self._succ[key] = np.unique(self.bwt[lo:hi], return_counts=True)
            else:
                # The C port: the reference's distinct_count sizes its output by sigma, which such a range can exceed
                # (its result then overruns a heap buffer).
                assert hi == self.m + 1
                from oracle.fm_oracle import PortFM
                if self._port is None:
                    self._port = PortFM(self.text.astype(np.uint64))
                buf = np.zeros(2 * min(hi - lo, 1 << self.L) + 4, dtype=np.uint64)
                k = int(self._port.L.fmo_distinct_count(self._port.h, lo, hi, buf.ctypes.data, len(buf)))
                assert k <= len(buf)
                d = buf[:k].astype(np.int64)
                self._succ[key] = d[0::2], d[1::2]
        return self._succ[key]

    def profile(self, syms):
        """distinct prefixes per tree level 0 ... L"""
        s = np.asarray(syms, dtype=np.int64)
        return [len(np.unique(s >> (self.L - k))) for k in range(self.L + 1)] if len(s) else [0] * (self.L + 1)


# ------------------------------------------------------------------------------------------------------------------
# texts and ranges
# ------------------------------------------------------------------------------------------------------------------
def _key(i):
    return [DIGITS[(i >> 12) & 15], DIGITS[(i >> 8) & 15], DIGITS[(i >> 4) & 15], DIGITS[i & 15]]


def designed_text(L, rng):
    """Payload s_0 ... s_{N-1} written as [s_i, MARK, key(i)]: the suffixes that start with MARK sort by key(i), so the
    BWT rows [C[MARK], C[MARK] + N) hold exactly the payload in order and a payload segment is an SA range whose
    successor set the segment chooses.  Largest symbol 2^(L-1)."""
    top = 1 << (L - 1)

    def spread(cnt, lev):          # cnt distinct prefixes at level lev (the frontier grows near the root)
        return [(j << (L - lev)) + 1 for j in range(cnt)]

    sets = []
    for cnt in (31, 32, 33, 64):
        sets.append(spread(cnt, 7))
    for cnt in (32, 33, 64):
        sets.append([top - j for j in range(cnt)])          # clustered: the frontier grows at the last level
        sets.append([top - 2 * j for j in range(cnt)])      # ... and at the level above it
    if L >= 13:
        sets += [spread(512, 10), spread(513, 11), [top - j for j in range(513)]]
    segs, payload = [], []
    for s in sets:
        reps = 3 if len(s) <= 64 else -(-2100 // len(s))
        seg = np.concatenate([rng.permutation(s) for _ in range(reps)])
        segs.append((len(payload), len(payload) + len(seg)))
        payload.extend(seg.tolist())
    noise = rng.integers(1, top + 1, size=6000)
    noise[::50] = rng.integers(1, 10, size=len(noise[::50]))               # symbols below the shift
    noise[np.isin(noise, [MARK] + DIGITS)] = 1
    noise[7] = top
    payload.extend(noise.tolist())
    text = []
    for i, s in enumerate(payload):
        text += [s, MARK] + _key(i)
    return np.asarray(text, dtype=np.uint64), segs


class Case:
    """One index: its text, reference, product handle (built lazily) and range list."""

    def __init__(self, label, text, segs=()):
        self.label, self.text, self.segs = label, text, segs
        self.ref = BWTRef(text)
        self._fm = None

    @property
    def fm(self):
        if self._fm is None:
            from seal_b200._lib import lib, check
            from seal_b200.cpp_modules.fm_index import FMIndex
            a = np.ascontiguousarray(self.text, dtype=np.uint64)
            out = C.c_void_p()
            check(lib.sealfm_build(a.ctypes.data, len(a), C.byref(out)))          # the host builder (pinned to sdsl)
            fm = FMIndex(); fm._adopt(out.value); fm.to_device(0)
            assert int(lib.sealfm_max_level(fm._handle())) == self.ref.L, self.label
            self._fm = fm
        return self._fm

    def ranges(self, n_random=400, seed=0):
        """(lo, hi) half-open: the threshold cases, then random ones."""
        m = self.ref.m
        rng = np.random.default_rng(seed)
        out = [(0, 0), (5, 5), (m - 1, m - 1), (3, 4), (m - 1, m), (0, 1), (9, 4), (m, m - 2), (0, m), (0, m + 1),
               (m - 7, m), (m - 7, m + 1), (m // 2, m + 1), (m, m + 1)]
        for w in (WIDE - 1, WIDE, WIDE + 1):
            if w <= m:
                out += [(0, w), (m - w, m), (m + 1 - w, m + 1)]
                x = int(rng.integers(0, m - w + 1)); out.append((x, x + w))
        base = int(self.ref.C(MARK))
        for a, b in self.segs:
            out += [(base + a, base + b), (base + a + 1, base + b)]
        w = rng.integers(0, 300, size=n_random)
        w[::5] = rng.integers(WIDE - 5, 5000, size=len(w[::5]))
        w = np.minimum(w, m)
        lo = rng.integers(0, m - w + 1)
        out += list(zip(lo.tolist(), (lo + w).tolist()))
        return [(int(a), int(b)) for a, b in out]


_CASES = {}


def case(label):
    if label not in _CASES:
        if label == "L1":
            _CASES[label] = Case(label, np.ones(3000, dtype=np.uint64))
        elif label == "L2":
            _CASES[label] = Case(label, np.random.default_rng(2).integers(1, 3, size=5000).astype(np.uint64))
        elif label.startswith("full"):           # every symbol of [0, 2^L) occurs
            L = int(label[4:])
            rng = np.random.default_rng(L)
            s = np.arange(1, 1 << L, dtype=np.uint64)
            _CASES[label] = Case(label, np.concatenate([rng.permutation(s), rng.permutation(s)]))
        else:
            L = int(label[1:])
            text, segs = designed_text(L, np.random.default_rng(100 + L))
            _CASES[label] = Case(label, text, segs)
    return _CASES[label]


LABELS = [f"L{L}" for L in HEIGHTS] + ["full12", "full16"]


@pytest.fixture(scope="module")
def need_gpu():
    import torch
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    yield
    for c in _CASES.values():
        c._fm = None


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference itself
# ------------------------------------------------------------------------------------------------------------------
def test_numpy_reference_matches_the_oracle():
    """Row convention, sentinel and C of the numpy reference against the C port's sections, and its queries against the
    oracle (the compiled reference where it was built) on small texts."""
    from oracle.fm_oracle import PortFM, make_backend
    rng = np.random.default_rng(1)
    texts = [np.array([3, 1, 2, 3, 1]), np.ones(40, dtype=np.int64), rng.integers(1, 5, size=300),
             rng.integers(1, 3000, size=500), designed_text(8, rng)[0][:600]]
    for text in texts:
        text = np.asarray(text, dtype=np.uint64)
        ref = BWTRef(text)
        p = PortFM(text)
        assert ref.m == p.size() and ref.L == p.max_level()
        assert np.array_equal(ref.sa, p.section("sa").astype(np.int64))
        assert np.array_equal(ref.bwt, p.section("bwt").astype(np.int64))
        alpha = p.section("alphabet").astype(np.int64)
        assert np.array_equal(ref.alphabet, alpha)
        assert np.array_equal(np.append(ref.C(alpha), ref.m), p.section("C").astype(np.int64))
        o = make_backend(text)
        m = ref.m
        for lo, hi in [(0, m), (1, m), (2, 5), (m - 3, m), (4, 4), (0, 1)] + [tuple(sorted(rng.integers(0, m + 1, 2))) for _ in range(30)]:
            s, c = ref.successors(lo, hi)
            d = np.asarray(o.distinct_count(lo, hi), dtype=np.int64)
            assert np.array_equal(d[0::2], s) and np.array_equal(d[1::2], c), (lo, hi)
        syms = list(ref.alphabet) + [int(ref.alphabet.max()) + 1, 1 << ref.L, 0]
        for c in syms:
            for l, r in [(0, m - 1), (0, 0), (3, 2), (1, m - 1), (m // 2, m - 1), (m - 1, m - 1)]:
                if l > r + 1 or r >= m:
                    continue
                assert ref.lf_one(c, l, r) == o.backward_search_step(int(c), l, r), (c, l, r)
        for row in range(m):
            assert ref.sa[row] == o.locate(row)
        for b, e in [(0, 3), (1, m - 1), (2, 2)]:
            assert o.extract_text(b, e).astype(np.int64).tolist() == ref.text[b:e][::-1].tolist()


# ------------------------------------------------------------------------------------------------------------------
# dispatch coverage
# ------------------------------------------------------------------------------------------------------------------
def classify(ref, lo, hi):
    w = hi - lo if hi > lo else 0
    s, _ = ref.successors(lo, hi)
    P = ref.profile(s)
    L = ref.L
    info = dict(width=w, wide=w >= WIDE, n_sym=len(s), P=P)
    # warp path: BFS while <= 32 nodes; the first level with more is handed to the depth-first phase
    sw = [(k, P[k]) for k in range(L + 1) if P[k] > 32]
    info["dfs_level"], info["dfs_roots"] = sw[0] if sw else (None, 0)
    # block path: the next level goes to global scratch when a non-last level holds more than 512 nodes
    info["block_max"] = max(P[:L - 1]) if L >= 2 else 0
    info["tiles"] = len(np.unique((s >> 5) >> 8)) if len(s) else 0
    return info


@gpu
def test_cases_cover_every_dispatch_threshold(need_gpu):
    seen = set()
    for label in LABELS:
        c = case(label)
        ref, m, L = c.ref, c.ref.m, c.ref.L
        for lo, hi in c.ranges():
            i = classify(ref, lo, hi)
            seen.add(("width", i["width"]))
            if lo > hi: seen.add("lo>hi")
            if hi == m: seen.add("hi=size")
            if hi == m + 1: seen.add("hi=size+1")
            if not i["wide"] and i["dfs_roots"]:
                seen.add(("dfs", i["dfs_roots"] == 33, i["dfs_roots"] > 33))
                seen.add(("dfs near", "leaves" if i["dfs_level"] >= L - 1 else "root" if i["dfs_level"] <= L - 3 else "mid"))
            if not i["wide"] and max(i["P"]) == 32:
                seen.add("bfs only, 32 nodes")
            if i["wide"]:
                seen.add(("block", i["block_max"]))
                if i["P"][L - 1] == 1 << (L - 1) and L in (12, 16):
                    seen.add(("global full", L))
            if i["tiles"] > 1:
                seen.add("tile carry")
    need = [("width", 0), ("width", 1), ("width", WIDE - 1), ("width", WIDE), ("width", WIDE + 1), "lo>hi", "hi=size",
            "hi=size+1", ("dfs", True, False), ("dfs", False, True), ("dfs near", "leaves"), ("dfs near", "root"),
            "bfs only, 32 nodes", ("block", SMEM_NODES), ("block", SMEM_NODES + 1), ("global full", 12),
            ("global full", 16), "tile carry"]
    missing = [n for n in need if n not in seen]
    assert not missing, missing


# ------------------------------------------------------------------------------------------------------------------
# mask sink
# ------------------------------------------------------------------------------------------------------------------
def expected_masks(ref, ranges, vocab, shift, ld):
    rows, syms = [], []
    for r, (lo, hi) in enumerate(ranges):
        s, _ = ref.successors(lo, hi)
        rows.append(np.full(len(s), r, dtype=np.int64)); syms.append(s)
    rows = np.concatenate(rows); syms = np.concatenate(syms)
    keep = (syms != 0) & (syms >= shift) & (syms - shift < vocab)
    tok = syms[keep] - shift
    out = np.zeros((len(ranges), ld), dtype=np.uint32)
    np.bitwise_or.at(out, (rows[keep], tok >> 5), (np.uint32(1) << (tok & 31).astype(np.uint32)))
    return out


def run_masks(fm, ranges, vocab, shift, ld):
    import torch
    from seal_b200._lib import lib, check
    lo = torch.tensor([a for a, _ in ranges], dtype=torch.int64, device="cuda")
    hi = torch.tensor([b for _, b in ranges], dtype=torch.int64, device="cuda")
    mask = torch.full((len(ranges), ld), -1, dtype=torch.int32, device="cuda")         # all-ones bits
    check(lib.sealfm_expand_mask_d(fm._dev(), torch.cuda.current_stream().cuda_stream, len(ranges), lo.data_ptr(),
                                   hi.data_ptr(), mask.data_ptr(), ld, vocab, shift))
    torch.cuda.synchronize()
    return mask.cpu().numpy().view(np.uint32)


def check_masks(c, ranges, combos):
    for vocab, shift, pad in combos:
        ld = -(-vocab // 32) + pad
        got = run_masks(c.fm, ranges, vocab, shift, ld)
        exp = expected_masks(c.ref, ranges, vocab, shift, ld)
        bad = np.nonzero((got != exp).any(axis=1))[0]
        assert not len(bad), f"{c.label} vocab={vocab} shift={shift} ld={ld}: {len(bad)} rows differ, first {ranges[bad[0]]}"


COMBOS = [(v, s, p) for v in (1, 31, 32, 33, 50265) for s in (0, 10) for p in (0, 3)]


@gpu
@pytest.mark.parametrize("label", LABELS)
def test_mask_sink_vs_reference(need_gpu, label):
    c = case(label)
    check_masks(c, c.ranges(), COMBOS)


@gpu
def test_mask_sink_20000_rows_pull_the_wide_work_list(need_gpu):
    """L = 16: 20 000 rows, more than the narrow grid has warps (16 x 4 per SM) and more wide rows than wide CTAs."""
    import torch
    c = case("L16")
    m = c.ref.m
    rng = np.random.default_rng(7)
    R, n_wide = 20000, 1600
    w = np.concatenate([rng.integers(WIDE, 6000, size=n_wide), rng.integers(0, WIDE, size=R - n_wide) // rng.integers(1, 40, size=R - n_wide)])
    lo = rng.integers(0, m - w + 1)
    ranges = list(zip(lo.tolist(), (lo + w).tolist()))
    rng.shuffle(ranges)
    ranges = [(int(a), int(b)) for a, b in ranges] + [(0, m + 1), (m - 3, m + 1)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert len(ranges) > 16 * 4 * sms and n_wide > 4 * sms
    check_masks(c, ranges, [(50265, 10, 0), (50265, 0, 3), (33, 10, 3), (1, 0, 0)])


# ------------------------------------------------------------------------------------------------------------------
# pair sink
# ------------------------------------------------------------------------------------------------------------------
def pairs_raw(fm, lows, highs, out_cap=None, sizing=False):
    from seal_b200._lib import lib
    lows = np.ascontiguousarray(lows, dtype=np.uint64); highs = np.ascontiguousarray(highs, dtype=np.uint64)
    n = len(lows)
    offs = np.full(n + 1, SENT, dtype=np.uint64)
    lp = lows.ctypes.data if n else None
    hp = highs.ctypes.data if n else None
    if sizing:
        rc = lib.sealfm_distinct_count_multi(fm._dev(), n, lp, hp, offs.ctypes.data, None, 0)
        return rc, offs, None
    out = np.full(max(out_cap, 1), SENT, dtype=np.uint64)
    rc = lib.sealfm_distinct_count_multi(fm._dev(), n, lp, hp, offs.ctypes.data, out.ctypes.data, out_cap)
    return rc, offs, out


def expected_pairs(ref, ranges):
    offs, flat = [0], []
    for lo, hi in ranges:
        s, k = ref.successors(lo, hi)
        p = np.empty(2 * len(s), dtype=np.uint64); p[0::2] = s; p[1::2] = k
        flat.append(p); offs.append(offs[-1] + len(p))
    return np.asarray(offs, dtype=np.uint64), np.concatenate(flat) if flat else np.zeros(0, dtype=np.uint64)


def check_pairs(c, ranges):
    eo, ef = expected_pairs(c.ref, ranges)
    lows = [a for a, _ in ranges]; highs = [b for _, b in ranges]
    rc, offs, out = pairs_raw(c.fm, lows, highs, out_cap=len(ef) + 5)
    if rc:
        from seal_b200._lib import lib
        pytest.fail(f"{c.label}: sealfm_distinct_count_multi returned {rc}: {lib.sealfm_last_error().decode()}")
    assert np.array_equal(offs, eo), c.label
    bad = [i for i in range(len(ranges)) if not np.array_equal(out[eo[i]:eo[i + 1]], ef[eo[i]:eo[i + 1]])]
    assert not bad, f"{c.label}: {len(bad)} ranges differ, first {ranges[bad[0]]}"
    assert (out[len(ef):len(ef) + 5] == SENT).all()
    return eo, ef


@gpu
@pytest.mark.parametrize("label", LABELS)
def test_pair_sink_vs_reference(need_gpu, label):
    """The threshold ranges, then 10 000 ranges (three chunks by count) in one call."""
    c = case(label)
    check_pairs(c, c.ranges())
    check_pairs(c, c.ranges(n_random=10000, seed=1))


@gpu
def test_pair_sink_edges(need_gpu):
    from seal_b200._lib import lib
    c = case("L16")
    m = c.ref.m
    rc, offs, _ = pairs_raw(c.fm, [], [], out_cap=0)
    assert rc == 0 and offs[0] == 0
    ranges = c.ranges()
    eo, ef = expected_pairs(c.ref, ranges)
    lows = [a for a, _ in ranges]; highs = [b for _, b in ranges]
    rc, offs, _ = pairs_raw(c.fm, lows, highs, sizing=True)
    assert rc == 0 and np.array_equal(offs, eo)
    rc, offs, out = pairs_raw(c.fm, lows, highs, out_cap=len(ef))
    assert rc == 0 and np.array_equal(out, ef)
    rc, _, _ = pairs_raw(c.fm, lows, highs, out_cap=len(ef) - 1)
    assert rc == -6, rc                                                   # SEALFM_ECAPACITY
    eo, ef = expected_pairs(c.ref, [(0, 5), (3, m + 1)])
    rc, offs, out = pairs_raw(c.fm, [0, 3], [5, m + 1], out_cap=len(ef))
    assert rc == 0 and np.array_equal(offs, eo) and np.array_equal(out, ef)
    rc, _, _ = pairs_raw(c.fm, [0, 3], [5, m + 2], out_cap=len(ef))
    assert rc == -1, rc                                                   # SEALFM_EINVAL
    assert b"size()+1" in lib.sealfm_last_error()


@gpu
def test_pair_sink_full_alphabet_ranges_split_by_pair_words(need_gpu):
    """300 ranges of (almost) the whole L = 16 full-alphabet text: 2^16 pairs each, more than two chunks of 2^24 words."""
    c = case("full16")
    m = c.ref.m
    rng = np.random.default_rng(4)
    lo = rng.integers(0, 60, size=300); hi = m + 1 - rng.integers(0, 60, size=300)
    ranges = [(int(a), int(b)) for a, b in zip(lo, hi)]
    assert sum(2 * min(b - a, 1 << 16) for a, b in ranges) > 2 * (1 << 24)
    eo, _ = check_pairs(c, ranges)
    assert int(eo[1] - eo[0]) >= 2 * 65000


# ------------------------------------------------------------------------------------------------------------------
# LF step, fold, locate, documents, extract
# ------------------------------------------------------------------------------------------------------------------
def lf_triples(ref, rng):
    m, L = ref.m, ref.L
    alpha = ref.alphabet
    syms = [int(v) for v in rng.choice(alpha[alpha > 0], size=min(6, len(alpha) - 1), replace=False)] if len(alpha) > 1 else []
    absent = sorted(set(rng.integers(1, 1 << L, size=50).tolist()) - set(alpha.tolist()))[:3]
    syms += absent + [1 << L, (1 << L) + 5, (1 << 63) + 1, 0]
    rows = [(0, m - 1), (0, m), (5, m), (0, 0), (m - 1, m - 1), (7, 7), (3, 2), (m, m - 1), (m // 3, m - 1)]
    rows += [tuple(sorted(rng.integers(0, m, size=2).tolist())) for _ in range(12)]
    # "absent from the range": a range of one symbol queried with another present one
    one = int(np.nonzero(ref.bwt != ref.bwt[m // 2])[0][0]) if (ref.bwt != ref.bwt[m // 2]).any() else None
    if one is not None:
        syms.append(int(ref.bwt[one])); rows.append((m // 2, m // 2))
    out = []
    for s in syms:
        for l, r in rows:
            out.append((s, l, r))
    return out


@gpu
@pytest.mark.parametrize("label", LABELS)
def test_lf_step_d_vs_reference(need_gpu, label):
    import torch
    from seal_b200._lib import lib, check
    c = case(label)
    ref = c.ref
    rng = np.random.default_rng(11)
    base = lf_triples(ref, rng)
    exp = np.array([ref.lf_one(s, l, r) for s, l, r in base], dtype=np.uint64)
    base = np.array(base, dtype=np.uint64)
    order = rng.permutation(len(base))
    for n in (1, 2, 3, 600001):              # 600 001: odd, and more than one grid pass of 2 x 256 x 8 x 132 triples
        pick = order[np.arange(n) % len(base)]
        trip, e = base[pick], exp[pick]
        s, l, r = (torch.from_numpy(np.ascontiguousarray(trip[:, k]).view(np.int64)).cuda() for k in range(3))
        ol = torch.full((n,), POISON, dtype=torch.int64, device="cuda"); oh = ol.clone()
        check(lib.sealfm_backward_search_step_d(c.fm._dev(), torch.cuda.current_stream().cuda_stream, n, s.data_ptr(),
                                                l.data_ptr(), r.data_ptr(), ol.data_ptr(), oh.data_ptr()))
        torch.cuda.synchronize()
        got = np.stack([ol.cpu().numpy().view(np.uint64), oh.cpu().numpy().view(np.uint64)], axis=1)
        bad = np.nonzero((got != e).any(axis=1))[0]
        assert not len(bad), f"n={n}: {len(bad)} triples differ, first index {bad[0]} {trip[bad[0]]}: {got[bad[0]]} != {e[bad[0]]}"


@gpu
@pytest.mark.parametrize("label", LABELS)
def test_fold_locate_docs_extract_vs_reference(need_gpu, label):
    from seal_b200._lib import lib, check
    c = case(label)
    ref, fm = c.ref, c.fm
    m, n = ref.m, ref.m - 1
    rng = np.random.default_rng(12)
    # backward_search_multi: fold of LF steps from (0, size()), the first step being the reference's quirk
    pats = [[]]
    for ln in range(1, 41):
        a = int(rng.integers(0, n - ln + 1)) if n >= ln else 0
        pats.append(ref.text[a:a + ln].tolist())
    pats += [[int(ref.text[0]), 1 << ref.L], [(1 << ref.L) + 3], [0], ref.text[:3].tolist()[::-1] + [1 << ref.L]]
    exp = []
    for p in pats:
        l, r = 0, m
        for s in p:
            l, r = ref.lf_one(s, l, r)
        exp.append((l, (r + 1) & U64MAX))
    lo, hi = fm.backward_search_multi_batch(pats)
    assert list(zip(lo.tolist(), hi.tolist())) == exp
    # locate at every row residue mod 32, and past the end
    rows = [int(x) for x in rng.integers(0, m, size=400)] + list(range(min(64, m))) + [m - 1, m, m + 5]
    rows += [int(r) for r in range(m) if r % 32 == 31][:5]
    assert {r % 32 for r in rows if r < m} == set(range(min(32, m)))
    got = fm.locate_batch(rows)
    want = [int(ref.sa[r]) if r < m else U64MAX for r in rows]
    assert got.tolist() == want
    # document ids
    beg = np.unique(np.concatenate([[0], rng.integers(0, n, size=40)])).astype(np.uint64)
    check(lib.sealfm_set_beginnings(fm._handle(), beg.ctypes.data, len(beg)))
    rr = np.asarray([r for r in rows if r < m], dtype=np.uint64)
    docs = np.zeros(len(rr), dtype=np.uint64)
    check(lib.sealfm_doc_index_from_rows(fm._dev(), len(rr), rr.ctypes.data, docs.ctypes.data))
    assert np.array_equal(docs, (np.searchsorted(beg, ref.sa[rr.astype(np.int64)], side="right") - 1).astype(np.uint64))
    # extract_text across ISA sample boundaries (every 64th position): the text slice, last position first
    iv = [(0, 0), (0, n), (max(n - 70, 0), n)]
    for k in range(1, n // 64 + 1):
        if k % max(1, n // 64 // 20) == 0:
            iv += [(64 * k - 1, min(64 * k + 1, n)), (max(64 * k - 70, 0), min(64 * k + 70, n))]
    got = fm.extract_text_batch([a for a, _ in iv], [b for _, b in iv])
    for (a, b), g in zip(iv, got):
        assert g.astype(np.int64).tolist() == ref.text[a:b][::-1].tolist(), (a, b)
