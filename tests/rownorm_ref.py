"""float64 references of the row-norm and gate producers (bart_kernels.cuh, t5_kernels.cuh, preln_kernels.cuh) with a
running-error bound that follows each kernel's own operation sequence, the crafted row sets they are checked on, and
a float32 emulation of each kernel's operation order (test_rownorm_host.py checks the bound against it without a GPU;
test_rownorm_gpu.py against the device).

The bound: every fp32 operation adds u |result| (u = 2^-24) to the propagated error of its operands; rsqrtf and tanhf
add 2 ulp (their maximum error in the CUDA C Programming Guide's accuracy tables), an ulp taken as 2^-23 |result|;
a sum of n terms computed through a reduction tree of depth D adds ((1 + u)^D - 1) * sum |term| -- D read from each
kernel, not the sequential sum's n - 1:
  - CTA per row (add_ln_row_kernel, preln_stats): a thread sums its float4 pair as (x + y) + (z + w) and adds the
    two, 5 shuffle levels, ((w0 + w1) + (w2 + w3)) over the 4 warps: D = 3 + 5 + 2 = 10;
  - warp per row (add_ln_kernel, embed_ln_kernel): a lane adds its nv = d / 128 float4 element by element in
    sequence, then 5 shuffle levels: D = 4 nv + 5;
  - T5 RMSNorm (t5_rms_row_kernel<NV>): a thread adds NV float4 terms (x^2 + y^2) + (z^2 + w^2), then 5 + 2 levels:
    D = NV + 2 + 5 + 2 (NV = 2 up to d = 1024, 8 above).
The reference reads the fp32 values the kernel reads, and the fp32 constants it uses (eps 1e-5f, gelu_new's)."""
import numpy as np

U = 2.0 ** -24
ULP_RSQRT = 2          # rsqrtf, tanhf: maximum ulp error
ULP_TANH = 2
EPS_LN = float(np.float32(1e-5))
GELU_K = float(np.float32(0.7978845608028654))
GELU_C = float(np.float32(0.044715))


def gamma_d(D):
    return (1.0 + U) ** D - 1.0


def depth_cta():
    return 10


def depth_warp(d):
    return 4 * (d // 128) + 5


def t5_nv(d):
    return 8 if d > 1024 else 2


def depth_t5(d):
    return t5_nv(d) + 9


def rsqrt_bound(t, et):
    """1 / sqrt(t) and the bound on rsqrtf(t_hat) - 1 / sqrt(t) for |t_hat - t| <= et"""
    r = 1.0 / np.sqrt(t)
    lo = np.maximum(t - et, np.finfo(np.float64).tiny)
    er = 1.0 / np.sqrt(lo) - r
    return r, er + ULP_RSQRT * 2.0 * U * (r + er)


def ln_ref(v, ev, gamma, beta, D, eps=EPS_LN):
    """LayerNorm (biased variance, eps inside) of rows v [rows][d] (float64 of the kernel's input, |kernel's - v| <=
    ev), in the kernels' sequence: mean; c = v - mean; var = sum c^2 / d; r = rsqrt(var + eps); (c * r) * g + b.
    Returns (reference, bound)."""
    v = np.asarray(v, np.float64); ev = np.broadcast_to(np.asarray(ev, np.float64), v.shape)
    g = np.asarray(gamma, np.float64)[None, :]; b = np.asarray(beta, np.float64)[None, :]
    d = v.shape[1]; gd = gamma_d(D)
    S = v.sum(1, keepdims=True)
    eS = ev.sum(1, keepdims=True) + gd * (np.abs(v) + ev).sum(1, keepdims=True)
    mean = S / d
    em = eS / d + U * (np.abs(mean) + eS / d)
    c = v - mean
    ec = ev + em + U * (np.abs(c) + ev + em)
    ac = np.abs(c) + ec
    Q = (c * c).sum(1, keepdims=True)
    eQ = (ac * ac - c * c + U * ac * ac).sum(1, keepdims=True) + gd * (ac * ac * (1 + U)).sum(1, keepdims=True)
    var = Q / d
    evar = eQ / d + U * (var + eQ / d)
    t = var + eps
    et = evar + U * (t + evar)
    r, er = rsqrt_bound(t, et)
    p = c * r
    ep = np.abs(c) * er + r * ec + ec * er
    ep = ep + U * (np.abs(p) + ep)
    pg = (np.abs(p) + ep) * np.abs(g)
    out = p * g + b
    bound = np.abs(g) * ep + U * pg + U * (pg + np.abs(b)) + 2.0 ** -45 * (pg + np.abs(b))
    return out, bound


def rms_ref(v, w, eps, out_scale, D):
    """T5's (w * (v * rsqrt(mean(v^2) + eps))) * out_scale on rows v [rows][d] (the kernel's own fp32 input)"""
    v = np.asarray(v, np.float64); w = np.asarray(w, np.float64)[None, :]
    d = v.shape[1]; eps = float(np.float32(eps)); osc = float(np.float32(out_scale))
    S = (v * v).sum(1, keepdims=True)
    eS = gamma_d(D + 1) * S
    ms = S / d
    ems = eS / d + U * (ms + eS / d)
    t = ms + eps
    et = ems + U * (t + ems)
    r, er = rsqrt_bound(t, et)
    p = v * r
    ep = np.abs(v) * er
    ep = ep + U * (np.abs(p) + ep)
    q = w * p
    eq = np.abs(w) * ep
    eq = eq + U * (np.abs(q) + eq)
    out = q * osc
    bound = abs(osc) * eq + U * (np.abs(out) + abs(osc) * eq) + 2.0 ** -45 * np.abs(out) + 2.0 ** -140
    return out, bound


def gate_ref(h):
    """gelu_new(h[:, :f]) * h[:, f:] of t5_gate_kernel: ((0.5 x) * (1 + tanh(k (x + c x^3)))) * g"""
    h = np.asarray(h, np.float64)
    f = h.shape[1] // 2
    x, g = h[:, :f], h[:, f:]
    ax = np.abs(x)
    ex3 = ax ** 3 * (2 * U + U * U)
    y = GELU_C * x ** 3
    ey = GELU_C * ex3 + U * (np.abs(y) + GELU_C * ex3)
    z = x + y
    ez = ey + U * (np.abs(z) + ey)
    w = GELU_K * z
    ew = GELU_K * ez + U * (np.abs(w) + GELU_K * ez)
    th = np.tanh(w)
    lo = np.maximum(np.abs(w) - ew, 0.0)
    with np.errstate(over="ignore"):
        sech2 = 1.0 / np.cosh(lo) ** 2                # tanh' over the interval: 0 once cosh overflows
    eth = ew * sech2 + ULP_TANH * 2.0 * U * np.abs(th) + 2.0 ** -149
    one = 1.0 + th
    eone = eth + U * (np.abs(one) + eth)
    hx = 0.5 * x
    gl = hx * one
    egl = 0.5 * ax * eone
    egl = egl + U * (np.abs(gl) + egl)
    out = gl * g
    eo = np.abs(g) * egl
    bound = eo + U * (np.abs(out) + eo) + 2.0 ** -45 * np.abs(out) + 2.0 ** -140
    return out, bound


# ---- crafted row sets ----------------------------------------------------------------------------------------------
DISTS = ("zero_mean", "offset", "outlier", "low_var", "constant")


def craft_rows(rng, dist, rows, d):
    """float32 [rows][d]: near-zero mean; a common offset of 2^10 standard deviations (per row 2^6 .. 2^10); one
    column about 100x the rest; variance about 1e-3 (eps = 1e-5 moves the norm by about 0.5 %); constant rows of a
    small dyadic value (0.75)"""
    if dist == "zero_mean":
        x = rng.standard_normal((rows, d))
    elif dist == "offset":
        sig = 2.0 ** rng.uniform(-3, 1, size=(rows, 1))
        ratio = 2.0 ** rng.uniform(6, 10, size=(rows, 1)); ratio[0] = 2.0 ** 10
        x = sig * (ratio * np.sign(rng.standard_normal((rows, 1))) + rng.standard_normal((rows, d)))
    elif dist == "outlier":
        x = rng.standard_normal((rows, d))
        col = rng.integers(0, d, size=rows)
        x[np.arange(rows), col] = 100.0 * np.sign(rng.standard_normal(rows)) * (3 + rng.random(rows))
    elif dist == "low_var":
        x = rng.uniform(-2, 2, size=(rows, 1)) + 0.0316 * rng.standard_normal((rows, d))
    elif dist == "constant":
        x = np.full((rows, d), 0.75)
    else:
        raise ValueError(dist)
    return x.astype(np.float32)


def norm_weights(rng, d):
    """gamma around 1 with spread, beta small"""
    g = (1.0 + 0.25 * rng.standard_normal(d)).astype(np.float32)
    b = (0.1 * rng.standard_normal(d)).astype(np.float32)
    return g, b


def add_parts(rng, v):
    """(a, b) float32 with fp32(a + b) close to v: the residual and the sub-layer output"""
    b = (rng.standard_normal(v.shape) * (0.5 * np.abs(v).mean() + 0.1)).astype(np.float32)
    a = (v.astype(np.float64) - b).astype(np.float32)
    return a, b


def split_k(rng, b, ks, unscale):
    """slices [ks][rows][d] and bias [d] with (sum of slices in index order) * unscale + bias == the returned finished
    value (fp32, as the consumers fold them; unscale a power of two, so no FMA can round differently)"""
    assert unscale == 2.0 ** round(np.log2(unscale))
    bias = (0.05 * rng.standard_normal(b.shape[1])).astype(np.float32)
    tot = (b.astype(np.float64) - bias) / unscale
    w = rng.dirichlet(np.ones(ks), size=b.shape) if ks > 1 else np.ones(b.shape + (1,))
    parts = np.moveaxis((tot[..., None] * w).astype(np.float32), -1, 0).copy()
    y = parts[0].copy()
    for s in range(1, ks):
        y = y + parts[s]
    return parts, bias, (y * np.float32(unscale) + bias).astype(np.float32)


# ---- float32 emulation of the kernels' operation order ---------------------------------------------------------------
def _f(x):
    return np.asarray(x, np.float32)


def _shfl_tree(x):
    """warp_sum over the last axis (32 lanes): v += shfl_xor(v, o), o = 16 .. 1; lane 0's value"""
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = _f(x + x[..., lane ^ o])
    return x[..., 0]


def cta_sum(t4):
    """t4 [rows][n4] fp32 per-float4 terms, n4 <= 128 * NV: thread t adds its terms c4 = t + 128 i in order, then
    warp_sum and ((w0 + w1) + (w2 + w3))"""
    rows, n4 = t4.shape
    nv = -(-n4 // 128)
    pad = np.zeros((rows, 128 * nv), np.float32); pad[:, :n4] = t4
    per = pad.reshape(rows, nv, 128)
    s = per[:, 0].copy()
    for i in range(1, nv):
        s = _f(s + per[:, i])
    w = _shfl_tree(s.reshape(rows, 4, 32))
    return _f(_f(w[:, 0] + w[:, 1]) + _f(w[:, 2] + w[:, 3]))


def warp_sum_row(x4):
    """x4 [rows][d/4][4] fp32: lane l adds the elements of float4 i * 32 + l in order for i < nv, then warp_sum"""
    rows, n4, _ = x4.shape
    nv = n4 // 32
    per = x4.reshape(rows, nv, 32, 4)
    s = np.zeros((rows, 32), np.float32)
    for i in range(nv):
        for k in range(4):
            s = _f(s + per[:, i, :, k])
    return _shfl_tree(s)


def _within_ulps(exact, n, rng):
    """a random fp32 value within n ulp of the float64 value exact: the correctly rounded one moved by up to n steps,
    kept where the move stays within n ulp"""
    r = _f(exact)
    k = rng.integers(-n, n + 1, size=r.shape)
    m = r.copy()
    for _ in range(n):
        m = np.where(k > 0, np.nextafter(m, np.float32(np.inf)), np.where(k < 0, np.nextafter(m, np.float32(-np.inf)), m))
        k = k - np.sign(k)
    ok = np.abs(m.astype(np.float64) - exact) <= n * np.spacing(np.abs(r)).astype(np.float64)
    return np.where(ok, m, r).astype(np.float32)


def _rsqrt(t, rng):
    return _within_ulps(1.0 / np.sqrt(t.astype(np.float64)), ULP_RSQRT, rng)


def emulate_ln(v, gamma, beta, form, rng, one_pass=False, eps=1e-5, unbiased=False):
    """LayerNorm as add_ln_row_kernel / preln_stats (form "cta") or warp_layernorm (form "warp") compute it in fp32,
    with rsqrtf within its 2 ulp.  Mutations: one_pass (E[v^2] - mean^2), eps, unbiased (/ (d - 1))."""
    v = _f(v); rows, d = v.shape
    v4 = v.reshape(rows, d // 4, 4)
    if form == "cta":
        S = cta_sum(_f(_f(v4[..., 0] + v4[..., 1]) + _f(v4[..., 2] + v4[..., 3])))
    else:
        S = warp_sum_row(v4)
    mean = _f(S / np.float32(d))[:, None]
    c = _f(v - mean)
    c4 = (v if one_pass else c).reshape(rows, d // 4, 4)
    sq = _f(c4 * c4)
    if form == "cta":
        Q = cta_sum(_f(_f(sq[..., 0] + sq[..., 1]) + _f(sq[..., 2] + sq[..., 3])))
    else:
        Q = warp_sum_row(sq)
    var = _f(Q / np.float32(d - 1 if unbiased else d))
    if one_pass:
        var = _f(var - _f(mean[:, 0] * mean[:, 0]))
    r = _rsqrt(_f(var + np.float32(eps)), rng)[:, None]
    return _f(_f(_f(c * r) * _f(gamma)[None, :]) + _f(beta)[None, :])


def emulate_rms(v, w, eps, out_scale, rng, residual_scale=False):
    """t5_rms_row_kernel in fp32: returns (residual, out).  Mutation residual_scale: out_scale applied to the residual
    instead of the output."""
    v = _f(v); rows, d = v.shape
    sq = _f(v * v).reshape(rows, d // 4, 4)
    S = cta_sum(_f(_f(sq[..., 0] + sq[..., 1]) + _f(sq[..., 2] + sq[..., 3])))
    r = _rsqrt(_f(_f(S / np.float32(d)) + np.float32(eps)), rng)[:, None]
    out = _f(_f(w)[None, :] * _f(v * r))
    if residual_scale:
        return _f(v * np.float32(out_scale)), out
    return v, _f(out * np.float32(out_scale))


def emulate_gate(h, rng, erf=False):
    """t5_gate_kernel in fp32 with tanhf within its 2 ulp (erf: the exact-erf GELU in its place)"""
    h = _f(h); f = h.shape[1] // 2
    x, g = h[:, :f], h[:, f:]
    if erf:
        from scipy.special import erf as _erf
        gl = _f(0.5 * x.astype(np.float64) * (1 + _erf(x.astype(np.float64) / np.sqrt(2))))
    else:
        x3 = _f(_f(x * x) * x)
        z = _f(x + _f(np.float32(GELU_C) * x3))
        th = np.clip(_within_ulps(np.tanh(_f(np.float32(GELU_K) * z).astype(np.float64)), ULP_TANH, rng), -1, 1)
        gl = _f(_f(np.float32(0.5) * x) * _f(np.float32(1) + th))
    return _f(gl * g)
