"""Plain float64 restatements of the normalisation kernels and the short passes beside them, and the error bounds a correct
kernel must meet against them:
  add_ln_kernel            out = LN(a + b) * g + beta (+ cadd) (+ vec[utterance]), eps 1e-5 (csrc/kernels.cuh)
  cv_ln_kernel             out = LN(a + gelu(y)) * g + beta, or LN(a) (csrc/contentvec.cuh)
  bert_embed_kernel        out = LN((word[id] + type0) + pos[t]) * g + beta, t counted per sentence (csrc/bert.cuh)
  dit_norm(_planes)_kernel v = FiLM(a) (+ gate * y) -> xo; no = LN(v) * (1 + scale) + shift, no affine (csrc/dit.cuh, st_tc.cu)
  cv_gn_kernel<0, 1, 2>    ContentVec's layer-0 conv, GroupNorm with one group per channel over the whole clip, GELU
  cv_gelu_kernel / dit_silu(_planes)_kernel / dit_gate(_planes)_kernel    erf GELU, SiLU, x + gate * y
LayerNorm and GroupNorm are biased (divide by the count), with eps inside the square root.  Planes are the device splits
of the fp32 value the same kernel wrote (conv_ref.split_bf16 / split_bf16_3), checked bit for bit by the GPU tests.

Bounds.  u = 2^-24 (one rounding), CUDA without --use_fast_math: rsqrtf, erff, expf within 2 ulp (2^-22 relative), `/`
and the __f*_rn intrinsics correctly rounded.  A sum computed as any tree in which every term passes through at most k
roundings is within gamma_k sum |t_i| of the exact sum, gamma_k = k u / (1 - k u) (Higham, Accuracy and Stability, 4.2).
The kernels' trees: a warp's row sum adds ceil(C / 32) values per lane and then five butterfly levels (warp_depth), and
GroupNorm adds <= 256 rows per chunk in one thread and then the clip's nch chunk sums in another (gn_depth).  The depth of
that tree, not the count of terms, is what keeps the bound of a row of mean 1e3 and sigma 1e-2 finite at C = 1024.
  inputs      each kernel first forms its fp32 row values v from its inputs; dv_i bounds their error (u per rounding of
              |the rounded value|, plus the GELU error below for cv_ln's y).  xo of dit_norm is v itself.
  mean        s = fp32 sum, m = s / C: |dm| <= ((gamma_ks sum |v_i| + sum dv_i) / C + u |m|) (1 + u).
  centring    d~_i = fl(v~_i - m~) = d_i - dm' + e'_i with |e'_i| <= e_i = dv_i + u (|d_i| + dv_i + dm); ed_i = e_i + dm.
              This is the term that grows with |mean| / sigma: dm is a multiple of |mean| while the output divides by
              sigma, so the bound is computed per row, never as one constant.
  variance    q = fp32 sum of d~_i^2.  The common shift dm' enters only squared (sum d_i = 0): dq <= sum (2 |d_i| e_i +
              e_i^2) + 2 dm sum e_i + C dm^2 + gamma_kq sum (|d_i| + ed_i)^2; var = q / C and S = var + eps each round
              once: dS <= dq / C + u (var + dq / C) + u (S + ...).  With rel = dS / S < 1/2 the exact rstd r = S^-1/2 is
              met by rsqrtf to rho = rel / (2 (1 - rel)) + 2^-22 (1 + rel / (2 (1 - rel))); rel >= 1/2 gives no bound.
  normalised  n~ = fl(d~ * r~): en_i = r (ed_i (1 + rho) + |d_i| rho) + u |n~|.
  affine      fmaf(n~, g, beta): |g| en + u (|out| + |g| en); add_ln's (n~ g + beta) + cadd + vec one rounding more per
              add; dit's fl(fl(n~ fl(1 + scale)) + shift): |1 + s| en + u |n (1 + s)| (two roundings) + u |out|.
  GELU        0.5 x (1 + erff(x * fl(1/sqrt 2))): erff's 2 ulp, the rounding of the argument (erf' <= 1.13) and three more
              roundings: |dgelu| <= 0.5 |x| (2^-22 |erf| + 1.13 * 0.71 |x| 2u + 2u) + 2u |gelu|; gelu is 1.13-Lipschitz.
  SiLU        v / (1 + expf(-v)): expf's 2 ulp and two roundings: 2^-21 |silu| + 2^-149.
  gate        fl(x + fl(gate * y)): u |gate y| + u |out|.
  GroupNorm   layer 0 is a K0-tap fp32 FMA chain on fl(x - mu) (mu the clip's fp32 mean): dv <= (K0 + 9) 2^-23 sum_k
              |w_k| |x - mu|; the statistics as above over the clip's L0 rows with GroupNorm's tree; then fmaf
              and GELU.  The conv of the raw samples differs from the centred one by mu sum_k w_k, the same for every row
              of a channel, which the GroupNorm removes exactly, so the reference convolves the raw samples.
The CPU tests (test_norm_ref.py) pin each reference to torch and to the oracles' modules and check that plausible kernel
mistakes (`mutate=`) break the bound on inputs the GPU tests run."""
import numpy as np
from scipy.special import erf

from conv_ref import offsets, split_bf16, split_bf16_3  # noqa: F401  (re-exported for the tests)

U23 = 2.0 ** -23
U24 = 2.0 ** -24
GN_CHUNK = 256              # contentvec.cuh CVG_CH: layer-0 rows per GroupNorm chunk
ROW_KINDS = ("random", "constant", "offset", "tiny", "spike", "large")


def f64(x):
    return np.asarray(x, np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------------- inputs
def rows_of(kind, n, C, rng):
    """n fp32 rows [n, C] of one kind: random N(0, 1); constant 1.5 (variance 0, and C copies sum exactly); offset: mean
    1e2..1e3 with sigma 1e-2; tiny: sigma 1e-3 around 0 (variance below eps = 1e-5); spike: zeros and one 1e3; large:
    values near +-1e4."""
    if kind == "random":
        x = rng.standard_normal((n, C))
    elif kind == "constant":
        x = np.full((n, C), 1.5)
    elif kind == "offset":
        x = rng.uniform(1e2, 1e3, (n, 1)) + 1e-2 * rng.standard_normal((n, C))
    elif kind == "tiny":
        x = 1e-3 * rng.standard_normal((n, C))
    elif kind == "spike":
        x = np.zeros((n, C))
        x[np.arange(n), rng.integers(0, C, n)] = 1e3
    elif kind == "large":
        x = rng.choice([-1.0, 1.0], (n, C)) * 1e4 + rng.standard_normal((n, C))
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


def mixed_rows(n, C, rng):
    """n rows cycling through ROW_KINDS (the GPU tests' row data): row i has kind ROW_KINDS[i % 6]."""
    x = np.empty((n, C), np.float32)
    for k, kind in enumerate(ROW_KINDS):
        idx = np.arange(k, n, len(ROW_KINDS))
        if idx.size:
            x[idx] = rows_of(kind, idx.size, C, rng)
    return x


def affine(C, rng):
    """LayerNorm weights as trained ones look: g around 1, beta around 0 (fp32)."""
    return (1 + 0.3 * rng.standard_normal(C)).astype(np.float32), (0.2 * rng.standard_normal(C)).astype(np.float32)


def bert_tables(C, P, seed, V=60):
    """The BERT tables of the GPU tests: word rows of every kind (by id), small position and type rows, so that the tiny
    rows' variance is below 1e-5 and positions show in every row; the last word row plus type0 is 1.5 exactly and position
    0 is zero, so that a sentence starting with that piece has one row of variance 0 (whose output is beta exactly)."""
    rng = np.random.default_rng(seed)
    word = mixed_rows(V, C, rng)
    pos = (1e-3 * rng.standard_normal((P, C))).astype(np.float32)
    pos[0] = 0
    type0 = (1e-3 * rng.standard_normal(C)).astype(np.float32)
    word[V - 1] = np.float32(1.5) - type0
    assert np.all(word[V - 1] + type0 == np.float32(1.5))
    return word, pos, type0, affine(C, rng)


# ---------------------------------------------------------------------------------------------------- activations
def gelu(x):
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1 + erf(x / np.sqrt(2)))


def gelu_tanh(x):
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1 + np.tanh(np.sqrt(2 / np.pi) * (x + 0.044715 * x ** 3)))


def gelu_err(x):
    x = np.abs(np.asarray(x, np.float64))
    return 0.5 * x * (2 * U23 * np.abs(erf(x / np.sqrt(2))) + 1.13 * 0.71 * x * 2 * U24 + 2 * U24) + 2 * U24 * np.abs(gelu(x)) + 2.0 ** -149


def silu(x):
    x = np.asarray(x, np.float64)
    return x / (1 + np.exp(-x))


def silu_err(x):
    return 2.0 ** -21 * np.abs(silu(x)) + 2.0 ** -149


# ---------------------------------------------------------------------------------------------------- LayerNorm core
def normalize(v, eps, mutate=None, axis=-1):
    """(v - mean) / sqrt(var + eps) along axis, biased variance, float64.  mutate: "one_pass" (fp32 E[v^2] - mean^2),
    "unbiased" (divide by C - 1), "eps_outside" (1 / sqrt(var) + eps)."""
    v = np.asarray(v, np.float64)
    C = v.shape[axis]
    if mutate == "one_pass":
        v32 = v.astype(np.float32)
        m = (v32.sum(axis, keepdims=True, dtype=np.float32) / np.float32(C)).astype(np.float32)
        e2 = ((v32 * v32).sum(axis, keepdims=True, dtype=np.float32) / np.float32(C)).astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore"):
            return (v - m) / np.sqrt(f64(e2 - m * m) + eps)
    m = v.mean(axis, keepdims=True)
    d = v - m
    var = (d * d).mean(axis, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        if mutate == "unbiased":
            return d / np.sqrt(var * C / (C - 1) + eps)
        if mutate == "eps_outside":
            return d * (1 / np.sqrt(var) + eps)
    if mutate is not None:
        raise ValueError(mutate)
    return d / np.sqrt(var + eps)


def gamma(k):
    """Higham's gamma_k (unit roundoff 2^-24): the relative bound of a sum whose every term passes through k roundings."""
    return k * U24 / (1 - k * U24)


def warp_depth(C):
    """Roundings on a term's path through a warp's row sum: one per add of a lane's ceil(C / 32) values, five butterfly
    levels (the sum of squares rounds at most twice per step: d * d and the add, unless contracted into one FMA)."""
    per = -(-C // 32)
    return per + 5, 2 * per + 5


def gn_depth(L0):
    """The same for GroupNorm's sums: <= 256 rows of a chunk in one thread, then the clip's chunk sums in one thread."""
    nch = -(-L0 // GN_CHUNK)
    return min(GN_CHUNK, L0) + nch, 2 * min(GN_CHUNK, L0) + nch


def normalize_bound(v, dv, eps, depth, axis=-1):
    """Bound on |fl(d~ * r~) - (v - mean) r| for the kernel's fp32 statistics of rows v (float64, exact) whose fp32 values
    are each within dv; depth: the roundings of the sum and of the sum of squares (warp_depth / gn_depth).  Derived in the
    module docstring."""
    v = np.asarray(v, np.float64)
    C = v.shape[axis]
    eps = float(np.float32(eps))
    gs, gq = gamma(depth[0]), gamma(depth[1])
    sm = lambda t: t.sum(axis, keepdims=True)
    m = v.mean(axis, keepdims=True)
    d = v - m
    ad = np.abs(d)
    dm = ((gs * sm(np.abs(v)) + sm(dv)) / C + U24 * np.abs(m)) * (1 + U24)
    e = dv + U24 * (ad + dv + dm)
    ed = e + dm
    var = (d * d).mean(axis, keepdims=True)
    dq = sm(2 * ad * e + e * e) + 2 * dm * sm(e) + C * dm * dm + gq * sm((ad + ed) ** 2)
    S = var + eps
    dvar = dq / C + U24 * (var + dq / C)
    dS = dvar + U24 * (S + dvar)
    rel = dS / S
    a = np.where(rel < 0.5, rel / (2 * (1 - np.minimum(rel, 0.5))), np.inf)
    rho = a + 2 * U23 * (1 + a)
    r = 1 / np.sqrt(S)
    with np.errstate(invalid="ignore"):
        en = np.where(np.isinf(rho), np.inf, r * (ed * (1 + rho) + ad * rho))
    return en + U24 * (ad * r + en)


def within(out, ref, bound):
    """Largest |out - ref| / bound (inf where out is not finite, or where a zero bound is not met exactly)."""
    out = np.asarray(out, np.float64)
    err = np.abs(out - ref)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    ratio = np.where(np.isfinite(out), ratio, np.inf)
    return float(ratio.max()) if ratio.size else 0.0


# ---------------------------------------------------------------------------------------------------- the kernels
def add_ln(a, b, g, beta, cadd=None, vec=None, mutate=None):
    """add_ln_kernel on rows a, b [n, C] (b may be None); cadd [n, C] and vec [n, C] (each row's utterance vector) or
    None.  Returns (ref, bound).  mutate: a normalize() mutation, or "cadd_before" / "vec_before" (added to the input)."""
    a64, C = f64(a), np.shape(a)[1]
    v = a64 + (f64(b) if b is not None else 0)
    dv = U24 * np.abs(v) if b is not None else np.zeros_like(v)
    extra = [f64(t) for t in (cadd, vec) if t is not None]
    if mutate in ("cadd_before", "vec_before"):
        v = v + f64(cadd if mutate == "cadd_before" else vec)
        extra = [f64(t) for t in ((vec,) if mutate == "cadd_before" else (cadd,)) if t is not None]
        mutate = None
    n = normalize(v, 1e-5, mutate)
    en = normalize_bound(v, dv, 1e-5, warp_depth(C))
    g, beta = f64(g), f64(beta)
    ng = n * g
    o = ng + beta
    bound = np.abs(g) * en + U24 * (np.abs(ng) + np.abs(o))
    for t in extra:
        o = o + t
        bound = bound + U24 * np.abs(o)
    return o, bound


def cv_ln(a, y, g, beta, eps, mutate=None):
    """cv_ln_kernel: LN(a + gelu(y)) * g + beta (y None: LN(a)).  mutate: a normalize() mutation, or "tanh" (tanh GELU)."""
    v = f64(a)
    C = v.shape[1]
    dv = np.zeros_like(v)
    if y is not None:
        gy = (gelu_tanh if mutate == "tanh" else gelu)(f64(y))
        v = v + gy
        dv = gelu_err(f64(y)) + U24 * np.abs(v)
    n = normalize(v, eps, None if mutate == "tanh" else mutate)
    en = normalize_bound(v, dv, eps, warp_depth(C))
    g, beta = f64(g), f64(beta)
    o = n * g + beta
    return o, np.abs(g) * en + U24 * (np.abs(o) + np.abs(g) * en)


def bert_positions(lens, mutate=None):
    """Each packed row's position: t within its sentence (mutate "batch_pos": the row's index from the first sentence's
    start instead), and the row indices of the sentences' pieces."""
    off = offsets(lens)
    rows = np.concatenate([np.arange(off[b], off[b] + n) for b, n in enumerate(lens)])
    t = np.concatenate([np.arange(n) for n in lens])
    return (rows if mutate == "batch_pos" else t), rows


def bert_embed(ids, t, word, pos, type0, g, beta, eps, mutate=None):
    """bert_embed_kernel on the rows with piece ids and positions t.  mutate: a normalize() mutation."""
    w = f64(word)[ids] + f64(type0)
    v = w + f64(pos)[t]
    C = v.shape[1]
    dv = U24 * (np.abs(w) + np.abs(v)) + U24 * U24 * np.abs(v)
    n = normalize(v, eps, mutate)
    en = normalize_bound(v, dv, eps, warp_depth(C))
    g, beta = f64(g), f64(beta)
    o = n * g + beta
    return o, np.abs(g) * en + U24 * (np.abs(o) + np.abs(g) * en)


def dit_norm(a, film, y, gate, shift, scale, mutate=None):
    """dit_norm_kernel on rows a [n, C] (already read at the kernel's pitch), film [2C] or None, y [n, C] or None, and each
    row's gate / shift / scale [n, C].  Returns (xo, xo bound, no, no bound).  mutate: a normalize() mutation, "film_swap"
    (gamma and beta exchanged), "scale" (scale for 1 + scale), "gate_at_shift" (the gate read from the shift columns)."""
    v = f64(a)
    C = v.shape[1]
    dv = np.zeros_like(v)
    if film is not None:
        fg, fb = f64(film[:C]), f64(film[C:])
        if mutate == "film_swap":
            fg, fb = fb, fg
        ga = fg * v
        v = ga + fb
        dv = U24 * np.abs(ga) + U24 * np.abs(v) * (1 + U24)
    if y is not None:
        gy = f64(shift if mutate == "gate_at_shift" else gate) * f64(y)
        v = v + gy
        dv = dv + U24 * np.abs(gy) + U24 * (np.abs(v) + dv + U24 * np.abs(gy))
    lm = mutate if mutate in ("one_pass", "unbiased", "eps_outside") else None
    n = normalize(v, 1e-5, lm)
    en = normalize_bound(v, dv, 1e-5, warp_depth(C))
    s1 = f64(scale) + (0 if mutate == "scale" else 1)
    ns = n * s1
    o = ns + f64(shift)
    return v, dv, o, np.abs(s1) * en + U24 * (np.abs(n) * np.abs(s1) + 2 * np.abs(ns) + np.abs(o))


def gate(x, y, g):
    """dit_gate_kernel: x + g * y; returns (ref, bound)."""
    gy = f64(g) * f64(y)
    o = f64(x) + gy
    return o, U24 * (np.abs(gy) + np.abs(o) + U24 * np.abs(gy))


# ---------------------------------------------------------------------------------------------------- GroupNorm
def layer0_rows(n, K0, s0):
    return (n - K0) // s0 + 1 if n >= K0 else 0


def groupnorm_clip(x, w0, g, beta, eps, K0, s0, mutate=None, block=128):
    """cv_gn_kernel's three passes on one clip x (fp32 samples) with the layer-0 weights w0 [C, K0]: gelu(GroupNorm(conv))
    [L0, C] and its bound.  The bound uses the centred samples the kernel convolves.  mutate: "chunk" (statistics per
    256-row chunk), "tanh" (tanh GELU), or a normalize() mutation."""
    x = f64(x)
    L0 = layer0_rows(x.size, K0, s0)
    mu = float(np.float32(x.sum() / x.size))
    idx = np.arange(L0)[:, None] * s0 + np.arange(K0)[None, :]
    X = x[idx]
    Xc = np.abs(X - mu)
    nch = (L0 + GN_CHUNK - 1) // GN_CHUNK
    C = w0.shape[0]
    ref = np.empty((L0, C))
    bound = np.empty((L0, C))
    for c0 in range(0, C, block):
        w = f64(w0[c0:c0 + block])
        v = X @ w.T
        dv = (K0 + 9) * U23 * (Xc @ np.abs(w).T)
        if mutate == "chunk":
            n = np.empty_like(v)
            for j in range(nch):
                n[j * GN_CHUNK:(j + 1) * GN_CHUNK] = normalize(v[j * GN_CHUNK:(j + 1) * GN_CHUNK], eps, axis=0)
        else:
            n = normalize(v, eps, None if mutate == "tanh" else mutate, axis=0)
        en = normalize_bound(v, dv, eps, gn_depth(L0), axis=0)
        gg, bb = f64(g[c0:c0 + block]), f64(beta[c0:c0 + block])
        z = n * gg + bb
        ez = np.abs(gg) * en + U24 * (np.abs(z) + np.abs(gg) * en)
        ref[:, c0:c0 + block] = (gelu_tanh if mutate == "tanh" else gelu)(z)
        bound[:, c0:c0 + block] = 1.13 * ez + gelu_err(z)
    return ref, bound
