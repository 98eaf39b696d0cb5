"""Plain float64 restatements of the duration path's kernels and the error bounds a correct kernel must meet against them:
  dds_stack        the three DDSConv layers (csrc/kernels.cuh dds_layer_kernel; modules.py:96-108), with the ConvFlow front
  spline_inverse   the rational-quadratic spline inverse with linear tails (spline_inverse_kernel; transforms.py:55-193)
  vits_durations   ceil durations, their scan, y_len = max(sum, 1), the frame offsets and the frame -> token map
                   (duration_kernel, sample_prior_kernel; models.py:1689-1700)
  stt_durations    the StableTTS duration rule and the expansion to frames (stt_dur_kernel, stt_expand_kernel,
                   stt_pause_fill_kernel; matcha_tts.py:143-197)
Rows are packed as the engine packs them (conv_ref.offsets: SEQ_GAP = 8 rows between utterances).

Bounds.  Each bound is a first-order forward error analysis of the kernel's fp32 op sequence, evaluated on the float64
intermediates.  A correctly rounded op (+ - * /, sqrt, fmaf) contributes u = 2^-24 of its result.  A library function
contributes its documented maximum error (CUDA C Programming Guide, "Mathematical Functions", single precision): expf 2
ulp, log1pf 1 ulp, erff 2 ulp, rsqrtf 2 ulp; one ulp is at most 2u of the value.
  - The spline is written once over a tape of ops (`_spline`), each op's result multiplied by (1 + d_k).  dy/dd_k is taken by
    complex-step differentiation (exact to rounding, no cancellation), and the bound is 2 * sum_k |dy/dd_k| * err_k.  The
    factor 2 covers the dropped second-order terms (products of two d's, each at most a few u).
  - The DDS layer propagates an absolute error per element through each stage: the k-tap sum (gamma_(k+1)), the 1x1 conv's
    fmaf chain (running error bound: u times the sum of the float64 partial sums, in the kernel's channel order),
    LayerNorm's sums (a 5-level warp butterfly and the warps in order: gamma_(5 + C/32 + 1)), LayerNorm (to first order the
    mean moves by the inputs' mean error and the variance by 2 mean(|v - mean| * error)), GELU (|gelu'| <= 1.13) and the
    residual.  Signs are taken worst case at every stage, which compounds across layers, so each layer is checked on its
    own, on the kernel's output of the layer before (vtts_debug_dds returns all three): the bound stays within a few 1e-4 of
    the output's magnitude, and test_duration_ref.py checks that it rejects a 1e-3 relative error and a skipped layer.
  - Durations: w = exp((z - m) * exp(-logs)) * length_scale has a relative error of at most 6u |logw| + 5u (two expf, three
    roundings).  ceil(w) is bit-exact except where the float64 w lies within that bound of an integer: there a neighbouring
    integer is acceptable too.  Everything after ceil is integer arithmetic and follows exactly from the kernel's own ceil.
  - StableTTS: the sigmoid sum over DC channels, summed in channel order, is within (DC + 6) u * sum + u |a| of the float64
    sum; rint is compared as ceil is.  The expansion copies rows, and the prior rows are two rounded ops: bit-exact against a
    NumPy float32 emulation."""
import numpy as np

from conv_ref import SEQ_GAP, offsets  # noqa: F401  (the packing)

U = 2.0 ** -24
ULP = 2 * U                       # one fp32 ulp, relative to the value, at most
EXPF, LOG1PF, ERFF, RSQRTF = 2 * ULP, 1 * ULP, 2 * ULP, 2 * ULP
LN_EPS = 1e-5
CEIL_CAP = 1.0e6                  # duration_kernel: frames of one token at most
INT32_MAX = 2 ** 31 - 1


# ---------------------------------------------------------------------------------------------------- DDSConv
def _gelu(v):
    from scipy.special import erf
    return 0.5 * v * (1.0 + erf(v / np.sqrt(2.0)))


def _ln(v, e, g, b):
    """LayerNorm over the channels of v [L, C] (float64) with input error e [L, C]: value and error bound of the kernel's
    block_ln_stats + (v - mean) * rstd * g + b (fp32 sums of C terms, rsqrtf, three roundings)."""
    C = v.shape[1]
    n_red = 5 + C // 32 + 1          # the sums: a 5-level warp butterfly, the warps' partials in order, / C
    mu = v.mean(1, keepdims=True)
    d = v - mu
    var = (d * d).mean(1, keepdims=True)
    sd = np.sqrt(var + LN_EPS)
    y = d / sd * g + b
    # first order: the mean moves by mean(e), the variance by 2 mean(|d| dd); plus the fp32 sums of C terms and / C
    dmu = e.mean(1, keepdims=True) + n_red * U * np.abs(v).mean(1, keepdims=True)
    dd = e + dmu + U * np.abs(d)
    dvar = (n_red + 2) * U * var + 2 * (np.abs(d) * dd).mean(1, keepdims=True) + U * LN_EPS   # (+ eps rounded to fp32)
    drs = dvar / (2 * (var + LN_EPS)) + RSQRTF + U                # relative error of rstd
    dy = np.abs(g) * (dd / sd + np.abs(d) / sd * drs) + 3 * U * (np.abs(d / sd * g) + np.abs(b))
    return y, dy


def _gelu_err(v, dv):
    """GELU of the kernel (0.5 x (1 + erff(x / sqrt 2))): value and error bound given an input error dv."""
    gv = _gelu(v)
    return gv, 1.13 * dv + 0.5 * np.abs(v) * (ERFF + 2 * U) + 3 * U * np.abs(gv)


def _running(g, W, bias, chunk=16):
    """Running error bound of the kernel's 1x1 conv, one fmaf chain per output channel over the input channels in order
    from the bias: sum_k |s_k| over the float64 partial sums s_k (each fmaf rounds once; Higham, eq. 3.7's running form)."""
    out = np.empty((g.shape[0], W.shape[0]))
    for t0 in range(0, g.shape[0], chunk):
        p = np.cumsum(g[t0:t0 + chunk, None, :] * W[None, :, :], axis=2) + bias[None, :, None]
        out[t0:t0 + chunk] = np.abs(p).sum(2)
    return out


def dds_layer(x, ex, L, w, dil, k):
    """One layer on one utterance: x [L, C] float64 input (exact fp32 values plus error ex).  w: dict of the layer's float64
    weights sep_w [C, k], sep_b, ln1g, ln1b, pw_w [C_out, C_in], pw_b, ln2g, ln2b.  Returns (y, bound)."""
    C = x.shape[1]
    half = (k - 1) // 2
    v = np.broadcast_to(w["sep_b"], (L, C)).copy()
    av = np.abs(v).copy()
    ev = np.zeros((L, C))
    for j in range(k):
        s = (j - half) * dil
        t0, t1 = max(0, -s), min(L, L - s)
        if t1 > t0:
            v[t0:t1] += w["sep_w"][:, j] * x[t0 + s:t1 + s]
            av[t0:t1] += np.abs(w["sep_w"][:, j] * x[t0 + s:t1 + s])
            ev[t0:t1] += np.abs(w["sep_w"][:, j]) * ex[t0 + s:t1 + s]
    ev += (k + 1) * U * av
    n1, en1 = _ln(v, ev, w["ln1g"], w["ln1b"])
    g1, eg1 = _gelu_err(n1, en1)
    W = w["pw_w"]
    v2 = g1 @ W.T + w["pw_b"]
    ev2 = eg1 @ np.abs(W).T + U * _running(g1, W, w["pw_b"])
    n2, en2 = _ln(v2, ev2, w["ln2g"], w["ln2b"])
    g2, eg2 = _gelu_err(n2, en2)
    y = x + g2
    return y, ex + eg2 + U * np.abs(y)


def dds_weights(sd, prefix, i):
    """Float64 weights of layer i of the DDSConv `prefix` ("dp.convs" or "dp.flows.<i>.convs") of a reference state dict."""
    f = lambda n: np.asarray(sd[n], np.float64)
    return dict(sep_w=f("%s.convs_sep.%d.weight" % (prefix, i))[:, 0, :], sep_b=f("%s.convs_sep.%d.bias" % (prefix, i)),
                ln1g=f("%s.norms_1.%d.gamma" % (prefix, i)), ln1b=f("%s.norms_1.%d.beta" % (prefix, i)),
                pw_w=f("%s.convs_1x1.%d.weight" % (prefix, i))[:, :, 0], pw_b=f("%s.convs_1x1.%d.bias" % (prefix, i)),
                ln2g=f("%s.norms_2.%d.gamma" % (prefix, i)), ln2b=f("%s.norms_2.%d.beta" % (prefix, i)))


def dds_layers(sd, prefix, k, lens, ys=None, x=None, x0=None, cond=None, pre=None):
    """Every layer (dilations 1, k, k^2) of every utterance, each on the kernel's own input: layer 0 on x [rows, C] (plain
    stack) or on the ConvFlow front h = pre_w * x0 + pre_b + cond (x0 [rows], cond [rows, C], pre = (pre_w [C], pre_b [C]):
    an fmaf and an add), layer i > 0 on ys[i - 1], the kernel's output of layer i - 1 ([3, rows, C]; None: the float64
    chain rounded to fp32 stands in for it).  Returns [layer][utterance] (rows, y [L, C], bound [L, C])."""
    offs = offsets(lens)
    ws = [dds_weights(sd, prefix, i) for i in range(3)]
    out = [[], [], []]
    for b, L in enumerate(lens):
        r = np.arange(offs[b], offs[b] + L)
        if x0 is not None:
            pw, pb = (np.asarray(a, np.float64) for a in pre)
            x0b = np.asarray(x0, np.float64)[r][:, None]
            h = pw * x0b + pb + np.asarray(cond, np.float64)[r]
            eh = U * (np.abs(pw * x0b + pb) + np.abs(h))
        else:
            h = np.asarray(x, np.float64)[r]
            eh = np.zeros_like(h)
        dil = 1
        for i in range(3):
            if i > 0:
                h = np.asarray(ys[i - 1], np.float64)[r] if ys is not None else out[i - 1][b][1].astype(np.float32).astype(np.float64)
                eh = np.zeros_like(h)
            y, ey = dds_layer(h, eh, L, ws[i], dil, k)
            out[i].append((r, y, ey))
            dil *= k
    return out


def dds_chain(sd, prefix, k, lens, x=None, x0=None, cond=None, pre=None):
    """The float64 stack of three layers, with no fp32 rounding between them: [utterance] y [L, C]."""
    offs = offsets(lens)
    ws = [dds_weights(sd, prefix, i) for i in range(3)]
    res = []
    for b, L in enumerate(lens):
        r = slice(offs[b], offs[b] + L)
        if x0 is not None:
            h = np.asarray(pre[0], np.float64) * np.asarray(x0, np.float64)[r][:, None] + np.asarray(pre[1], np.float64) + \
                np.asarray(cond, np.float64)[r]
        else:
            h = np.asarray(x, np.float64)[r]
        dil = 1
        for i in range(3):
            h, _ = dds_layer(h, np.zeros_like(h), L, ws[i], dil, k)
            dil *= k
        res.append(h)
    return res


# the DDS cases of the GPU test (test_gpu_durations.py), also checked on the CPU (test_duration_ref.py)
DDS_VARIANTS = {"c32": 32, "c96": 96, "c160": 160, "c192": 192, "c256": 256, "c96s": 96}
DDS_SEP_SCALE = {"c96s": 1e-3}       # depthwise weights and biases scaled: LayerNorm 1 sees a variance far below its epsilon
DDS_LENS = [[1], [3], [4], [5], [7], [8], [9], [300]]
DDS_RAGGED = [[9, 3, 27, 5], [1, 4, 2, 300, 8, 7]]       # dilation-9 halos past an utterance's end


def dds_cases():
    """(variant, stack, lens, kind, seed) of every DDS case."""
    cases = []
    for v in ("c32", "c96", "c160", "c192", "c256"):
        for lens in DDS_LENS + DDS_RAGGED:
            cases.append((v, "dp.convs", lens, "plain", len(lens)))
    for v in ("c32", "c160", "c256"):
        for flow in (3, 5, 7):
            for lens in [[1], [5], [300]] + DDS_RAGGED:
                cases.append((v, "dp.flows.%d.convs" % flow, lens, "plain", flow))
    for v in ("c96", "c160", "c192", "c256", "c96s"):
        for stack in ("dp.convs", "dp.flows.3.convs"):
            for kind in ("offset", "flat"):
                cases.append((v, stack, DDS_RAGGED[0], kind, 11))
    return cases


# ---------------------------------------------------------------------------------------------------- spline inverse
# op kinds of the spline tape and their relative errors: kernel vs exact (float64 reference), and kernel vs the fp32 oracle
# (rq_spline_inverse in torch fp32: the same ops in the same order, but not bit for bit: a CPU run differs from a NumPy float32
# emulation of the kernel's op sequence by 3 ulps on a 2-bin row, so every op may round differently in the two, 2u; beyond
# that what differs is torch's exp / log1p (SLEEF and glibc:
# <= 1 and <= 2 ulp), its softmax (a vectorised sum in another order, and a multiply by the reciprocal of the sum) and the
# division by sqrt(filter_channels), which torch may also take as a multiply by the reciprocal; and torch.cumsum, which on the
# CPU accumulates float32 in double and rounds each partial sum once, where the kernel rounds a running fp32 sum)
SPLINE_ERR_EXACT = {"op": U, "const": U, "exp": EXPF, "log1p": LOG1PF, "sum": U, "norm": U, "scale": U, "cum": U}
SPLINE_ERR_ORACLE = {"op": 2 * U, "const": 0.0, "exp": EXPF + 1 * ULP, "log1p": LOG1PF + 2 * ULP, "sum": 2 * U, "norm": 2 * ULP,
                     "scale": ULP, "cum": 2 * U}
# kernel vs spline_emulate (the kernel's op sequence in NumPy float32, exp / log1p correctly rounded through float64): only
# expf and log1pf differ (their documented error plus the emulation's half ulp); every other op is the same IEEE op
SPLINE_ERR_EMU = {"op": 0.0, "const": 0.0, "exp": EXPF + ULP / 2, "log1p": LOG1PF + ULP / 2, "sum": 0.0, "norm": 0.0, "scale": 0.0,
                  "cum": 0.0}
# ... and once an expf / log1pf difference reaches a row, any later op's rounding may flip by an ulp: there every op gets 2u
SPLINE_ERR_FLIP = {"op": 2 * U, "const": 0.0, "exp": EXPF + ULP / 2, "log1p": LOG1PF + ULP / 2, "sum": 2 * U, "norm": 2 * U,
                   "scale": 2 * U, "cum": 2 * U}
_H = 1e-30                        # complex step


class _Tape:
    """Counts the ops of one evaluation; the op numbered `active` gets the relative perturbation i * _H on its result."""

    def __init__(self, active=-1):
        self.active, self.kinds, self.exact = active, [], []

    def __call__(self, v, kind="op", exact=False):
        """exact: where (per row) the op's result is exact in every implementation (exp(0) = 1)."""
        k = len(self.kinds)
        self.kinds.append(kind)
        self.exact.append(exact)
        return v * (1 + 1j * _H) if k == self.active else v


def _spline(h, x, nb, bound, den, t, force_bin=None, last_eps=1e-6, tail_lt=False):
    """The kernel's op sequence in complex float64 over rows: h [N, >= 3nb-1], x [N].  Returns (y, bin, inside, knots ch)."""
    N = x.shape[0]
    h = h.astype(np.complex128)
    coef = t(1.0 - 1e-3 * nb + 0j, "const")
    mw = t(1e-3 + 0j, "const")
    cums = []
    for p in range(2):
        u = [t(h[:, p * nb + i] / den, "scale") for i in range(nb)]
        mx = np.max(np.stack([v.real for v in u]), axis=0)
        z = [t(v - mx) for v in u]
        e = [t(np.exp(v), "exp", exact=(v.real == 0)) for v in z]
        s = e[0]
        for v in e[1:]:
            s = t(s + v, "sum")
        run = np.zeros(N, np.complex128)
        cum = [np.full(N, -bound, np.complex128)]
        for i in range(nb):
            wi = t(mw + t(coef * t(e[i] / s, "norm")))
            run = t(run + wi, "cum")
            cum.append(t(t(2 * bound * run) - bound))
        cum[nb] = np.full(N, bound, np.complex128)
        cums.append(np.stack(cum, 1))
    cw, ch = cums
    cst = t(np.log(np.exp(1 - 1e-3) - 1) + 0j, "const")
    dv = []
    for i in range(nb + 1):
        ud = cst if i in (0, nb) else h[:, 2 * nb + i - 1]
        ud = np.broadcast_to(ud, (N,))
        sp = np.where(ud.real > 20, ud, t(np.log1p(t(np.exp(ud), "exp")), "log1p"))
        dv.append(t(mw + sp))
    dv = np.stack(dv, 1)
    if force_bin is None:
        loc = ch.real.copy()
        loc[:, nb] = loc[:, nb] + last_eps
        b = np.clip((x[:, None] >= loc).sum(1) - 1, 0, nb - 1)
    else:
        b = np.asarray(force_bin)
    g = lambda a, o=0: np.take_along_axis(a, (b + o)[:, None], 1)[:, 0]
    in_cw, in_w = g(cw), t(g(cw, 1) - g(cw))
    in_ch, in_h = g(ch), t(g(ch, 1) - g(ch))
    delta = t(in_h / in_w)
    d0, d1 = g(dv), g(dv, 1)
    tsum = t(t(d0 + d1) - t(2 * delta))
    dx = t(x - in_ch)
    a = t(t(dx * tsum) + t(in_h * t(delta - d0)))
    bq = t(t(in_h * d0) - t(dx * tsum))
    c = t(-delta * dx)
    disc = t(t(bq * bq) - t(t(4 * a) * c))
    root = t(t(2 * c) / t(-bq - t(np.sqrt(disc))))
    y = t(t(root * in_w) + in_cw)
    inside = (x >= -bound) & ((x < bound) if tail_lt else (x <= bound))
    return y, b, inside, ch


def spline_inverse(h, x, nb, bound, den, err=SPLINE_ERR_EXACT, force_bin=None, **mut):
    """Float64 spline inverse of every row and its bound: h [N, >= 3nb-1] raw parameter rows (widths and heights are divided
    by den = sqrt(filter_channels)), x [N] float32 values.  Rows outside [-bound, bound] pass through (bound 0).
    Returns (y, bound, bin, knots ch [N, nb+1] with their bound)."""
    h = np.asarray(h, np.float64)
    x = np.asarray(x, np.float32).astype(np.float64)
    y, b, inside, ch = _spline(h, x, nb, bound, den, _Tape(), force_bin, **mut)
    kinds = _Tape()
    _spline(h, x, nb, bound, den, kinds, b)
    bnd = np.zeros(x.shape)
    kb = np.zeros(ch.shape)
    for k, kind in enumerate(kinds.kinds):
        e = np.where(kinds.exact[k], 0.0, err[kind])
        if not np.any(e):
            continue
        yk, _, _, chk = _spline(h, x, nb, bound, den, _Tape(k), b)
        bnd += np.abs(yk.imag / _H) * e
        kb += np.abs(chk.imag / _H) * np.reshape(e, (-1, 1) if np.ndim(e) else ())
    y = np.where(inside, y.real, x)
    return y, np.where(inside, 2 * bnd, 0.0), b, (ch.real, 2 * kb)


def spline_emulate(h, x, nb, bound, den):
    """spline_inverse_kernel's op sequence in NumPy float32 (no FMA contraction), expf / log1pf correctly rounded from
    float64.  h [N, >= 3nb-1], x [N] float32.  Returns y [N] float32."""
    f = np.float32
    h = np.asarray(h, f)
    x = np.asarray(x, f)
    N = x.shape[0]
    bound, den = f(bound), f(den)
    ex = lambda v: np.exp(v.astype(np.float64)).astype(f)
    coef = f(1.0 - 1e-3 * nb)
    cums = []
    for p in range(2):
        u = (h[:, p * nb:(p + 1) * nb] / den).astype(f)
        mx = u.max(1)
        e = [ex((u[:, i] - mx).astype(f)) for i in range(nb)]
        s = np.zeros(N, f)
        for v in e:
            s = (s + v).astype(f)
        run = np.zeros(N, f)
        cum = [np.full(N, -bound, f)]
        for i in range(nb):
            wi = (f(1e-3) + (coef * (e[i] / s).astype(f)).astype(f)).astype(f)
            run = (run + wi).astype(f)
            cum.append(((f(2) * bound * run).astype(f) + (-bound)).astype(f))
        cum[nb] = np.full(N, bound, f)
        cums.append(np.stack(cum, 1))
    cw, ch = cums
    cst = f(0.5397424172369522)
    dv = []
    for i in range(nb + 1):
        ud = np.full(N, cst, f) if i in (0, nb) else h[:, 2 * nb + i - 1]
        sp = np.where(ud > 20, ud, np.log1p(ex(ud).astype(np.float64)).astype(f))
        dv.append((f(1e-3) + sp).astype(f))
    dv = np.stack(dv, 1)
    loc = ch.copy()
    loc[:, nb] = (loc[:, nb] + f(1e-6)).astype(f)
    b = np.clip((x[:, None] >= loc).sum(1) - 1, 0, nb - 1)
    g = lambda a, o=0: np.take_along_axis(a, (b + o)[:, None], 1)[:, 0]
    in_cw, in_w = g(cw), (g(cw, 1) - g(cw)).astype(f)
    in_ch, in_h = g(ch), (g(ch, 1) - g(ch)).astype(f)
    delta = (in_h / in_w).astype(f)
    d0, d1 = g(dv), g(dv, 1)
    tsum = ((d0 + d1).astype(f) - (f(2) * delta).astype(f)).astype(f)
    dx = (x - in_ch).astype(f)
    a = ((dx * tsum).astype(f) + (in_h * (delta - d0).astype(f)).astype(f)).astype(f)
    bq = ((in_h * d0).astype(f) - (dx * tsum).astype(f)).astype(f)
    c = (-delta * dx).astype(f)
    disc = ((bq * bq).astype(f) - ((f(4) * a).astype(f) * c).astype(f)).astype(f)
    with np.errstate(invalid="ignore", divide="ignore"):
        root = ((f(2) * c).astype(f) / (-bq - np.sqrt(disc)).astype(f)).astype(f)
    y = ((root * in_w).astype(f) + in_cw).astype(f)
    return np.where((x >= -bound) & (x <= bound), y, x)


def emulation_exact(h, x, nb, bound, den, b=None):
    """Rows on which no expf / log1pf result can reach the output: equal widths and equal heights (every exp is exp(0) = 1,
    exact everywhere), x inside an interior bin, and that bin's two derivative parameters past the softplus threshold."""
    h = np.asarray(h, np.float32)
    if b is None:
        b = spline_inverse(h, x, nb, bound, den)[2]
    eq = np.all(h[:, :nb] == h[:, :1], 1) & np.all(h[:, nb:2 * nb] == h[:, nb:nb + 1], 1)
    inner = (b >= 1) & (b <= nb - 2)
    bi = np.clip(b, 1, max(nb - 2, 1))
    d0 = np.take_along_axis(h, (2 * nb + bi - 1)[:, None], 1)[:, 0] if nb >= 3 else np.zeros(len(b))
    d1 = np.take_along_axis(h, (2 * nb + bi)[:, None], 1)[:, 0] if nb >= 3 else np.zeros(len(b))
    xv = np.asarray(x, np.float64)
    return eq & inner & (d0 > 20) & (d1 > 20) & (np.abs(xv) < bound)


def emulation_check(h, x, out, nb, bound, den):
    """|out - spline_emulate| / its budget, per row.  Where no expf / log1pf result can reach the output (emulation_exact)
    the budget is 0: out must equal the emulation bit for bit.
    Elsewhere the budget is SPLINE_ERR_FLIP's, and rows whose x lies within the knots' budget of an interior knot (where
    the bin may differ) get 0."""
    emu = spline_emulate(h, x, nb, bound, den).astype(np.float64)
    _, bnd, b, (ch, kb) = spline_inverse(h, x, nb, bound, den, err=SPLINE_ERR_FLIP)
    bnd = np.where(emulation_exact(h, x, nb, bound, den, b), 0.0, bnd)
    xv = np.asarray(x, np.float64)
    near = np.any((np.abs(ch - xv[:, None]) <= kb)[:, 1:-1], 1)       # (the end knots are +-bound exactly in both)
    err = np.abs(np.asarray(out, np.float64) - emu)
    r = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1.0), np.where(err == 0, 0.0, np.inf))
    return np.where(near, 0.0, np.where(np.isnan(out), np.inf, r))


def spline_check(h, x, out, nb, bound, den, err=SPLINE_ERR_EXACT):
    """Largest |out - ref| / bound over the rows, accepting at a knot (x within the knot's bound of it) the bin on either side.
    NaN or a row whose error exceeds every acceptable bin's bound gives inf."""
    y, bnd, b, (ch, kb) = spline_inverse(h, x, nb, bound, den, err)
    out = np.asarray(out, np.float64)
    xv = np.asarray(x, np.float32).astype(np.float64)
    ratio = _ratio(out, y, bnd, xv)
    for o in (-1, 1):
        alt = np.clip(b + o, 0, nb - 1)
        knot = np.take_along_axis(ch, np.maximum(b, alt)[:, None], 1)[:, 0]
        kbd = np.take_along_axis(kb, np.maximum(b, alt)[:, None], 1)[:, 0]
        near = (alt != b) & (np.abs(xv - knot) <= kbd) & (bnd > 0)
        if near.any():
            ya, ba, _, _ = spline_inverse(h[near], x[near], nb, bound, den, err, force_bin=alt[near])
            ratio[near] = np.minimum(ratio[near], _ratio(out[near], ya, ba, xv[near]))
    return ratio


def _ratio(out, ref, bnd, x):
    err = np.abs(out - ref)
    r = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1.0), np.where(err == 0, 0.0, np.inf))
    return np.where(np.isnan(out), np.inf, r)


def spline_rows(nb, bound, den, seed=0):
    """Edge rows of the spline (raw parameter rows [N, 3nb-1] and x [N] float32), shared by the CPU and GPU tests:
    x at +-bound, one fp32 ulp inside and outside, far outside; x on interior knots and on the last knot; derivative
    parameters below, at and above the softplus threshold 20 and strongly negative; nearly one-hot widths and heights
    (bins of minimum width); and plain random rows."""
    rng = np.random.default_rng(seed)
    P = 3 * nb - 1
    rows, xs = [], []

    def add(hr, xv):
        rows.append(np.asarray(hr, np.float32))
        xs.append(np.float32(xv))
    f = np.float32(bound)
    for xv in (f, -f, np.nextafter(f, np.float32(0)), np.nextafter(-f, np.float32(0)), np.nextafter(f, np.float32(np.inf)),
               np.nextafter(-f, np.float32(-np.inf)), 4 * f, -1e6 * f):
        add(rng.standard_normal(P), xv)
    for d in (19.99, 20.0, 20.01, 25.0, -20.0, -60.0):
        for xv in rng.uniform(-bound, bound, 3):
            hr = rng.standard_normal(P)
            hr[2 * nb:] = d
            add(hr, xv)
    for hot in range(2):                                          # nearly one-hot widths, then heights
        for j in range(min(nb, 4)):
            hr = rng.standard_normal(P)
            hr[hot * nb:(hot + 1) * nb] = -30.0 * den
            hr[hot * nb + j] = 30.0 * den
            for xv in rng.uniform(-bound, bound, 3):
                add(hr, xv)
    for _ in range(16):                                           # at exactly +-bound with random parameters
        add(rng.standard_normal(P) * 1.5, f)
        add(rng.standard_normal(P) * 1.5, -f)
    for _ in range(24):                                           # equal widths and heights (every exp is exp(0) = 1) and
        hr = np.full(P, rng.standard_normal())                    # derivatives past the softplus threshold: no expf / log1pf
        hr[nb:2 * nb] = rng.standard_normal()                     # reaches an interior bin's output
        hr[2 * nb:] = rng.uniform(20.5, 40.0, nb - 1)
        add(hr, rng.uniform(-bound, bound))
    for _ in range(24):                                           # on the knots (fp32 knot values of a first evaluation)
        add(rng.standard_normal(P) * 2, 0.0)
    for _ in range(64):
        add(rng.standard_normal(P) * 1.5, rng.uniform(-bound * 1.1, bound * 1.1))
    h, x = np.stack(rows), np.asarray(xs, np.float32)
    k0 = len(rows) - 64 - 24
    _, _, _, (ch, _) = spline_inverse(h[k0:k0 + 24], x[k0:k0 + 24], nb, bound, den)
    for i in range(24):
        x[k0 + i] = np.float32(ch[i, 1 + i % nb] if i % 3 else ch[i, nb])        # interior knots and the last knot
    return h, x


def oracle_points(h, x, nb, bound, den):
    """Rows away from ill-conditioned points, where the fp32 oracle comparison is made: inside the domain, not within 1e-3 of
    a knot, and with widths and heights not at their minimum."""
    _, _, _, (ch, _) = spline_inverse(h, x, nb, bound, den)
    xv = np.asarray(x, np.float64)
    far = np.min(np.abs(ch - xv[:, None]), 1) > 1e-3
    return far & (np.abs(xv) < bound)


# ---------------------------------------------------------------------------------------------------- VITS durations
def vits_w(z, m, logs, length_scale):
    """Float64 w = exp((z - m) * exp(-logs)) * length_scale and its bound (relative error of the kernel's two expf and three
    roundings, and fp32 underflow: where exp(logw) is below fp32's range a token may get 0 frames; NaN z gives NaN)."""
    z = np.asarray(z, np.float32).astype(np.float64)
    length_scale = float(np.float32(length_scale))               # the kernel's scalars are fp32: the reference takes their values
    logw = (z - m) * np.exp(-logs)
    w = np.exp(logw) * length_scale
    # (+ the absolute error of a result in fp32's subnormal range: expf below 2^-126 rounds to a multiple of 2^-149)
    return w, np.abs(w) * (6 * U * np.abs(logw) + EXPF + 3 * U) + 2.0 ** -148 * abs(length_scale)


def ceil_ok(wc, w, bw):
    """True per token when the kernel's ceil wc is the float64 ceil clamped to [0, 1e6] (NaN: 0), or a neighbour of it where
    w lies within bw of an integer."""
    wc = np.asarray(wc, np.int64)
    nan = np.isnan(w)
    wv = np.where(nan, 0.0, w)
    ref = np.clip(np.ceil(wv), 0, CEIL_CAP)
    lo = np.clip(np.ceil(wv - bw), 0, CEIL_CAP)
    hi = np.clip(np.ceil(wv + bw), 0, CEIL_CAP)
    return np.where(nan, wc == 0, (wc == ref) | ((wc >= lo) & (wc <= hi) & (np.abs(wc - ref) <= 1)))


def vits_layout(wceil, lens, cap=0):
    """What follows exactly from the kernel's ceil durations wceil [rows] (packed by lens): cum [rows] (inclusive scan),
    ylen_real = max(sum, 1) per utterance, ylen (capped at cap > 0), the device offsets (capped layout) and the offsets the
    host reads (uncapped).  Sums past INT32_MAX are returned as they are (Python ints)."""
    offs = offsets(lens)
    cum = np.zeros(len(wceil), np.int64)
    real = []
    for b, n in enumerate(lens):
        s = np.cumsum(np.asarray(wceil[offs[b]:offs[b] + n], np.int64))
        cum[offs[b]:offs[b] + n] = s
        real.append(max(int(s[-1]), 1))
    capped = [min(v, cap) if cap > 0 else v for v in real]
    return cum, real, capped, offsets(capped), offsets(real)


def frame_tokens(cum_b, n_frames):
    """Token of every frame of one utterance: #{i : cum_i <= j} (== T when the durations sum to less than the frames)."""
    return np.searchsorted(np.asarray(cum_b, np.int64), np.arange(n_frames), side="right")


def prior(stats_b, tok, eps_b, noise_scale, I):
    """z_p [frames, I] = m + eps * exp(logs) * noise_scale of each frame's token (m = logs = 0 for token index T) and its bound
    (expf, two products and the sum)."""
    st = np.asarray(stats_b, np.float64)
    noise_scale = float(np.float32(noise_scale))                 # (fp32 in the kernel, as length_scale in vits_w)
    T = st.shape[0]
    ok = tok < T
    row = st[np.where(ok, tok, 0)]
    m = np.where(ok[:, None], row[:, :I], 0.0)
    ls = np.where(ok[:, None], row[:, I:], 0.0)
    n = np.asarray(eps_b, np.float64).T * np.exp(ls) * noise_scale
    v = m + n
    return v, np.abs(n) * (EXPF + 2 * U) + U * np.abs(v)


# ---------------------------------------------------------------------------------------------------- StableTTS durations
def stt_pre_round(mu_dp, pause, length_scale):
    """Float64 value before rounding (sum of sigmoids, the pause where it is not 0, times length_scale) and its bound: (DC + 6)
    u of the sum of the sigmoids (expf, add, divide per term, the channel-order sum) plus the product's rounding.  Pause
    tokens are exact in fp32 (one product), bound 0 with the fp32 value."""
    m = np.asarray(mu_dp, np.float32).astype(np.float64)
    DC = m.shape[1]
    s = (1.0 / (1.0 + np.exp(-m))).sum(1)
    p = np.asarray(pause, np.float32)
    ls = np.float32(length_scale)
    a = s * float(ls)
    bnd = ((DC + 6) * U * s + U * s) * float(ls) + U * np.abs(a)
    pv = (p * ls).astype(np.float32).astype(np.float64)
    return np.where(p != 0, pv, a), np.where(p != 0, 0.0, bnd)


def stt_rule(a, wmax):
    """Durations of the pre-rounding values a (float64): round half to even, at least 1, at most wmax."""
    return np.clip(np.rint(a), 1, wmax).astype(np.int64)


def rint_ok(dur, a, bnd, wmax):
    """The kernel's durations against the float64 pre-rounding values: equal to the rule, or to the rule at a +- bnd where a
    lies within bnd of a half-integer."""
    d = np.asarray(dur, np.int64)
    return (d == stt_rule(a, wmax)) | (d == stt_rule(a - bnd, wmax)) | (d == stt_rule(a + bnd, wmax))


def stt_expand(x, mu_mel, pause, dur, lens, flens, denorm=None, frame_rows=None):
    """NumPy float32 emulation of stt_expand_kernel: frame rows packed by flens; mu, pau, prior of every frame (prior rows
    v * std + mean in two fp32 roundings when denorm = (mean, std)).  Returns (mu, pau, prior, mask of written frame rows)."""
    to, fo = offsets(lens), offsets(flens)
    n_rows = fo[-1] if frame_rows is None else frame_rows
    mu = np.zeros((n_rows, x.shape[1]), np.float32)
    pau = np.zeros(n_rows, np.float32)
    pr = np.zeros((n_rows, mu_mel.shape[1]), np.float32)
    mask = np.zeros(n_rows, bool)
    for b, n in enumerate(lens):
        d = np.asarray(dur[to[b]:to[b] + n], np.int64)
        tok = to[b] + np.repeat(np.arange(n), d)
        rows = fo[b] + np.arange(len(tok))
        mu[rows] = x[tok]
        pau[rows] = pause[tok]
        v = mu_mel[tok].astype(np.float32)
        if denorm is not None:
            v = (v * np.float32(denorm[1])).astype(np.float32) + np.float32(denorm[0])
        pr[rows] = v
        mask[rows] = True
    return mu, pau, pr, mask


def pause_fill(mel, pau, flens):
    """stt_pause_fill_kernel: every frame t > 0 of an utterance whose pau > 0 takes the utterance's own frame 0."""
    out = np.array(mel, np.float32)
    fo = offsets(flens)
    for b, n in enumerate(flens):
        r = np.arange(fo[b] + 1, fo[b] + n)
        r = r[pau[r] > 0]
        out[r] = out[fo[b]]
    return out


# ---------------------------------------------------------------------------------------------------- shared edge inputs
def dds_inputs(kind, lens, C, seed=0, tail=16):
    """Rows of a DDS case (finite garbage in the gap and tail rows): kind "plain" (N(0, 1)), "offset" (1000 + N(0, 1): a large
    common offset) or "flat" (every channel of a row nearly equal: 0.3 + 1e-4 N(0, 1)).  Returns (x [rows, C], x0 [rows],
    cond [rows, C]) float32."""
    rng = np.random.default_rng(seed)
    offs = offsets(lens)
    rows = offs[-1] + tail
    x = rng.uniform(-1e3, 1e3, (rows, C))
    x0 = rng.uniform(-1e3, 1e3, rows)
    cond = rng.uniform(-1e3, 1e3, (rows, C))
    for b, n in enumerate(lens):
        r = slice(offs[b], offs[b] + n)
        if kind == "plain":
            x[r], x0[r], cond[r] = rng.standard_normal((n, C)), rng.standard_normal(n), rng.standard_normal((n, C))
        elif kind == "offset":
            x[r] = 1000 + rng.standard_normal((n, C))
            x0[r] = 1000 + rng.standard_normal(n)
            cond[r] = 1000 + rng.standard_normal((n, C))
        else:
            x[r] = 0.3 + 1e-4 * rng.standard_normal((n, C))
            x0[r] = 0.3 + 1e-4 * rng.standard_normal(n)
            cond[r] = 0.3 + 1e-4 * rng.standard_normal((n, C))
    return x.astype(np.float32), x0.astype(np.float32), cond.astype(np.float32)


def vits_logw(kind, n, seed=0):
    """logw of a duration case: "plain" (N(0, 1)), "under" (every token below -200: exp underflows, 0 frames), "some_zero"
    (every third token below -200), "cap" (w past 1e6), "near" (w within a few ulps of an integer), "nan" (one NaN)."""
    rng = np.random.default_rng(seed)
    lw = rng.standard_normal(n)
    if kind == "under":
        lw = -200.0 - rng.uniform(0, 10, n)
    elif kind == "some_zero":
        lw[::3] = -250.0
    elif kind == "cap":
        lw[::2] = 15.0 + rng.uniform(0, 3, len(lw[::2]))
    elif kind == "near":
        lw = np.log(rng.integers(1, 20, n).astype(np.float64)) + rng.choice([-1, 1], n) * 1e-7
    elif kind == "nan":
        lw[n // 2] = np.nan
    return lw


def z_of_logw(logw, m, logs):
    """The flows' output z whose logw = (z - m) * exp(-logs) is `logw` (float32)."""
    return (np.asarray(logw) * np.exp(logs) + m).astype(np.float32)


STT_PAUSES = [0.5, 1.5, 2.5, 3.5, -1.0, -0.5, 5000.0, 4096.5, 0.0]
