"""Plain float64 restatement of one problem of a grouped dense-conv launch (csrc/conv_tc.cuh conv_tc_body,
csrc/kernels.cuh conv_kernel) and the error bound a correct kernel must meet against it.

Layout (as the engine packs utterances): utterance b starts at unit offs[b] (SEQ_GAP = 8 units between utterances),
a unit is `rmul` rows.  Logical input position p of utterance b (0 <= p < L_b = lens[b] * rmul + in_extra) is
  tensor cores   row offs[b] * rmul + b * in_extra + p of the split-bf16 input planes
  FFMA           row offs[b] * rmul + pr, pr = reflect ? (p == 0 ? 1 : p - 1) : p, of the fp32 input (ldx / xoff),
                 through lrelu(., slope) with the PRO_LRELU prologue
and positions outside [0, L_b) are zero.  Output t of utterance b goes to row offs[b]*rmul*out_mul + b*out_seq_extra
+ t*out_mul + out_add.  Epilogue in the kernels' order: a = acc + bias + cond[b] -> gate (tanh(a_2i) * sigmoid(a_2i+1)) /
ReLU / tanh -> * alpha -> + residual; output planes hold split(lrelu(out, pl_slope)).

Tolerance.  The tensor-core kernel multiplies exactly the bf16 planes it is given (a bf16 x bf16 product is exact in fp32)
and sums the products in fp32: np = 2 issues hi*hi + hi*lo + lo*hi, np = 3 the six products hh, hm, mh, hl, lh, mm.
`tc_terms` forms the float64 sum of exactly those products ("operand-exact emulation"), so what is left between it and the
GPU is fp32 accumulation alone.  Recursive summation of n terms in floating point with unit roundoff u satisfies
|fl(sum) - sum| <= gamma_(n-1) * sum|t_i|, gamma_m = m*u / (1 - m*u) (Higham, Accuracy and Stability of Numerical
Algorithms, 2nd ed., eq. 4.4), for ANY order of the additions, so the wgmma k-order, the split-K partial sums and the FFMA
kernel's thread-group reduction are all covered.  We take u = 2^-23 instead of 2^-24 because tensor-core accumulation is
not guaranteed to round to nearest (truncating alignment and normalisation give errors up to one ulp, not half), and
n = n_terms + 8 for the bias, cond and up to 8 split-K partials: bound_acc = (n_terms + 8) * 2^-23 * (sum|terms| + |bias|
+ |cond|); m*u << 1 here, so the 1/(1 - m*u) factor is below 1.002 and absorbed in the slack of u.  The activations are
1-Lipschitz (tanh, ReLU; the gate is tanh(a)*sigmoid(s) with |d/da| <= 1, |d/ds| <= 1/4) and tanhf / expf / the division
add a few fp32 ulps of a value <= 1 (16 * 2^-24 taken); alpha scales the bound; the alpha product and the residual sum
each add one rounding (2^-24 relative) of their result.
The FFMA kernel runs fp32 FMAs on the fp32 operands: the same bound with n_terms = Cin * k against the exact float64
conv of the fp32 operands.

Splits.  `split_bf16` / `split_bf16_3` restate the device functions (kernels.cuh): round half away from zero by adding
0x8000 to the bit pattern and masking (the host packer, weights.conv_tc_planes, rounds to nearest even instead).
x - hi is exact in fp32, so hi + lo = x to 2^-16 relative (two 8-bit roundings) and hi + mid + lo = x exactly (24 bits).
For np = 2 the emulated product (ah + al)(wh + wl) - al*wl therefore differs from x*w by at most ~3 * 2^-16 |x w|; for
np = 3 the dropped products mid*lo, lo*mid, lo*lo are below 2 * 2^-24 |x w|, i.e. under fp32 accumulation -- the design
claims of conv_tc.cuh (~1e-5) and of mode 3 ("products exact to the last fp32 bit") that test_conv_ref.py checks."""
import numpy as np

SEQ_GAP = 8
U23 = 2.0 ** -23
U24 = 2.0 ** -24
FN_ERR = 16 * U24          # tanhf / expf / division on values <= 1
EPI_RELU, EPI_GATE, EPI_TANH = 1, 2, 4
# product pairs (activation plane, weight plane) the tensor-core kernel issues; planes are (hi, lo) / (hi, mid, lo)
PAIRS = {2: [(0, 0), (0, 1), (1, 0)], 3: [(0, 0), (0, 1), (1, 0), (0, 2), (2, 0), (1, 1)]}


def offsets(lens):
    """Packed unit offsets of the utterances (engine: SEQ_GAP units between consecutive utterances); offs[B] = total."""
    o = [0]
    for b, n in enumerate(lens):
        o.append(o[-1] + int(n) + (SEQ_GAP if b + 1 < len(lens) else 0))
    return o


# ---------------------------------------------------------------------------------------------------- device splits
def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _f(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def split_bf16(x):
    """Device split_bf16: fp32 -> (hi, lo) bf16 bit planes (uint16), hi + lo == x to ~2^-16 relative."""
    x = np.asarray(x, np.float32)
    h = (_bits(x) + np.uint32(0x8000)) & np.uint32(0xFFFF0000)
    r = (x - _f(h)).astype(np.float32)
    lo = (_bits(r) + np.uint32(0x8000)) >> np.uint32(16)
    return (h >> np.uint32(16)).astype(np.uint16), lo.astype(np.uint16)


def split_bf16_3(x):
    """Device split_bf16_3: fp32 -> (hi, mid, lo), hi + mid + lo == x exactly."""
    x = np.asarray(x, np.float32)
    h = (_bits(x) + np.uint32(0x8000)) & np.uint32(0xFFFF0000)
    r1 = (x - _f(h)).astype(np.float32)
    m = (_bits(r1) + np.uint32(0x8000)) & np.uint32(0xFFFF0000)
    r2 = (r1 - _f(m)).astype(np.float32)
    lo = (_bits(r2) + np.uint32(0x8000)) >> np.uint32(16)
    return (h >> np.uint32(16)).astype(np.uint16), (m >> np.uint32(16)).astype(np.uint16), lo.astype(np.uint16)


def split_planes(x, n):
    return np.stack(split_bf16(x) if n == 2 else split_bf16_3(x))


def bf16_value(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << np.uint32(16)).view(np.float32).astype(np.float64)


def lrelu32(v, slope):
    v = np.asarray(v, np.float32)
    return np.where(v > 0, v, (v * np.float32(slope)).astype(np.float32)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- the conv itself
def conv_taps(X, W, dil, pad, shift=None):
    """out[t] = sum_j X[t + j*dil - pad] @ W[:, :, j].T for t < len(X), X zero outside [0, len(X)).  X [L, Ci], W [Co, Ci, k]
    (float64).  shift = (j, s) reads tap j at row offset s more (corruption studies only)."""
    L = X.shape[0]
    out = np.zeros((L, W.shape[0]))
    for j in range(W.shape[2]):
        d = j * dil - pad + (shift[1] if shift is not None and shift[0] == j else 0)
        t0, t1 = max(0, -d), min(L, L - d)
        if t1 > t0:
            out[t0:t1] += X[t0 + d:t1 + d] @ W[:, :, j].T
    return out


def tc_inputs(planes, lens, rmul, in_extra):
    """Per-utterance float64 views [np][L_b, Cin] of the tensor-core input planes (uint16 [np][rows][Cin])."""
    offs = offsets(lens)
    v = bf16_value(planes)
    out = []
    for b, n in enumerate(lens):
        r0 = offs[b] * rmul + b * in_extra
        out.append(v[:, r0:r0 + n * rmul + in_extra])
    return out


def ffma_inputs(x, lens, rmul, q):
    """Per-utterance float64 [L_b, Cin] fp32 operands of the FFMA conv (row map, reflect, prologue)."""
    offs = offsets(lens)
    x = np.asarray(x, np.float32).reshape(-1)
    out = []
    for b, n in enumerate(lens):
        L = n * rmul + q.get("in_extra", 0)
        p = np.arange(L)
        pr = np.where(p == 0, 1, p - 1) if q.get("reflect", 0) else p
        rows = offs[b] * rmul + pr
        idx = rows[:, None] * q["ldx"] + q.get("xoff", 0) + np.arange(q["Cin"])[None, :]
        v = x[idx]
        if q.get("pro", 0):
            v = lrelu32(v, q["slope"])
        out.append(v.astype(np.float64))
    return out


def tc_terms(Xp, Wp, n_planes, dil, pad, drop_pair=None, shift=None):
    """Operand-exact emulation: the float64 sum of exactly the products the tensor-core kernel issues, and the sum of their
    magnitudes.  Xp [np][L, Ci] activation planes (float64 values), Wp [np][Co, Ci, k] weight planes."""
    s = a = 0.0
    for ia, iw in PAIRS[n_planes]:
        if (ia, iw) == drop_pair:
            continue
        s = s + conv_taps(Xp[ia], Wp[iw], dil, pad, shift)
        a = a + conv_taps(np.abs(Xp[ia]), np.abs(Wp[iw]), dil, pad)
    return s, a


def reference(kind, q, w, bias, lens, rmul, inputs, n_planes=2, wplanes=None, cond=None, res_buf=None, exact=False,
              corrupt=None):
    """Float64 reference of one problem for every utterance.  Returns a list of (rows [L], cols [ncol], out [L, ncol],
    bound [L, ncol]): output rows / columns (relative to yoff) and the value a correct kernel is within `bound` of.
      kind      "tc" or "ffma"
      inputs    tc: per-utterance planes from tc_inputs; ffma: per-utterance operands from ffma_inputs
      wplanes   tc: float64 [np][Co, Ci, k] weight planes (bf16 values)
      exact     tc: conv of the fp32 operands (planes summed) instead of the operand-exact emulation
      corrupt   dict of deliberate errors for the rejection studies: drop_pair, shift, drop_chunk, halo_from_prev,
                cond_prev, gate_swap"""
    corrupt = corrupt or {}
    k, dil, pad = q["k"], q.get("dil", 1), q.get("pad", 0)
    Co, Ci = q["Cout"], q["Cin"]
    offs = offsets(lens)
    out_mul, out_add = q.get("out_mul", 1), q.get("out_add", 0)
    epi, alpha = q.get("epi", 0), float(np.float32(q.get("alpha", 1.0)))
    gate = bool(epi & EPI_GATE)
    ncol = Co // 2 if gate else Co
    bias64 = np.asarray(bias, np.float64)[:Co]
    results = []
    for b in range(len(lens)):
        X = inputs[b]
        if "halo_from_prev" in corrupt and b > 0 and pad > 0:
            prev = inputs[b - 1][..., -pad:, :]                          # the left halo reads the previous utterance's rows
            fill = np.zeros(prev.shape[:-2] + (pad - prev.shape[-2], prev.shape[-1]))
            X = np.concatenate([fill, prev, X], axis=-2)
            trim = pad
        else:
            trim = 0
        if "drop_chunk" in corrupt:
            X = X.copy()
            X[..., Ci - 64:] = 0.0
        shift = corrupt.get("shift")
        if kind == "tc":
            if exact:
                xs = X.sum(axis=0)
                ws = wplanes.sum(axis=0)
                acc = conv_taps(xs, ws, dil, pad, shift)
                asum = conv_taps(np.abs(xs), np.abs(ws), dil, pad)
                n_terms = Ci * k
            else:
                acc, asum = tc_terms(X, wplanes, n_planes, dil, pad, corrupt.get("drop_pair"), shift)
                n_terms = len(PAIRS[n_planes]) * Ci * k
        else:
            W = np.asarray(w, np.float64)
            acc = conv_taps(X, W, dil, pad, shift)
            asum = conv_taps(np.abs(X), np.abs(W), dil, pad)
            n_terms = Ci * k
        if trim:
            acc, asum = acc[trim:], asum[trim:]
        L = acc.shape[0]
        bc = np.broadcast_to(bias64, (L, Co)).copy()
        if cond is not None:
            cb = b - 1 if ("cond_prev" in corrupt and b > 0) else b
            bc = bc + np.asarray(cond, np.float64)[cb, :Co]
            bc_abs = np.abs(bias64) + np.abs(np.asarray(cond, np.float64)[b, :Co])
        else:
            bc_abs = np.abs(bias64)
        a = acc + bc
        da = (n_terms + 8) * U23 * (asum + bc_abs)
        if gate:
            ta, sa = a[:, 0::2], a[:, 1::2]
            if "gate_swap" in corrupt:
                ta, sa = sa, ta
            v = np.tanh(ta) / (1.0 + np.exp(-sa))
            dv = da[:, 0::2] + 0.25 * da[:, 1::2] + FN_ERR
        else:
            v, dv = a, da
        if epi & EPI_RELU:
            v = np.maximum(v, 0.0)
        if epi & EPI_TANH:
            v, dv = np.tanh(v), dv + FN_ERR
        v = v * alpha
        dv = dv * abs(alpha) + U24 * np.abs(v)
        rows = offs[b] * rmul * out_mul + b * q.get("out_seq_extra", 0) + np.arange(L) * out_mul + out_add
        if q.get("res", 0):
            r = np.asarray(res_buf, np.float32).reshape(-1)
            ridx = rows[:, None] * q["ldr"] + q.get("roff", 0) + np.arange(ncol)[None, :]
            rv = r[ridx].astype(np.float64)
            v = v + rv
            dv = dv + U24 * (np.abs(v) + np.abs(rv))
        results.append((rows, np.arange(ncol), v, dv))
    return results


def within(out, ref, bound):
    """True when every |out - ref| <= bound (NaN fails)."""
    err = np.abs(np.asarray(out, np.float64) - ref)
    return bool(np.all(err <= bound))


def scatter(results, n, ld, off, fill=None):
    """Flat buffers of n floats: expected values, bounds and the mask of written positions for one problem's results."""
    exp = np.zeros(n) if fill is None else fill
    bnd = np.zeros(n)
    mask = np.zeros(n, bool)
    for rows, cols, v, dv in results:
        idx = (rows[:, None] * ld + off + cols[None, :]).reshape(-1)
        exp[idx] = v.reshape(-1)
        bnd[idx] = dv.reshape(-1)
        mask[idx] = True
    return exp, bnd, mask
