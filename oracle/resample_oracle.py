"""Float64 restatement of the engine's resampler and silence trim (vtts_resample).

The resampler is scipy.signal.resample_poly(x, up, down) with its defaults: up / down = to_rate / from_rate reduced by
their gcd, a firwin low-pass of 2 * 10 * max(up, down) + 1 taps with cutoff 1 / max(up, down) (Nyquist = 1), a Kaiser
window of beta 5.0 and gain `up`, zero padding at both ends, ceil(n * up / down) outputs.  It is not librosa.load's
default (soxr_hq): that resampler uses a different filter design of the same band-limited kind.

The trim is librosa.effects.trim(y, top_db) (librosa >= 0.10): frames of 2048 samples with hop 512, centred with zero
padding; a frame is non-silent iff 10 log10(max(1e-10, mse)) - 10 log10(max(1e-10, max mse)) > -top_db; the clip keeps
[first * 512, min(n, (last + 1) * 512)).  numpy only."""
from math import gcd

import numpy as np

FRAME, HOP = 2048, 512          # librosa.effects.trim's frame_length and hop_length
AMIN = 1e-10                    # amplitude_to_db's amin ** 2


def ratio(from_rate, to_rate):
    """(up, down): to_rate / from_rate in lowest terms."""
    g = gcd(int(from_rate), int(to_rate))
    return int(to_rate) // g, int(from_rate) // g


def taps(up, down):
    """The low-pass of resample_poly for (up, down): float64 [2 * 10 * max(up, down) + 1], gain `up`."""
    m = max(up, down)
    half = 10 * m
    n = np.arange(2 * half + 1) - half
    h = np.sinc(n / m) / m * np.kaiser(2 * half + 1, 5.0)       # firwin: right * sinc(right * n) * window, right = 1 / m
    return h / h.sum() * up                                     # firwin scales to unit DC gain; resample_poly multiplies by up


def polyphase(up, down):
    """The taps laid out per phase as the engine uploads them: [up][ceil(L / up)], phase p holding h[p + up * q], zeros past L."""
    h = taps(up, down)
    K = -(-h.size // up)
    out = np.zeros(up * K)
    out[:h.size] = h
    return out.reshape(K, up).T.copy()


def out_length(n, from_rate, to_rate):
    up, down = ratio(from_rate, to_rate)
    return -(-int(n) * up // down)


def _chain(x, from_rate, to_rate, P):
    """sum_q P[p, q] x[j0 - q] of every output: t = m down + half, p = t mod up, j0 = t div up, x zero outside [0, n)."""
    up, down = ratio(from_rate, to_rate)
    K, half, n = P.shape[1], 10 * max(up, down), x.size
    t = np.arange(out_length(n, from_rate, to_rate), dtype=np.int64) * down + half
    p, j0 = t % up, t // up
    xp = np.concatenate([np.zeros(K), x, np.zeros(1)])          # xp[j + K] = x[j]; index -1 (+ K) is a zero of the left pad
    y = np.zeros(t.size)
    for q in range(K):
        j = j0 - q
        y += P[p, q] * xp[np.where(j < n, j, -1) + K]
    return y


def resample(x, from_rate, to_rate):
    """resample_poly(x, up, down) of a 1-D signal, in float64 (equal rates: a copy)."""
    x = np.asarray(x, np.float64).reshape(-1)
    up, down = ratio(from_rate, to_rate)
    return x.copy() if up == down else _chain(x, from_rate, to_rate, polyphase(up, down))


def bound(x, from_rate, to_rate):
    """Per-output bound on |fp32 engine - resample(x)|.  The engine evaluates output m as a K-term fp32 FMA chain over taps
    rounded to fp32 once.  With S = sum_q |h||x| (= sum |h x|): each of the K roundings of the chain is at most 2^-24 of a
    partial sum, and |partial sum| <= S, so the chain is off by at most K 2^-24 S <= (K + 8) 2^-23 S (the margin covers the
    rounding of the chain's products and of the fp64 reference); a tap rounded to fp32 moves by at most 2^-24 |h|, which
    adds 2^-24 S.  Equal rates are an exact copy: 0."""
    x = np.asarray(x, np.float64).reshape(-1)
    up, down = ratio(from_rate, to_rate)
    if up == down:
        return np.zeros(x.size)
    P = np.abs(polyphase(up, down))
    S = _chain(np.abs(x), from_rate, to_rate, P)
    return (P.shape[1] + 8) * 2.0 ** -23 * S + 2.0 ** -24 * S


def frame_energies(y):
    """Sum of squares of every centred 2048-sample frame at hop 512 (1 + n // 512 frames), float64: frame f covers
    y[512 f - 1024, 512 f + 1024), zeros outside the clip, as four 512-sample blocks."""
    y = np.asarray(y, np.float64).reshape(-1)
    nf = 1 + y.size // HOP
    pad = np.zeros((nf + 3) * HOP)
    pad[FRAME // 2:FRAME // 2 + y.size] = y
    blk = (pad * pad).reshape(-1, HOP).sum(axis=1)
    return blk[:nf] + blk[1:nf + 1] + blk[2:nf + 2] + blk[3:nf + 3]


def trim_bounds(energies, n, top_db=20.0):
    """[start, end) that librosa.effects.trim(y, top_db) keeps, from the frame energies of y (n samples).  None when the clip
    is digital silence (every frame's mean square at or below 1e-10): librosa then keeps the whole clip, which has no voice
    to keep; the engine refuses it."""
    mse = np.asarray(energies, np.float64) / FRAME
    top = float(mse.max())
    if top <= AMIN:
        return None
    db = 10.0 * np.log10(np.maximum(AMIN, mse)) - 10.0 * np.log10(max(AMIN, top))
    nz = np.flatnonzero(db > -float(top_db))
    return int(nz[0]) * HOP, min(int(n), (int(nz[-1]) + 1) * HOP)


def trim(y, top_db=20.0):
    """y[start:end] of trim_bounds, or None for digital silence."""
    y = np.asarray(y, np.float64).reshape(-1)
    b = trim_bounds(frame_energies(y), y.size, top_db)
    return None if b is None else y[b[0]:b[1]]
