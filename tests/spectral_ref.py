"""Plain float64 restatements of the spectral kernels and the error bounds a correct kernel must meet against them:
  stft_mag_kernel          magnitude spectrogram (csrc/vc.cuh), from the definition: reflect padding, periodic Hann, rfft
  mel_log_kernel           log(max(mel @ mag, 1e-5)) on the kernel's own fp32 magnitude rows
  spec_pack_kernel         caller features [C][T] -> rows [T][ldo], exact (checked directly by the GPU test)
  istft_pqmf_kernel        exp / pi*sin / cos,sin -> transposed conv with the blob's basis -> (QuickVC) / window envelope ->
                           zero-stuffing x subbands -> 63-tap synthesis filter (csrc/kernels.cuh)
  mrf_mean_kernel / mrf_mean_planes_kernel    ((a + b) + c) / n in fp32, exact; planes split_bf16(lrelu(mean))
Utterances / clips are packed as the engine packs them (conv_ref.offsets: SEQ_GAP rows between them).

Bounds.  An fp32 sum of n terms, FMA or not and in any order, is within gamma_(n-1) * sum|t_i| of the exact sum (Higham,
eq. 4.4); as in conv_ref we take (n + 8) * 2^-23 * sum|t_i|, which also covers the fp32 rounding of each operand (the
DFT basis and the mel / synthesis banks are fp32 copies of float64 values: 2^-24 relative each).
  magnitude   E = (n_fft + 8) 2^-23 sum_n |x_n w_n| on re and on im; |d sqrt(re^2 + im^2 + e)| <= sqrt(2) E (1-Lipschitz in
              (re, im)), plus 4 roundings of the result (two squares, two adds, sqrt: 2^-24 relative each, halved through
              the square root) -> 4 * 2^-24 * mag.
  log-mel     the sum's bound Em = (nbins + 8) 2^-23 sum_k fb_k mag_k (all terms >= 0); the kernel's value must lie in
              [log(max(s - Em, 1e-5)), log(max(s + Em, 1e-5))] widened by logf's 1 ulp (2^-23 |log| + 2^-149): where the
              exact sum is within Em of the clamp either side of it is accepted.
  tail        CUDA's ulp table without --use_fast_math: expf, sinf, sincosf within 2 ulp (2 * 2^-23 relative of the
              result).  mag = expf(p): 2^-22 mag.  ph = pi_f * sinf(p): |dph| <= |ph| (2^-22 + 2 * 2^-24) (sinf, the
              product, pi rounded to fp32).  re, im = mag * (cos, sin)(ph): expf's and sincosf's errors (2^-22 each), the
              product's rounding and the phase error (cos, sin are 1-Lipschitz): drec = mag (2^-21 + 2^-24 + |dph|).  y = scale * sum over <= 4 frames x 18 channels: |dy| <= scale *
              (sum |basis| drec + 80 * 2^-23 sum |basis rec|), scale = n_fft / hop (a power of two: exact), or for QuickVC
              n_fft / hop / env with env a 4-term fp32 sum >= 1.25 (7 more roundings of y: 7 * 2^-24 |y|).  The filter:
              out = sum over <= 64 (tap, band) terms of h * subbands * y: |dout| <= sum |h| subbands |dy| + 72 * 2^-23 *
              sum |h subbands y|.
The CPU tests (test_spectral_ref.py) pin each reference to the oracles / torch and check that plausible kernel mistakes
(`mutate=`) break the bound on inputs the GPU tests run."""
import numpy as np

from conv_ref import offsets, split_bf16, lrelu32  # noqa: F401  (re-exported for the tests)

U23 = 2.0 ** -23
U24 = 2.0 ** -24
LOG_FLOOR = float(np.float32(1e-5))
EPS = float(np.float32(1e-6))
TAPS = 63
# the GPU tests' configurations: (name, filter_length, hop, mel channels or 0 for linear, model) -- model "vits2" or "quickvc"
FRONT_CONFIGS = [("lin1024", 1024, 256, 0, "vits2"), ("mel1024", 1024, 256, 80, "vits2"), ("qvc1280", 1280, 320, 80, "quickvc"),
                 ("mel2048", 2048, 512, 80, "vits2"), ("mel64", 64, 16, 80, "vits2"), ("mel1024h512", 1024, 512, 80, "vits2"),
                 ("mel3072", 3072, 768, 80, "vits2")]
TAIL_TY = [1, 2, 3, 4, 5, 17, 64, 1000]


# ---------------------------------------------------------------------------------------------------- front end
def min_clip(nfft, hop):
    """The shortest clip the engine frames: more samples than the reflect padding, and one frame."""
    return max((nfft - hop) // 2 + 1, hop)


def frames_of(L, nfft, hop):
    pad = (nfft - hop) // 2
    return (L + 2 * pad - nfft) // hop + 1


def length_for_frames(F, nfft, hop, extra=0):
    """A clip length giving F frames: the smallest one plus `extra` (< hop) samples."""
    pad = (nfft - hop) // 2
    L = max((F - 1) * hop + nfft - 2 * pad + extra, min_clip(nfft, hop))
    assert frames_of(L, nfft, hop) == F, (F, L)
    return L


def signal(kind, L, nfft, rng):
    """Test signals in [-1, 1] (float32)."""
    n = np.arange(L)
    if kind == "noise":
        x = rng.uniform(-1, 1, L)
    elif kind == "silence":
        x = np.zeros(L)
    elif kind == "dc":
        x = np.full(L, 0.75)
    elif kind == "nyquist":
        x = np.where(n % 2 == 0, 1.0, -1.0)
    elif kind == "tone":                 # centred on bin 5 (of n_fft)
        x = 0.9 * np.cos(2 * np.pi * 5 * n / nfft + 0.3)
    else:
        raise ValueError(kind)
    return x.astype(np.float32)


def _frames(x, nfft, hop, mutate=None):
    """Frames [F][n_fft] of the reflect-padded clip (float64)."""
    pad = (nfft - hop) // 2
    xp = np.pad(np.asarray(x, np.float64), pad, mode="symmetric" if mutate == "symmetric" else "reflect")
    h = hop + 1 if mutate == "hop+1" else hop
    F = frames_of(len(x), nfft, hop)
    idx = np.arange(F)[:, None] * h + np.arange(nfft)[None, :]
    idx = np.minimum(idx, len(xp) - 1)
    return xp[idx]


def hann(n):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)


def magnitude(x, nfft, hop, mutate=None):
    """Float64 magnitude spectrogram [F][n_fft/2 + 1] of one clip, and its bound.  mutate: "symmetric", "hop+1",
    "swap_dc_nyquist", "no_eps" (plausible kernel mistakes, for the sharpness tests)."""
    fr = _frames(x, nfft, hop, mutate) * hann(nfft)[None, :]
    X = np.fft.rfft(fr, axis=1)
    if mutate == "swap_dc_nyquist":
        X[:, [0, -1]] = X[:, [-1, 0]]
    eps = 0.0 if mutate == "no_eps" else EPS
    mag = np.sqrt(X.real ** 2 + X.imag ** 2 + eps)
    E = (nfft + 8) * U23 * np.abs(fr).sum(1, keepdims=True)
    bound = np.sqrt(2.0) * E + 4 * U24 * mag + 1e-12
    return mag, bound


def log_mel(mag32, fb32, floor=LOG_FLOOR):
    """Accepted interval [lo, hi] of mel_log_kernel's output on the kernel's fp32 magnitude rows [F][nbins] with the packed
    mel bank [nmel][nbins], and the float64 value."""
    m = np.asarray(mag32, np.float64)
    fb = np.asarray(fb32, np.float64)
    s = m @ fb.T
    Em = (fb.shape[1] + 8) * U23 * s
    v = np.log(np.maximum(s, floor))
    lo = np.log(np.maximum(s - Em, floor))
    hi = np.log(np.maximum(s + Em, floor))
    w = 2 * U23 * np.maximum(np.abs(lo), np.abs(hi)) + 1e-30
    return v, lo - w, hi + w


# ---------------------------------------------------------------------------------------------------- decoder tail
def post_values(kind, rows, pc, rng, nbins=9):
    """conv_post rows [rows][subbands * 18]: "normal" N(0, 1); "logmag" log-magnitudes spread over [-30, 8] (phases N(0,1));
    "phase" phase pre-activations 0, +-pi/2 and |x| ~ 100 (log-magnitudes N(0, 1))."""
    p = rng.standard_normal((rows, pc // (2 * nbins), 2, nbins))
    if kind == "logmag":
        p[:, :, 0, :] = rng.uniform(-30, 8, p[:, :, 0, :].shape)
    elif kind == "phase":
        choice = np.array([0.0, np.pi / 2, -np.pi / 2, 100.0, -100.25, 99.5])
        p[:, :, 1, :] = rng.choice(choice, p[:, :, 1, :].shape) + rng.choice([0.0, 1e-3], p[:, :, 1, :].shape)
    elif kind != "normal":
        raise ValueError(kind)
    return p.reshape(rows, pc).astype(np.float32)


def envelope(L1, w2, hop):
    """sum_f w2[u - f hop] over the frames covering u, for the kept samples u = n_fft/2 .. n_fft/2 + (L1 - 1) hop."""
    nfft = len(w2)
    full = np.zeros((L1 - 1) * hop + nfft)
    for f in range(L1):
        full[f * hop:f * hop + nfft] += np.asarray(w2, np.float64)
    return full[nfft // 2:nfft // 2 + (L1 - 1) * hop]


def tail(P, basis, bank, hop, w2=None, mutate=None):
    """Float64 iSTFT + synthesis filter of one utterance's conv_post rows P [L1][subbands * (n_fft + 2)] (fp32), with the
    blob's basis [n_fft + 2][n_fft], bank [subbands][63] and w2 [n_fft] (QuickVC) or None.  Returns (wav [subbands * M],
    bound).  mutate: "drop_last_frame", "pqmf_shift", "no_envelope"."""
    basis = np.asarray(basis, np.float64)
    bank = np.asarray(bank, np.float64)
    cps, nfft = basis.shape
    nb = cps // 2
    L1 = P.shape[0]
    sb = P.shape[1] // cps
    P = np.asarray(P, np.float64).reshape(L1, sb, cps)
    mag = np.exp(P[:, :, :nb])
    ph = np.pi * np.sin(P[:, :, nb:])
    rec = np.concatenate([mag * np.cos(ph), mag * np.sin(ph)], axis=2)              # [L1][sb][18]
    dph = np.abs(ph) * (2 * U23 + 2 * U24)
    drec = np.concatenate([mag * (2 * U23 + U24 + dph)] * 2, axis=2)
    if mutate == "drop_last_frame":
        rec = rec.copy()
        rec[-1] = 0.0
    Z = rec @ basis                                                                   # [L1][sb][n_fft]
    Zb = (drec + 80 * U23 * np.abs(rec)) @ np.abs(basis)
    M = (L1 - 1) * hop
    y = np.zeros((sb, (L1 - 1) * hop + nfft))
    yb = np.zeros_like(y)
    for pos in range(nfft):
        y[:, pos:pos + L1 * hop:hop][:, :L1] += Z[:, :, pos].T
        yb[:, pos:pos + L1 * hop:hop][:, :L1] += Zb[:, :, pos].T
    y = y[:, nfft // 2:nfft // 2 + M]
    yb = yb[:, nfft // 2:nfft // 2 + M]
    scale = nfft / hop
    if w2 is not None and mutate != "no_envelope":
        env = envelope(L1, w2, hop)
        y = y * (scale / env)
        yb = yb * (scale / env) + 7 * U24 * np.abs(y)
    else:
        y = y * scale
        yb = yb * scale
    # zero-stuffing x subbands, then out[n] = sum_k sum_j h[k][j] up_k[n + j - 31], zero outside [0, sb * M)
    n_out = sb * M
    up = np.zeros((sb, n_out))
    upb = np.zeros((sb, n_out))
    up[:, ::sb] = sb * y
    upb[:, ::sb] = sb * yb
    pad = (TAPS - 1) // 2
    out = np.zeros(n_out)
    ob = np.zeros(n_out)
    sh = 1 if mutate == "pqmf_shift" else 0
    for k in range(sb):
        c = np.convolve(up[k], bank[k][::-1], mode="full")                            # c[i] = sum_j h[j] up[i - 62 + j]
        cb = np.convolve(np.abs(up[k]), np.abs(bank[k][::-1]), mode="full")
        cbb = np.convolve(upb[k], np.abs(bank[k][::-1]), mode="full")
        s = TAPS - 1 - pad + sh
        out += c[s:s + n_out]
        ob += cbb[s:s + n_out] + 72 * U23 * cb[s:s + n_out]
    return out, ob + 1e-30


def tail_layout(lens, up_total, hop_total, first=0):
    """Post-row and sample offsets of packed utterances from row `first`: (post row of b, sample of b, rows, samples)."""
    offs = [o + first for o in offsets(lens)]
    prow = [offs[b] * up_total + b for b in range(len(lens))]
    wav0 = [offs[b] * hop_total for b in range(len(lens))]
    return prow, wav0, offs[-1] * up_total + len(lens), offs[-1] * hop_total


# ---------------------------------------------------------------------------------------------------- MRF mean
def mrf_mean(xs):
    """((a + b) + c) / n in fp32, the kernels' order."""
    s = np.asarray(xs[0], np.float32)
    for x in xs[1:]:
        s = (s + np.asarray(x, np.float32)).astype(np.float32)
    return (s / np.float32(len(xs))).astype(np.float32)
