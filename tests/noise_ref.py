"""Restatement of the engine's Gaussian noise (kernels.cuh philox_normal) and of the four kernels that draw it when the caller
gives no noise, with a bound on how far each device value may lie from the float64 value of the same draw.

philox_normal(seed, stream, a, bidx) runs Philox4x32-10 (t2s_ref.philox4x32) on the counter (a, bidx, stream, 0x5eed) under
the key (seed lo, seed hi).  Words 0 and 1 become u1 and u2 exactly as the kernel rounds them in float32:
u = ((float)(w >> 8) + 0.5f) * 2^-24.  For k = w >> 8 < 2^23 that is (k + 1/2) 2^-24.  For k >= 2^23 the sum k + 0.5 is a
tie between two floats one apart and rounds to the even one, so u1 = 1.0 exactly for k = 2^24 - 1, and that draw is 0.  The
smallest u is 2^-25, so no draw exceeds E_MAX = sqrt(-2 ln 2^-25) = 5.8870.  The draw is then
e = sqrt(-2 ln u1) cos(2 pi u2), which is evaluated here in float64 from those exact float32 u.

Counters by kernel (b: the utterance's index in the batch, t: token or frame, c: channel; I = inter_channels, NC =
noise_channels):
  dp_noise_kernel          stream 1   e0 = (t, 2b), e1 = (t, 2b + 1)          za, zb = e * noise_scale_w
  sample_prior_kernel      stream 2   (t, b I + c)                            z_p = m + e * exp(logs) * noise_scale
  posterior_sample_kernel  stream 3   (t, b I + c)                            z = m + e * exp(logs) * noise_scale
  dit_init_kernel          stream 7   (t, b NC + c), both branches of b       x = e * temperature

Device error bounds.  u = 2^-24 is the float32 unit roundoff.  The maximum errors of the CUDA single-precision functions are
those in the CUDA C++ Programming Guide, appendix "Mathematical Functions", table of single-precision functions with their
maximum ulp error:
  logf 1 ulp, cospif 1 ulp, expf 2 ulp, and sqrtf 0 ulp (correctly rounded) when compiled with -prec-sqrt=true.  That is
  nvcc's default without -use_fast_math, and vosk_tts_b200/build.py does not pass -use_fast_math.
An error of n ulp of a normal float32 result r is at most n 2^-23 |r|.
  draw: L = logf(u1) has a relative error of at most 2u.  -2 L is exact.  sqrtf(-2 L) adds u, and sqrt halves the error
    of L, which gives u.  cospif(2 u2) has 2u, and 2 u2 is exact.  The product adds u.  Together:
        |e_dev - e| <= 5 u |e| (1 + 2^-20)                                                      (normal_bound)
    The 1 + 2^-20 covers the second-order terms and the float64 evaluation of e (about 2^-52 relative).  The only zero of
    the cosine the grid reaches is 2 u2 = 3/2 (u2 = 0.75), where a 1-ulp cospif is exactly 0.  Everywhere else 2 u2 is at
    least 2^-24 from a half-integer, so |cos| > 1e-7 and the result is a normal float.
  e * s (dp_noise_kernel, dit_init_kernel): one rounding of the product, so
        |fl(e_dev s) - e s| <= |s| (B_e (1 + u) + u |e|)                                        (scaled_bound)
  m + e * exp(ls) * s (the samplers: __fadd_rn(m, __fmul_rn(__fmul_rn(e, expf(ls)), s))): expf has 4u relative, and each
  of the two products u.  With P the device product and T = e exp(ls) s,
        |P - T| <= |s| exp(ls) (B_e + 6u |e|) (1 + 2^-20)
        |fl(m + P) - (m + T)| <= |P - T| + u (|m + T| + |P - T|) + 2^-149                        (sample_bound)
    The last term is a denormal result's absolute rounding."""
import math

import numpy as np

from t2s_ref import MASK, philox4x32

U = 2.0 ** -24
STREAMS = {"dp": 1, "prior": 2, "posterior": 3, "dit": 7}
E_MAX = math.sqrt(-2.0 * math.log(2.0 ** -25))
REL_E = 5 * U * (1 + 2.0 ** -20)


def uniform(w):
    """The kernel's float32 u of Philox words w (uint32): ((float)(w >> 8) + 0.5f) * 2^-24, rounded as float32 rounds it."""
    w = np.asarray(w, np.uint32)
    return ((w >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


def cospi(x):
    """cos(pi x) in float64 for float32 x in [0, 2], relatively accurate near its zeros: it is rewritten as sin(pi d) with d =
    1/2 - x or x - 3/2.  Both are exact in float64, and |pi d| <= pi / 2."""
    x = np.asarray(x, np.float64)
    d = np.where(x <= 1.0, 0.5 - x, x - 1.5)
    return np.sin(np.pi * d)


def philox_normal(seed, stream, a, bidx):
    """The kernel's draw for counter (a, bidx) of `stream` under the 64-bit `seed` (each broadcast; seed a Python int or
    uint64 array).  Returns (e float64, u1 float32, u2 float32)."""
    seed = np.asarray(seed, np.uint64)
    a, bidx, stream = (np.asarray(v, np.uint64) for v in (a, bidx, stream))
    z = np.zeros(np.broadcast(seed, stream, a, bidx).shape, np.uint64)
    w = philox4x32((a + z, bidx + z, stream + z, z + np.uint64(0x5EED)), (seed & MASK, seed >> np.uint64(32)))
    u1, u2 = uniform(w[0]), uniform(w[1])
    e = np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * cospi(2.0 * u2.astype(np.float64))
    return e, u1, u2


def offsets(lens, gap=8):
    """Row offsets of utterances packed as the engine packs them: SEQ_GAP (8) rows between neighbours; the last entry is
    the row count."""
    off = [0]
    for i, n in enumerate(lens):
        off.append(off[-1] + int(n) + (gap if i + 1 < len(lens) else 0))
    return np.asarray(off, np.int64)


def layout(lens, C):
    """(b, t, c, row) of every element an utterance of `lens` covers, C channels per row, rows packed by offsets(lens)."""
    off = offsets(lens)
    b = np.concatenate([np.full(int(n), i, np.int64) for i, n in enumerate(lens)])
    t = np.concatenate([np.arange(int(n), dtype=np.int64) for n in lens])
    row = off[b] + t
    c = np.arange(C, dtype=np.int64)
    return (np.repeat(b, C), np.repeat(t, C), np.tile(c, b.size), np.repeat(row, C))


def draws(kernel, seed, lens, C=1):
    """Every draw a kernel makes for utterances of `lens` rows (dit: extents), C channels.  dp: e float64 [2, n] (e0 and e1
    of each token in packed order) and the rows [n]; the others: e [n * C] and (row, c) of each."""
    s = STREAMS[kernel]
    if kernel == "dp":
        b, t, _, row = layout(lens, 1)
        e0 = philox_normal(seed, s, t, 2 * b)[0]
        e1 = philox_normal(seed, s, t, 2 * b + 1)[0]
        return np.stack([e0, e1]), row
    b, t, c, row = layout(lens, C)
    return philox_normal(seed, s, t, b * C + c)[0], (row, c)


def normal_bound(e):
    return REL_E * np.abs(e)


def scaled_bound(e, s):
    s = abs(float(np.float32(s)))
    return s * (normal_bound(e) * (1 + U) + U * np.abs(e))


def sample_ref(e, m, ls, s):
    """The float64 value m + e exp(ls) s (m, ls, s at their float32 values) and its bound for the device."""
    m, ls = np.asarray(m, np.float64), np.asarray(ls, np.float64)
    s = float(np.float32(s))
    ref = m + e * np.exp(ls) * s
    dp = abs(s) * np.exp(ls) * (normal_bound(e) + 6 * U * np.abs(e)) * (1 + 2.0 ** -20)
    return ref, dp + U * (np.abs(ref) + dp) + 2.0 ** -149
