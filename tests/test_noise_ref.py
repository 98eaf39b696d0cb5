"""The Gaussian noise restatement of tests/noise_ref.py on the CPU.  The draws must be N(0, 1) by their moments and by a
Kolmogorov-Smirnov test, their largest magnitude must be the one the u grid allows, and neighbouring counters, streams and
seeds must be uncorrelated.  Every seed is fixed, so each test gives the same answer on every run."""
import math

import numpy as np
import pytest
from scipy import stats

import noise_ref as R
import t2s_ref as T

N22 = 2 ** 22


def _grid(seed, stream, n_a=2048, n_b=2048, a0=0, b0=0):
    a, b = np.meshgrid(np.arange(a0, a0 + n_a, dtype=np.int64), np.arange(b0, b0 + n_b, dtype=np.int64), indexing="ij")
    return R.philox_normal(seed, stream, a, b)[0].reshape(-1)


def test_words_and_rounding():
    """The counter is (a, bidx, stream, 0x5eed) under the key (seed lo, seed hi).  u1 and u2 come from words 0 and 1 and
    are rounded as float32 rounds them: (k + 1/2) 2^-24 below 2^23, ties to even above, and 1.0 at the top word."""
    seed, stream, a, bidx = 0x0123456789ABCDEF, 3, 77, 1234
    w = T.philox4x32((a, bidx, stream, 0x5EED), (seed & 0xFFFFFFFF, seed >> 32))
    e, u1, u2 = R.philox_normal(seed, stream, a, bidx)
    assert u1 == R.uniform(w[0]) and u2 == R.uniform(w[1])
    assert e == pytest.approx(math.sqrt(-2 * math.log(float(u1))) * math.cos(2 * math.pi * float(u2)), rel=1e-14)
    k = np.arange(2 ** 24, dtype=np.uint64)
    u = R.uniform((k << np.uint64(8)).astype(np.uint32)).astype(np.float64)
    lo = k < 2 ** 23
    assert np.array_equal(u[lo], (k[lo] + 0.5) * 2.0 ** -24)
    hi = k[~lo]
    assert np.array_equal(u[~lo], (hi + (hi & np.uint64(1))).astype(np.float64) * 2.0 ** -24)     # k + 0.5 to even
    assert np.count_nonzero(u == 1.0) == 1 and u[-1] == 1.0
    assert u.min() == 2.0 ** -25 and np.all(u > 0)


def test_largest_draw_is_the_grid_edge():
    """No draw exceeds sqrt(-2 ln 2^-25) = 5.887, the value of the smallest u1 with cos = 1, and the u1 = 1 draw is 0."""
    assert abs(R.E_MAX - 5.887) < 5e-4
    u = R.uniform(np.arange(2 ** 24, dtype=np.uint64).astype(np.uint32) << np.uint32(8)).astype(np.float64)
    r = np.sqrt(-2 * np.log(u))
    assert r.max() == R.E_MAX and r.min() == 0.0
    assert R.cospi(np.float32(2 * 2.0 ** -25)) == pytest.approx(1.0, abs=1e-13)
    assert R.cospi(np.float32(1.5)) == 0.0
    e = np.concatenate([_grid(s, st) for s, st in ((0, 1), (2 ** 64 - 1, 7))])
    assert np.abs(e).max() <= R.E_MAX
    assert np.abs(e).max() > 5.0                             # the largest of 2^23 normals is about 5.4


@pytest.mark.parametrize("seed,stream", [(0, 1), (0x0123456789ABCDEF, 2), (2 ** 64 - 1, 3), (0x7FC000007F800001, 7)])
def test_moments_and_ks(seed, stream):
    """2^22 draws: mean, variance, skewness and excess kurtosis within 6 standard errors of N(0, 1)'s, and a
    Kolmogorov-Smirnov test against N(0, 1) at p > 1e-6."""
    e = _grid(seed, stream)
    n = e.size
    assert n == N22
    mean, var = e.mean(), e.var()
    skew = stats.skew(e)
    kurt = stats.kurtosis(e)                                # excess kurtosis: 0 for a normal
    assert abs(mean) < 6 / math.sqrt(n), mean
    assert abs(var - 1) < 6 * math.sqrt(2 / n), var
    assert abs(skew) < 6 * math.sqrt(6 / n), skew
    assert abs(kurt) < 6 * math.sqrt(24 / n), kurt
    assert stats.kstest(e, "norm").pvalue > 1e-6


def _uncorrelated(x, y):
    assert x.size == y.size
    r = np.corrcoef(x, y)[0, 1]
    assert abs(r) < 6 / math.sqrt(x.size), r
    assert np.count_nonzero(x == y) < 4                     # no shared draws


SEED = 0x0123456789ABCDEF


@pytest.mark.parametrize("da,db", [(1, 0), (-1, 0), (0, 1), (0, -1)])
def test_neighbouring_counters(da, db):
    """Counters a +- 1 and bidx +- 1 (the next frame, the next channel or utterance) give uncorrelated draws."""
    x = _grid(SEED, 3, 1024, 1024, a0=1, b0=1)
    y = _grid(SEED, 3, 1024, 1024, a0=1 + da, b0=1 + db)
    _uncorrelated(x, y)


@pytest.mark.parametrize("s1,s2", [(1, 2), (1, 3), (1, 7), (2, 3), (2, 7), (3, 7)])
def test_streams(s1, s2):
    """Each pair of the four kernels' streams gives uncorrelated draws at the same counter."""
    _uncorrelated(_grid(SEED, s1, 1024, 1024), _grid(SEED, s2, 1024, 1024))


@pytest.mark.parametrize("bit", [0, 1, 31, 32, 33, 63])
def test_seeds_one_bit_apart(bit):
    """Seeds one bit apart, in the low half or the high half, give uncorrelated draws."""
    _uncorrelated(_grid(SEED, 2, 1024, 1024), _grid(SEED ^ (1 << bit), 2, 1024, 1024))


def test_kernel_layouts():
    """draws() keys each kernel as its source does: dp (t, 2b) and (t, 2b + 1) on stream 1, the others (t, b C + c) on
    their own stream; rows packed with 8 rows between utterances."""
    lens = [3, 1, 5]
    off = R.offsets(lens)
    assert list(off) == [0, 11, 20, 25]
    (e, row) = R.draws("dp", 5, lens)
    assert list(row) == [0, 1, 2, 11, 20, 21, 22, 23, 24]
    assert e[1, 3] == R.philox_normal(5, 1, 0, 3)[0]           # utterance 1, token 0, e1
    e, (row, c) = R.draws("posterior", 5, lens, C=4)
    i = np.nonzero((row == 22) & (c == 3))[0][0]               # utterance 2, frame 2, channel 3
    assert e[i] == R.philox_normal(5, 3, 2, 2 * 4 + 3)[0]
    e, (row, c) = R.draws("dit", 5, lens, C=4)
    assert e[0] == R.philox_normal(5, 7, 0, 0)[0]


def test_bounds_cover_an_fp32_restatement():
    """A float32 evaluation of the kernel's arithmetic (numpy's float32 log, sqrt and exp, and cos(2 pi u2) rounded to
    float32, each within the CUDA functions' ulp bounds) lies within each bound, and the draw's bound is under 6 u
    relative."""
    rng = np.random.default_rng(5)
    e, u1, u2 = R.philox_normal(SEED, 3, np.arange(200000), 9)
    c32 = np.float32(R.cospi(2.0 * u2.astype(np.float64)))
    e32 = np.sqrt(np.float32(-2) * np.log(u1)) * c32
    assert np.all(np.abs(e32 - e) <= R.normal_bound(e))
    assert R.REL_E < 6 * R.U
    s = np.float32(0.667)
    assert np.all(np.abs((e32 * s).astype(np.float64) - e * float(s)) <= R.scaled_bound(e, s))
    m = rng.normal(0, 2, e.size).astype(np.float32)
    ls = rng.uniform(-3, 1.5, e.size).astype(np.float32)
    out = m + (e32 * np.exp(ls)) * s
    ref, b = R.sample_ref(e, m, ls, s)
    assert out.dtype == np.float32
    assert np.all(np.abs(out.astype(np.float64) - ref) <= b)


def test_bounds_catch_a_wrong_constant():
    """Draws of cospif(u2) instead of cospif(2 u2), or of sqrt(-logf(u1)), break the bound almost everywhere."""
    e, u1, u2 = R.philox_normal(SEED, 2, np.arange(10000), 0)
    wrong = np.sqrt(-2 * np.log(u1.astype(np.float64))) * R.cospi(u2.astype(np.float64))
    assert np.mean(np.abs(wrong - e) > R.normal_bound(e)) > 0.99
    wrong = np.sqrt(-np.log(u1.astype(np.float64))) * R.cospi(2.0 * u2.astype(np.float64))
    assert np.mean(np.abs(wrong - e) > R.normal_bound(e)) > 0.99
