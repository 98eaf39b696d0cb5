"""The sampler restatements of tests/t2s_ref.py on the CPU: the Philox stream against Random123's known answers, its
uniformity and its keying, and the support against oracle.t2s_oracle.sample."""
import numpy as np
import pytest
import torch
from scipy import stats

import t2s_ref as R
from oracle import t2s_oracle as O

M32 = 0xFFFFFFFF


@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((M32, M32, M32, M32), (M32, M32), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))])
def test_philox_known_answers(ctr, key, out):
    """Random123's kat_vectors for philox4x32 with 10 rounds."""
    assert tuple(int(w) for w in R.philox4x32(ctr, key)) == out


def test_philox_exp_words():
    """u is the top 24 bits of word 0 plus a half, rounded to float32 as the kernel's float arithmetic rounds it, and the
    draw is -log(u); the counter is (step, v, 11, 0x5eed) and the key the seed's low then high word."""
    seed, step, v = 0x123456789ABCDEF0, 7, 1000
    d, u, w = R.philox_exp(seed, step, v)
    assert int(w) == int(R.philox4x32((step, v, 11, 0x5EED), (seed & M32, seed >> 32))[0])
    assert u == np.float32((np.float32(int(w) >> 8) + np.float32(0.5)) * np.float32(2.0 ** -24))
    assert d == -np.log(np.float64(u))
    # the largest word: 2^24 - 0.5 rounds to even, u = 1 and the draw 0 (the one draw the float32 rounding leaves at an end)
    top = np.uint32(0xFFFFFF00)
    assert ((top >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24) == np.float32(1.0)


@pytest.mark.parametrize("seed", [0, 1, 0x5EED, 2 ** 63 + 12345])
def test_philox_exp_uniform(seed):
    """u over a (step, v) grid is uniform on (0, 1) and the draws are Exp(1): Kolmogorov-Smirnov at p > 1e-6."""
    step, v = np.meshgrid(np.arange(16), np.arange(4096), indexing="ij")
    d, u, _ = R.philox_exp(seed, step, v)
    assert stats.kstest(u.ravel().astype(np.float64), "uniform").pvalue > 1e-6
    assert stats.kstest(d.ravel(), "expon").pvalue > 1e-6
    assert 0.0 < u.min() and u.max() <= 1.0


def test_philox_streams_are_keyed():
    """Seeds s and s + 1 (and s + 2^32, the key's high word) give streams that do not coincide, and so do neighbouring
    steps and entries under one seed."""
    step, v = np.meshgrid(np.arange(16), np.arange(4096), indexing="ij")
    for s in (0, 77, 2 ** 40 + 5):
        w = R.philox_exp(s, step, v)[2]
        for other in (R.philox_exp(s + 1, step, v)[2], R.philox_exp(s + 2 ** 32, step, v)[2], R.philox_exp(s, step + 1, v)[2],
                      R.philox_exp(s, step, v + 1)[2]):
            assert np.count_nonzero(w == other) <= 2           # (a chance collision of 32-bit words: 1.5e-5 expected)
        assert np.unique(w).size >= w.size - 2


def _case(r, trial):
    V = int(r.choice([2, 3, 5, 33, 65, 200]))
    l = (r.standard_normal(V) * 3).astype(np.float32)
    kind = trial % 4
    if kind == 1:
        l = -np.abs(l) - 1.0                                   # all negative: the pivot is negative
    elif kind == 2:
        l = np.round(l).astype(np.float32)                     # many exact ties
    elif kind == 3 and V > 2:
        l[r.integers(0, V, max(1, V // 3))] = l.max()          # ties at the top
    prev = r.integers(0, V, int(r.integers(0, 6)))
    k = int(r.choice([1, 3, 20, V, V + 5]))
    tp = float(r.choice([1.0, 0.95, 0.6, 1e-6]))
    temp = float(r.choice([1e-6, 0.6, 1.0, 1.7]))
    pen = float(r.choice([1.0, 1.35, 0.7]))
    return l.astype(np.float32), prev, k, tp, temp, pen


def test_support_contains_oracle_samples():
    """Every entry oracle.t2s_oracle.sample returns is in the support (or undecided), under random Exp(1) draws and under
    probe draws that single an entry out (q = 2^-120 there, 2^100 elsewhere): an entry the support keeps and calls live,
    O.sample returns under its probe; expected_token agrees with O.sample wherever both call the step firm."""
    r = np.random.default_rng(0)
    compared = 0
    for trial in range(120):
        l, prev, k, tp, temp, pen = _case(r, trial)
        V = l.size
        s = R.support(l, prev, k, tp, temp, pen)
        lt = torch.from_numpy(l.astype(np.float64))
        for v in range(V):
            q = np.full(V, 2.0 ** 100)
            q[v] = 2.0 ** -120
            tok = O.sample(lt, prev, k, tp, temp, pen, q)[0]
            assert s.kept[tok] or s.undecided[tok], (trial, v, tok)
            if s.live[v] and not s.undecided[v]:
                assert tok == v, (trial, v, tok)
        for _ in range(8):
            q = r.exponential(1.0, V).astype(np.float32)
            tok = O.sample(lt, prev, k, tp, temp, pen, q.astype(np.float64))[0]
            assert s.kept[tok] or s.undecided[tok], (trial, tok)
            etok, margin, bound, firm = R.expected_token(l, prev, k, tp, temp, pen, q, sup=s)
            if firm:
                assert etok == tok, (trial, etok, tok)
                compared += 1
    assert compared >= 600, compared


def test_support_edges():
    """top_p 1e-6 keeps the first sorted entry alone (the smaller index of a tie at the top), top_k 1 every entry tied with
    it (the pivot is a value); top_k >= V with top_p 1 keeps everything above the underflow edge; a clamped temperature
    keeps exact ties with the maximum only."""
    l = np.array([1.0, 3.0, 3.0, -2.0, 0.5], np.float32)
    assert np.nonzero(R.support(l, [], 20, 1e-6, 1.0, 1.0).kept)[0].tolist() == [1]
    assert np.nonzero(R.support(l, [], 1, 1.0, 1.0, 1.0).kept)[0].tolist() == [1, 2]
    assert np.nonzero(R.support(l, [], 2, 1.0, 1.0, 1.0).kept)[0].tolist() == [1, 2]
    assert np.nonzero(R.support(l, [], 3, 1.0, 1.0, 1.0).kept)[0].tolist() == [0, 1, 2]
    s = R.support(l, [], 100, 1.0, 1.0, 1.0)
    assert s.live.all() and not s.undecided.any()
    s = R.support(l, [], 100, 1.0, 1e-6, 1.0)
    assert np.nonzero(s.live)[0].tolist() == [1, 2]
    # the penalty, once per entry however often it repeats: 3 / 1.35 falls below 2.5
    s = R.support(np.array([3.0, 2.5, 1.0, 0.5], np.float32), [0, 0, 2], 1, 1.0, 1.0, 1.35)
    assert np.nonzero(s.kept)[0].tolist() == [1]
    assert s.pen[0] == np.float32(3.0) / np.float32(1.35) and s.pen[2] == np.float32(1.0) / np.float32(1.35)
