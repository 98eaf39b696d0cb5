"""Restatements of the GPT-SoVITS sampler (t2s.cu t2s_sample_kernel) for the kernel tests: its Philox Exp(1) draws, the set
of entries it can sample, and the token it samples from given draws.

philox_exp restates philox4x32_t2s and philox_exp bit for bit: Philox4x32-10 on the counter (step, v, 11, 0x5eed) under the
key (seed lo, seed hi), the top 24 bits of word 0 to a float32 u in (0, 1) as the kernel rounds it, and -log(u).

support and expected_token follow oracle.t2s_oracle.sample's order of operations (repetition penalty, top-p cut, temperature,
top-k pivot, softmax, argmax of probs / q), ties to the smaller index as its stable sort gives them.  The penalty is one
correctly rounded float32 multiply or divide, as the kernel computes it, so that ties the caller builds after the penalty
stay ties; everything after it is float64.  The scalars are taken at their float32 values, as the kernel reads them.

Where the kernel's float32 arithmetic can decide an entry either way, the entry is "undecided" and the tests do not compare
it.  The bounds (float32 unit roundoff u = 2^-24):
  - top-k pivot: the kernel compares fl(l / temp) with fl(pivot / temp), which is monotone but may round two different values
    to one; entries within 2^-21 relative of the pivot (8 u) are undecided.  Exact ties with the pivot are decided (kept).
  - top-p cut: the kernel's inclusive cumulative sum of expf(l - max) / sum, per-thread runs of up to 4 entries, a 32-lane
    scan and a sum over 32 warps, has an absolute error below (4 + 5 + 32 + 4) u + 3 u < 3e-6; entries whose |cum - top_p|
    is below 1e-5 are undecided.
  - float32 underflow: a probability below 2^-150 (log -103.97) rounds to 0.  The kernel's log-probability of an entry is
    off by the rounding of fl(l / temp) - mx, at most 2^-22 (|l| + |max|) / temp, and by the denormal rounding of expf and
    of the division, under 1 in log units; entries within 1 + 2^-22 (|l| + |max|) / temp of the edge are undecided.
  - sampled token: the kernel's log score log(p / q) of a live entry is off by at most
    ERR(v) = 2^-22 (|l_v| + |l_max|) / temp + 2^-22 |x_v| + 16 u  (x_v = (l_v - l_max) / temp: the roundings of fl(l / temp)
    and of the subtraction, 4x over; none for an exact tie with the maximum, whose x is exactly 0; 16 u covers expf, the
    divisions by the sum and by q, and logf of a Philox draw), and the winner is decided when log(s1 / s2) > 2 max ERR over
    live entries; expected_token reports that margin and bound times the temperature, in logit units as O.sample does."""
import math

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)
UNDERFLOW = -150.0 * math.log(2.0)       # log of half the smallest float32 denormal: below it a probability rounds to 0
U = 2.0 ** -24
PIVOT_REL = 2.0 ** -21
CUT_TOL = 1e-5


def philox4x32(ctr, key, rounds=10):
    """Philox4x32 (Random123's philox4x32_R) on uint32 words, vectorised: ctr 4 arrays, key 2 arrays (broadcast together).
    The 32x32-bit products are taken in uint64, hi = p >> 32 and lo = p & 0xffffffff."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) for c in ctr)
    k0, k1 = (np.asarray(k, np.uint64) for k in key)
    for _ in range(rounds):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def philox_exp(seed, step, v):
    """The kernel's Exp(1) draw of entry v at sampling step `step` under `seed` (each broadcast).  Returns (draw float64
    = -log(u), u float32, word uint32: Philox's word 0, whose top 24 bits make u)."""
    seed = np.asarray(seed, np.uint64)
    step, v = np.asarray(step, np.uint64), np.asarray(v, np.uint64)
    z = np.zeros(np.broadcast(seed, step, v).shape, np.uint64)
    w = philox4x32((step + z, v + z, z + np.uint64(11), z + np.uint64(0x5EED)), (seed & MASK, seed >> np.uint64(32)))[0]
    u = ((w >> np.uint32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)
    return -np.log(u.astype(np.float64)), u, w


def penalised(logits, previous, penalty):
    """The logits with the repetition penalty on every entry of `previous` (once per entry), in float32 as the kernel does."""
    l = np.array(logits, np.float32)
    pen = np.float32(penalty)
    prev = np.unique(np.asarray(previous, np.int64).reshape(-1))
    if prev.size:
        s = l[prev]
        l[prev] = np.where(s < 0, s * pen, s / pen)
    return l


class Support:
    """What support() returns; arrays are indexed by vocabulary entry.
    kept        survives the top-p cut and the top-k pivot (float64)
    live        kept, and its float32 probability is not 0
    undecided   within a margin of the pivot, the top-p cut or the underflow edge
    piv, cut, under     the margins: |l - pivot| (0 on an exact tie, which is decided), |cum - top_p| (inf for the first
                sorted entry), |log p - UNDERFLOW| (inf where not kept)
    pen         the penalised logits; order the sorted order; K the entries the top-p cut keeps; pivot; temp; logp"""


def support(logits, previous, top_k, top_p, temperature, penalty):
    """The entries the kernel can sample from one step's logits (1-d, the EOS column already dropped at step 0)."""
    l = penalised(logits, previous, penalty)
    n = l.size
    lp = l.astype(np.float64)
    order = np.lexsort((np.arange(n), -lp))            # descending, smaller index first on ties (a stable sort)
    sl = lp[order]
    tp = float(np.float32(top_p))
    cut = np.full(n, np.inf)
    K = n
    if tp < 1.0:
        e = np.exp(sl - sl[0])
        cum = np.cumsum(e) / e.sum()
        cut[order[1:]] = np.abs(cum[1:] - tp)
        drop = np.nonzero(cum[1:] > tp)[0]
        if drop.size:
            K = int(drop[0]) + 1
    temp = max(float(np.float32(temperature)), float(np.float32(1e-5)))
    kk = min(int(top_k), n)
    pivot = sl[kk - 1] if kk - 1 < K else -np.inf
    pos = np.empty(n, np.int64)
    pos[order] = np.arange(n)
    kept = (pos < K) & (lp >= pivot)
    piv = np.where(pos < K, np.abs(lp - pivot), np.inf)
    piv_und = (piv > 0) & (piv <= PIVOT_REL * np.maximum(np.abs(lp), abs(pivot) if np.isfinite(pivot) else 0.0))
    x = np.where(kept, (lp - sl[0]) / temp, -np.inf)
    logp = x - (math.log(np.exp(x[kept]).sum()))
    under = np.where(kept, np.abs(logp - UNDERFLOW), np.inf)
    under_tol = 1.0 + 2.0 ** -22 * (np.abs(lp) + abs(sl[0])) / temp
    s = Support()
    s.kept, s.live = kept, kept & (logp > UNDERFLOW)
    s.undecided = piv_und | (cut < CUT_TOL) | (under < under_tol)
    s.piv, s.cut, s.under = piv, cut, under
    s.pen, s.order, s.K, s.pivot, s.temp, s.logp = l, order, K, pivot, temp, logp
    return s


def expected_token(logits, previous, top_k, top_p, temperature, penalty, q, sup=None):
    """The float64 argmax of probs / q (the smaller index on ties) over the live entries.  Returns (token, margin, bound,
    firm): margin = log(s1 / s2) times the temperature between the winner and the runner-up (inf with one live entry),
    bound = twice the largest ERR of a live entry times the temperature (logit units, as O.sample's margin), firm = the
    margin exceeds the bound and no entry is undecided at the pivot or the top-p cut."""
    s = support(logits, previous, top_k, top_p, temperature, penalty) if sup is None else sup
    q = np.asarray(q, np.float64)
    live = np.nonzero(s.live)[0]
    sc = s.logp[live] - np.log(q[live])
    o = np.lexsort((live, -sc))
    tok = int(live[o[0]])
    margin = float(sc[o[0]] - sc[o[1]]) * s.temp if live.size > 1 else math.inf
    lmax = abs(float(s.pen.astype(np.float64)[s.order[0]]))
    x = s.logp[live] - s.logp[live].max()
    lv = s.pen[live].astype(np.float64)
    err = np.where(lv == float(s.pen[s.order[0]]), 0.0, 2.0 ** -22 * (np.abs(lv) + lmax) / s.temp) + 2.0 ** -22 * np.abs(x) + 16 * U
    bound = 2.0 * float(err.max()) * s.temp
    near = (s.piv > 0) & (s.piv <= PIVOT_REL * np.maximum(np.abs(s.pen.astype(np.float64)), abs(s.pivot) if np.isfinite(s.pivot) else 0.0))
    firm = margin > bound and not near.any() and not (s.cut < CUT_TOL).any()
    return tok, margin, bound, firm
