"""The GPT-SoVITS sampler (t2s_sample_kernel, one launch through Engine.debug_t2s_sample) against the float64 restatements of
tests/t2s_ref.py at every vocabulary size regime and sampling setting the engine takes, and the decode step at the head widths
above 32 against oracle/t2s_oracle.py.

Sampler.  Support probes: a row whose draws are 2^-120 at entry v and 2^100 elsewhere samples v if and only if v's float32
probability is not 0 (2^-149 * 2^120 beats any probability * 2^-100), so Vv rows with equal logits read out the kernel's
whole support in one launch; it must equal t2s_ref.support on every entry that is not undecided (its margins, stated in
t2s_ref.py).  Every probe launch runs twice and must give the same bits.  Sampled tokens, from the caller's Exp(1) draws or
the Philox stream, must equal t2s_ref.expected_token on every row whose margins exceed the kernel's float32 error bound
(t2s_ref.py: ERR(v) = 2^-22 (|l_v| + |l_max|) / temp + 2^-22 |x_v| + 16 u in log units, the first term 0 for an exact tie
with the maximum); at least 90 % of rows are compared.

Decode step.  Logit budgets as tests/test_gpu_t2s.py keeps them (max |engine - float64 oracle| over every sampled step's
logits teacher-forced along the engine's tokens): 2e-4 in mode 0, 5e-3 in mode 1.  Measured on an H100 80GB HBM3 (700 W
power limit):
    D64   (128 wide, 2 heads of 64, V 1024)             mode 0 1.5e-6    mode 1 2.1e-5
    D96   (192 wide, 2 heads of 96, V 2049)             mode 0 1.4e-6    mode 1 2.3e-5
    D96_1 (96 wide, 1 head of 96, V 65)                 mode 0 8.0e-7
    D128  (256 wide, 2 heads of 128, V 4096)            mode 0 1.7e-6    mode 1 2.2e-5
    MAX   (1024 wide, 8 heads of 128, FFN 4096, V 4096) mode 0 2.9e-6    mode 1 3.5e-5
so the budgets hold 69x and 142x headroom at the widest.  None exceeds the 3.9e-6 / 5.9e-5 measured at 64 wide, below what
sqrt(width) scaling from there predicts (1.6e-5 / 2.4e-4 at 1024).
Sampled rows compared on the same H100: caller's q 100 % at V 3 and 65, 98.8 % at 1025, 94.0 % at 4096; Philox draws 99.7 %
at 65, 98.8 % at 1025, 96.9 % at 4096."""
import numpy as np
import pytest
import torch

import t2s_inputs as TI
import t2s_ref as R
from oracle import t2s_oracle as O

pytestmark = pytest.mark.gpu

VOCABS = [2, 3, 33, 65, 1024, 1025, 2048, 2049, 4095, 4096]
ST_T, ST_P, ST_KV, ST_NY, ST_GEN, ST_STOP, ST_YOFF = range(7)
BUDGET = {0: 2e-4, 1: 5e-3}
P0 = 3                                   # prompt tokens of every sampler row
_E = {}


def _engine(V):
    """A 1-layer, width-32 engine with a V-entry semantic vocabulary (the sampler reads only the vocabulary size)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if V not in _E:
        from vosk_tts_b200.gpt_sovits import Text2Semantic
        sd, cfg = TI.model({"hidden_dim": 32, "embedding_dim": 32, "head": 1, "n_layer": 1, "vocab_size": V, "phoneme_vocab_size": 8,
                            "dropout": 0.0, "EOS": V - 1})
        _E[V] = Text2Semantic((sd, cfg), precision=0)
    return _E[V].engine


def _state(B, P, gen, ny=None, stop=0):
    st = np.zeros((B, 8), np.int32)
    st[:, ST_P], st[:, ST_GEN], st[:, ST_NY], st[:, ST_STOP] = P, gen, P + gen if ny is None else ny, stop
    return st


def _bitmap(y, n, V):
    """The seen bitmap of each row's first n[b] tokens."""
    out = np.zeros((y.shape[0], (V + 31) // 32), np.uint32)
    for b in range(y.shape[0]):
        for t in y[b, :n[b]]:
            out[b, t >> 5] |= np.uint32(1) << np.uint32(t & 31)
    return out


def _logits(kind, V, r):
    """One step's logits (V entries, EOS last) and the row's previous tokens (P0 prompt tokens in [0, EOS), then one sampled
    token for steps after the first).  kinds: normal (spread 3), negative (every logit below -1: a negative pivot), dups (few
    distinct values: ties at the top, at the pivot and across the top-p cut), eos_tie (EOS equal to the largest penalised
    other logit), prev_max (the previous tokens repeat, the current maximum among them)."""
    z = r.standard_normal(V)
    l = z * 3.0
    if kind == "negative":
        l = -np.abs(l) - 1.0
    elif kind == "dups":
        l = np.round(z * 1.5)
        top = np.argsort(-l, kind="stable")[:3]
        l[top] = l.max()
    l = l.astype(np.float32)
    hi = max(V - 1, 1)
    prev = r.integers(0, hi, P0 + 1)
    if kind == "prev_max":
        am = int(np.argmax(l[:hi]))
        prev = np.array([am, am, int(r.integers(0, hi)), am], np.int64)
    if kind == "eos_tie" and V > 2:
        l[V - 1] = R.penalised(l[:V - 1], prev, 1.35).max()     # (the penalty the grid's eos_tie cases use)
    return l, prev.astype(np.int32)


def _launch_twice(eng, **kw):
    a = eng.debug_t2s_sample(**kw)
    b = eng.debug_t2s_sample(**kw)
    for k in ("state", "y", "seen"):
        assert np.array_equal(a[k], b[k]), k
    assert a["n_stopped"] == b["n_stopped"]
    return a


def _read_support(eng, l, prev, gen, top_k, top_p, temperature, penalty):
    """One probe launch, run twice: Vv rows of the logits l after the previous tokens prev (P0 + gen of them), row v's draws
    2^-120 at v and 2^100 elsewhere.  Returns (the launch's outputs, each row's token, the kernel's support mask)."""
    V = l.size
    Vv = V - 1 if gen == 0 else V
    n = P0 + gen
    q = np.full((Vv, gen + 1, V), 2.0 ** 100, np.float32)
    q[np.arange(Vv), gen, np.arange(Vv)] = 2.0 ** -120
    y = np.zeros((Vv, n + 1), np.int32)
    y[:, :n] = prev
    o = _launch_twice(eng, logits=np.tile(l, (Vv, 1)), state=_state(Vv, P0, gen), y=y, q=q, top_k=top_k, top_p=top_p,
                      temperature=temperature, repetition_penalty=penalty)
    tok = o["y"][:, n]
    return o, tok, tok == np.arange(Vv)


def _probe(V, kind, gen, top_k, top_p, temperature, penalty, seed):
    """Reads the kernel's support of one step out of one launch and checks it, the state after it, EOS at step 0 and the
    stop count.  Returns the number of entries compared."""
    eng = _engine(V)
    r = np.random.default_rng(seed)
    l, prev = _logits(kind, V, r)
    if kind == "eos_tie" and V > 2:
        l[V - 1] = R.penalised(l[:V - 1], prev[:P0 + gen], penalty).max()
    Vv = V - 1 if gen == 0 else V
    n = P0 + gen
    o, tok, got = _read_support(eng, l, prev[:n], gen, top_k, top_p, temperature, penalty)
    s = R.support(l[:Vv], prev[:n], **{"top_k": top_k, "top_p": top_p, "temperature": temperature, "penalty": penalty})
    dec = ~s.undecided
    bad = np.nonzero(dec & (got != s.live))[0]
    assert bad.size == 0, ("V %d %s gen %d k %d p %g t %g pen %g: entries %s kernel %s float64 %s" %
                           (V, kind, gen, top_k, top_p, temperature, penalty, bad[:8], got[bad[:8]], s.live[bad[:8]]))
    # a row that does not sample its own entry samples the smallest index of the largest probability
    other = tok[~got]
    assert np.all(s.live[other] | s.undecided[other])
    assert tok.max() < Vv                              # step 0 never draws EOS
    # the state: every row sampled once; it stops when the penalised argmax or the token is EOS
    st = o["state"]
    assert np.all(st[:, ST_GEN] == gen + 1) and np.all(st[:, ST_NY] == n)
    pen_arg = int(np.argmax(s.pen))
    stop = (pen_arg == V - 1) | (tok == V - 1)
    assert np.array_equal(st[:, ST_STOP], stop.astype(np.int32))
    assert o["n_stopped"] == int(stop.sum())
    if kind == "eos_tie" and gen > 0 and V > 2:
        assert pen_arg < V - 1                         # the tie goes to the smaller index: no stop on the argmax
    assert np.array_equal(o["seen"], _bitmap(o["y"], np.full(Vv, n + 1), V))
    return int(dec.sum())


KINDS = ["normal", "negative", "dups", "eos_tie", "prev_max"]
TOP_KS = [1, 20, 33, 64, 100, 1000, 5000]


@pytest.mark.parametrize("V", VOCABS)
def test_support_every_vocabulary(V):
    """Every vocabulary size, every top_k (5000 >= every V), both kinds of step, every kind of logits in turn."""
    compared = 0
    for i, k in enumerate(TOP_KS):
        for gen in (0, 1):
            if V == 2 and gen == 0:
                compared += _probe(V, "normal", 0, k, 1.0, 0.6, 1.35, 10 * i)   # one entry: it is always the token
                continue
            compared += _probe(V, KINDS[(i + gen) % len(KINDS)], gen, k, (1.0, 0.95)[gen], 0.6, 1.35, 100 * V + 10 * i + gen)
    assert compared > 0


def test_top_p_cut_exact_tie():
    """A cumulative probability exactly equal to top_p is not above it: four equal logits at the top and the rest 200 below
    (float32 probability exactly 0) give the sorted cumulative sums 0.25, 0.5, 0.75 and 1 exactly, so top_p 0.5 keeps the
    first two of the tie (the smaller indices), 0.75 three and 0.25 one.  (The float64 support calls such exact ties
    undecided; here the sums are exact in float32 too.)"""
    V = 65
    l = np.full(V, -200.0, np.float32)
    l[[5, 9, 17, 40]] = 3.0
    for tp, keep in ((0.5, [5, 9]), (0.75, [5, 9, 17]), (0.25, [5])):
        got = _read_support(_engine(V), l, np.zeros(P0 + 1, np.int32), 1, V, tp, 1.0, 1.0)[2]
        assert np.nonzero(got)[0].tolist() == keep, tp


GRID = [(tp, t, pen) for tp in (1.0, 0.95, 0.6, 1e-6) for t in (1e-6, 0.6, 1.0, 1.7) for pen in (1.0, 1.35, 0.7)]


@pytest.mark.parametrize("V", [65, 1025, 4096])
def test_support_sampling_grid(V):
    """Every combination of top_p, temperature (1e-6: clamped to 1e-5) and penalty, both kinds of step, the kinds of logits and
    top_k (20, 33, 100, >= V) in turn."""
    for i, (tp, t, pen) in enumerate(GRID):
        for gen in (0, 1):
            _probe(V, KINDS[(i + 2 * gen) % len(KINDS)], gen, (20, 33, 100, 5000)[(i + gen) % 4], tp, t, pen, 7 * i + gen + V)


def _sampled(V, cases, rows=32, seeded=False, seed=0):
    """Rows with their own logits, previous tokens and draws (the caller's q, or the Philox stream under per-row seeds); the
    kernel's token against expected_token on the firm rows.  Returns (compared, total)."""
    eng = _engine(V)
    r = np.random.default_rng(seed)
    compared = total = 0
    for ci, (kind, gen, k, tp, t, pen) in enumerate(cases):
        Vv = V - 1 if gen == 0 else V
        n = P0 + gen
        L = np.zeros((rows, V), np.float32)
        y = np.zeros((rows, n + 1), np.int32)
        for b in range(rows):
            l, prev = _logits(kind, V, r)
            if kind == "eos_tie" and V > 2:
                l[V - 1] = R.penalised(l[:V - 1], prev[:n], pen).max()
            L[b], y[b, :n] = l, prev[:n]
        kw = dict(top_k=k, top_p=tp, temperature=t, repetition_penalty=pen)
        if seeded:
            seeds = r.integers(0, 2 ** 63, rows, dtype=np.int64).astype(np.uint64)
            o = _launch_twice(eng, logits=L, state=_state(rows, P0, gen), y=y, seeds=seeds, **kw)
            draws = [R.philox_exp(seeds[b], gen, np.arange(V))[0] for b in range(rows)]
        else:
            q = r.exponential(1.0, (rows, gen + 1, V)).astype(np.float32)
            o = _launch_twice(eng, logits=L, state=_state(rows, P0, gen), y=y, q=q, **kw)
            draws = [q[b, gen] for b in range(rows)]
        for b in range(rows):
            tok, margin, bound, firm = R.expected_token(L[b, :Vv], y[b, :n], k, tp, t, pen, draws[b][:Vv])
            total += 1
            if firm:
                compared += 1
                assert o["y"][b, n] == tok, (V, ci, kind, gen, k, tp, t, pen, b, int(o["y"][b, n]), tok, margin, bound)
    return compared, total


@pytest.mark.parametrize("V", [3, 65, 1025, 4096])
def test_sampled_tokens_caller_q(V):
    """The sampling grid with the caller's Exp(1) rows (a seeded numpy stream), 32 rows of their own logits per cell."""
    cases = [(KINDS[i % len(KINDS)], i % 2, (20, 33, 100, 5000)[i % 4], tp, t, pen) for i, (tp, t, pen) in enumerate(GRID)]
    compared, total = _sampled(V, cases, seed=V)
    print("t2s sampler V %d, caller's q: %d of %d rows compared" % (V, compared, total))
    assert compared >= 0.9 * total, (compared, total)


@pytest.mark.parametrize("V", [2, 65, 1025, 4096])
def test_seeded_draws_exact(V):
    """Uniform logits, top_k >= V, top_p 1: every entry has the same probability, so the token is the entry of the largest
    restated u(seed, GEN, v), the smaller index on ties; checked wherever the two largest u are more than a quantum apart."""
    eng = _engine(V)
    rows, compared = 256, 0
    for gen in (0, 1, 5, 1000):
        Vv = V - 1 if gen == 0 else V
        seeds = (np.arange(rows, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(gen)).astype(np.uint64)
        o = eng.debug_t2s_sample(np.zeros((rows, V), np.float32), _state(rows, 0, gen), np.zeros((rows, gen + 1), np.int32), top_k=V,
                                 top_p=1.0, temperature=1.0, repetition_penalty=1.0, seeds=seeds)
        for b in range(rows):
            w = (R.philox_exp(seeds[b], gen, np.arange(Vv))[2] >> np.uint32(8)).astype(np.int64)
            o2 = np.lexsort((np.arange(Vv), -w))
            if Vv > 1 and w[o2[0]] - w[o2[1]] < 2:
                continue
            compared += 1
            assert o["y"][b, gen] == o2[0], (gen, b)
    assert compared >= 0.9 * rows * 4, compared


@pytest.mark.parametrize("V", [65, 1025, 4096])
def test_seeded_distribution(V):
    """Non-uniform logits on the Philox path: tokens equal expected_token under the restated draws on the firm rows."""
    cases = [("normal", 1, 20, 0.95, 0.6, 1.35), ("negative", 0, 100, 1.0, 1.0, 1.0), ("dups", 1, 5000, 0.6, 1.7, 0.7),
             ("prev_max", 1, 33, 1.0, 0.6, 1.35), ("normal", 0, 5000, 1.0, 1.0, 1.0)]
    compared, total = _sampled(V, cases, rows=64, seeded=True, seed=V + 1)
    print("t2s sampler V %d, Philox draws: %d of %d rows compared" % (V, compared, total))
    assert compared >= 0.9 * total, (compared, total)


def test_seed_per_sentence():
    """seeds=s gives sentence b the seed s + b: its tokens are those it gets alone under s + b."""
    eng = _engine(65)
    cfg = _E[65].cfg
    phs = [TI.phones(cfg, n, 50 + n) for n in (4, 9, 6)]
    kw = dict(early_stop_num=30, step_cap=40)
    toks, _ = eng.t2s_decode(phs, seeds=1000, **kw)
    for b in range(3):
        alone, _ = eng.t2s_decode([phs[b]], seeds=1000 + b, **kw)
        assert np.array_equal(toks[b], alone[0]), b
    assert not np.array_equal(eng.t2s_decode([phs[1]], seeds=1000, **kw)[0][0], toks[1]) or len(toks[1]) < 3


def test_state_machine():
    """Each rule of one launch, read back from the state, y, seen, the stop count and the raw-logit rows."""
    V = 65
    eng = _engine(V)
    r = np.random.default_rng(3)
    EOS = V - 1

    def rows(specs, **kw):
        B = len(specs)
        L = (r.standard_normal((B, V)) * 2).astype(np.float32)
        L[:, EOS] = -50.0
        st = np.zeros((B, 8), np.int32)
        y = np.zeros((B, 12), np.int32)
        q = r.exponential(1.0, (B, 12, V)).astype(np.float32)
        for b, sp in enumerate(specs):
            st[b, ST_P], st[b, ST_GEN], st[b, ST_STOP] = sp["P"], sp["gen"], sp.get("stop", 0)
            st[b, ST_NY] = sp.get("ny", sp["P"] + sp["gen"])
            st[b, ST_YOFF] = b * 12
            y[b, :sp["P"] + sp["gen"]] = r.integers(0, EOS, sp["P"] + sp["gen"])
            if "setup" in sp:
                sp["setup"](L[b], y[b], q[b])
        raw = np.full((B, 2, V), -7.0, np.float32)
        o = eng.debug_t2s_sample(L, st, y, q=q, raw=raw, **kw)
        return o, L, st, y, q

    def eos_argmax(l, y, q):          # the largest logit is a previous token's; penalised, EOS is the argmax; never sampled
        l[:] = np.clip(l, -3, 3)
        l[y[0]] = 10.0
        l[EOS] = 9.0
        q[:, EOS] = 2.0 ** 100

    def eos_sampled(l, y, q):         # EOS live but not the argmax, its draw tiny
        l[EOS] = l[:EOS].max() - 0.5
        q[:, EOS] = 2.0 ** -120

    def eos_tie(l, y, q):             # EOS tied with the penalised maximum: the argmax is the other entry, no stop
        l[EOS] = R.penalised(l[:EOS], y[:4], 1.35).max()
        q[:, EOS] = 2.0 ** 100

    specs = [dict(P=4, gen=3, stop=1), dict(P=5, gen=0, ny=2), dict(P=5, gen=2, ny=6), dict(P=3, gen=1), dict(P=4, gen=0),
             dict(P=2, gen=2, setup=eos_argmax), dict(P=2, gen=2, setup=eos_sampled), dict(P=3, gen=1, setup=eos_tie)]
    o, L, st, y, q = rows(specs, top_k=64, top_p=1.0, temperature=1.0, repetition_penalty=1.35, early_stop_num=-1, step_cap=100)
    s2 = o["state"]
    n_prev = st[:, ST_P] + st[:, ST_GEN]
    # a stopped row: untouched
    assert np.array_equal(s2[0], st[0]) and np.array_equal(o["y"][0], y[0]) and np.all(o["raw"][0] == -7.0)
    assert np.array_equal(o["seen"][0], _bitmap(y[:1], n_prev[:1], V)[0])
    # NY below P + GEN - 1: NY advances, nothing is sampled
    assert s2[1, ST_NY] == 3 and s2[1, ST_GEN] == 0 and s2[1, ST_STOP] == 0 and np.array_equal(o["y"][1], y[1])
    assert np.all(o["raw"][1] == -7.0)
    # NY one below: it advances to P + GEN and samples; at NY == P + GEN it samples
    for b in (2, 3, 4):
        assert s2[b, ST_NY] == n_prev[b] and s2[b, ST_GEN] == st[b, ST_GEN] + 1, b
    # the sampled token: expected_token's, its seen bit set, the raw-logit row of its step (EOS included at step 0)
    for b in (2, 3, 4, 5, 6, 7):
        gen, n = st[b, ST_GEN], n_prev[b]
        Vv = V - 1 if gen == 0 else V
        tok, _, _, firm = R.expected_token(L[b, :Vv], y[b, :n], 64, 1.0, 1.0, 1.35, q[b, gen, :Vv])
        if firm:
            assert o["y"][b, n] == tok, b
        assert np.array_equal(o["seen"][b], _bitmap(o["y"][b:b + 1], [n + 1], V)[0])
        if gen < 2:
            assert np.array_equal(o["raw"][b, gen], L[b]), b
            assert np.all(o["raw"][b, 1 - gen] == -7.0)
    assert o["raw"][4, 0, EOS] == -50.0                  # step 0: the EOS column is in the raw row
    # the stop rules: the penalised argmax EOS (row 5), a sampled EOS (row 6); a tie with EOS stops neither (row 7)
    assert o["y"][5, 4] != EOS and s2[5, ST_STOP] == 1
    assert o["y"][6, 4] == EOS and s2[6, ST_STOP] == 1
    assert o["y"][7, 4] != EOS and s2[7, ST_STOP] == 0
    assert np.array_equal(s2[2:5, ST_STOP], [0, 0, 0])
    assert o["n_stopped"] == 2
    assert np.array_equal(s2[:, ST_YOFF], np.arange(8) * 12)
    # early_stop: the row stops when GEN after the step exceeds it; step_cap: when it reaches the cap
    specs = [dict(P=2, gen=2), dict(P=2, gen=3), dict(P=0, gen=6)]
    o = rows(specs, top_k=20, top_p=0.9, temperature=0.8, repetition_penalty=1.35, early_stop_num=3, step_cap=100)[0]
    assert o["state"][:, ST_STOP].tolist() == [0, 1, 1] and o["n_stopped"] == 2
    o = rows(specs, top_k=20, top_p=0.9, temperature=0.8, repetition_penalty=1.35, early_stop_num=-1, step_cap=4)[0]
    assert o["state"][:, ST_STOP].tolist() == [0, 1, 1] and o["n_stopped"] == 2
    o = rows(specs, top_k=20, top_p=0.9, temperature=0.8, repetition_penalty=1.35, early_stop_num=-1, step_cap=7)[0]
    assert o["state"][:, ST_STOP].tolist() == [0, 0, 1] and o["n_stopped"] == 1


def test_sample_refusals():
    from vosk_tts_b200.engine import VttsError
    V = 33
    eng = _engine(V)
    L = np.zeros((2, V), np.float32)
    ok = dict(logits=L, state=_state(2, 1, 1), y=np.zeros((2, 3), np.int32), q=np.ones((2, 2, V), np.float32))
    eng.debug_t2s_sample(**ok)
    bad_y = np.zeros((2, 3), np.int32)
    bad_y[1, 0] = V
    neg_y = np.zeros((2, 3), np.int32)
    neg_y[0, 1] = -1
    for kw in (dict(y=bad_y), dict(y=neg_y), dict(q=np.ones((2, 1, V), np.float32)), dict(y=np.zeros((2, 2), np.int32)),
               dict(state=_state(2, 1, 1, ny=3)), dict(top_k=0), dict(repetition_penalty=0.0), dict(seeds=np.zeros(2, np.uint64))):
        args = dict(ok)
        args.update(kw)
        with pytest.raises(VttsError) as e:
            eng.debug_t2s_sample(**args)
        assert e.value.code == -1, kw
    for B in (0, 4097):
        with pytest.raises(VttsError) as e:
            eng.debug_t2s_sample(np.zeros((B, V), np.float32), _state(B, 0, 1), np.zeros((B, 2), np.int32), seeds=np.zeros(B, np.uint64))
        assert e.value.code == -1, B


# ---------------------------------------------------------------------------------------------------------------------------
# decode step at the head widths above 32
# ---------------------------------------------------------------------------------------------------------------------------
TS = (1, 31, 32, 33, 63, 600)
PS = (0, 1, 31, 33, 0, 40)
STEPS = 80
# the EOS logit of each block's hidden rows (t2s_inputs.model eos_logit): rows stop between steps 4 and 80, some reach the cap
EOS_LOGIT = {"D64": 1.4, "D96": 1.6, "D96_1": 0.6, "D128": 1.8, "MAX": 1.5}
_W = {}


def _wide(block, precision):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.gpt_sovits import Text2Semantic
    key = (block, precision)
    if key not in _W:
        sd, cfg = TI.model(getattr(TI, block), seed=11, eos_logit=EOS_LOGIT[block])
        _W[key] = (Text2Semantic((sd, cfg), precision=precision), sd, cfg)
    return _W[key]


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("block", ["D64", "D96", "D96_1", "D128", "MAX"])
def test_decode_widths(block, precision):
    """A ragged batch of 6 (not a multiple of the 4-row tiles): texts crossing the prefix attention's 32-key chunks, cache
    lengths crossing 64 and 128 during the run, a split count rounding past 8; rows stopping at different steps, frozen
    while the others run on.  Every row's logits against the float64 oracle, and its tokens and logits alone, bit for bit."""
    if block == "D96_1" and precision == 1:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        from vosk_tts_b200.engine import VttsError
        from vosk_tts_b200.gpt_sovits import Text2Semantic
        sd, cfg = TI.model(TI.D96_1, seed=11)
        with pytest.raises(VttsError, match="multiples of 64"):
            Text2Semantic((sd, cfg), precision=1)
        return
    m, sd, cfg = _wide(block, precision)
    V = cfg["t2s_vocab"]
    phs = [TI.phones(cfg, T, 300 + i) for i, T in enumerate(TS)]
    prs = [TI.prompt(cfg, P, 400 + i, repeat=i == 3) for i, P in enumerate(PS)]
    q = np.random.default_rng(7).exponential(1.0, (6, STEPS, V)).astype(np.float32)
    kw = dict(early_stop_num=-1, step_cap=STEPS, logits_steps=STEPS)
    toks, idx, lg = m.engine.t2s_decode(phs, prs, q=q, **kw)
    err, steps = 0.0, []
    for b in range(6):
        P = PS[b]
        n = len(toks[b]) - P + 1
        steps.append(n)
        ref = O.step_logits(sd, cfg, phs[b], toks[b], P=P).numpy()
        assert ref.shape[0] == n
        err = max(err, float(np.abs(lg[b, :n] - ref).max()))
        alone, aidx, alg = m.engine.t2s_decode([phs[b]], [prs[b]], q=q[b:b + 1], **kw)
        assert np.array_equal(alone[0], toks[b]) and aidx[0] == idx[b], b
        assert np.array_equal(alg[0], lg[b]), b
    print("t2s %s mode %d: steps %s, max logit error %.3g" % (block, precision, steps, err))
    assert len(set(steps)) > 2, steps                    # rows stop at different steps
    assert err < BUDGET[precision], err
