"""The GPT-SoVITS text prefill's kernels alone (Engine.debug_t2s_*, each through the launch helper vtts_t2s_decode uses)
against float64 references, and the composed prefill at real prompt lengths against oracle/t2s_oracle.py.

Prefix attention (t2s_prefix_attn_kernel) against attn_ref.reference(T=...) and its bound, on ragged batches of 64
utterances packed as vtts_t2s_decode packs them (T + P rows from a multiple of 8, no gap), the (200, 3700) sequence near
the position table in three of them, with NaN on every row outside the utterances; every output finite, every launch
twice with the same bits, each utterance alone with its bits in the batch, an oversized launch row count changing
nothing, planes the split of out bit for bit, sentinels outside the utterances kept.  Mask
probes: a key scored +30 for every query with a one-hot 1e4 v marker dominates every row that sees it and leaves no trace
in any other.  Measured worst error / bound on an H100 80GB HBM3 (700 W power limit): see DESIGN.md 4.s.

Embedding, ReLU, cache store and decode-state init are exact: t2s_prefill_ref restates them bit for bit.

The composed prefill: vtts_t2s_decode with two logit steps against the float64 oracle (step 0 reads only the prefill, step 1
the stored cache), with the logit budgets of tests/test_gpu_t2s.py (2e-4 in mode 0, 5e-3 in mode 1).  A wide engine must keep
decoding after a narrower one is bound in the same process."""
import numpy as np
import pytest
import torch

import attn_ref as A
import conv_ref as CR
import t2s_inputs as TI
import t2s_prefill_ref as R
from oracle import t2s_oracle as O

pytestmark = pytest.mark.gpu

WIDTHS = [(16, 32), (2, 64), (2, 96), (1, 128), (8, 128)]          # (heads, dk): 512 wide as upstream, 1024 wide
PATTERNS = ["random", "rising", "large", "equal"]
BUDGET = {0: 2e-4, 1: 5e-3}
SENT = np.float32(-7.25)
PSENT = np.uint16(0xABCD)
_M = {}
_W = {}


def _t2s(block, precision=0):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.gpt_sovits import Text2Semantic
    key = (block, precision)
    if key not in _M:
        sd, cfg = TI.model(getattr(TI, block))
        _M[key] = (Text2Semantic((sd, cfg), precision=precision), sd, cfg)
    return _M[key]


def _worst(name, w):
    _W[name] = float(np.max([_W.get(name, 0.0), w]))           # (a NaN stays NaN)
    print("%s: worst error / bound %.3f (largest so far %.3f)" % (name, w, _W[name]))


def _tp(pairs):
    return [p[0] for p in pairs], [p[1] for p in pairs]


def _attn(eng, pairs, heads, qkv, launch_rows=0):
    T, P = _tp(pairs)
    rows, H = qkv.shape[0], qkv.shape[1] // 3
    out = np.full((rows, H), SENT, np.float32)
    hi = np.full((rows, H), PSENT, np.uint16)
    lo = np.full((rows, H), PSENT, np.uint16)
    return eng.debug_t2s_prefix_attn(T, P, heads, qkv, out, hi, lo, launch_rows=launch_rows)


def _same(a, b):
    return all(np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)
               for x, y in zip(a, b))


def _check_attention(eng, pairs, heads, dk, qkv, name, alone=True):
    T, P = _tp(pairs)
    lens = [t + p for t, p in pairs]
    offs, tot = R.offsets(T, P)
    got = _attn(eng, pairs, heads, qkv)
    assert _same(got, _attn(eng, pairs, heads, qkv)), "two launches differ"
    assert _same(got, _attn(eng, pairs, heads, qkv, launch_rows=max(lens) + 37)), "an oversized launch changes the output"
    out, hi, lo = got
    inside = R.rows_of(T, P)
    assert np.all(np.isfinite(out[inside])), "a non-finite output"
    res = A.reference(qkv, lens, heads, 0, None, "ffma", T=T, offs=offs)
    w = A.worst(out, res)
    _worst(name, w)
    assert w <= 1.0
    outside = np.setdiff1d(np.arange(out.shape[0]), inside)
    assert np.all(out[outside].view(np.uint32) == SENT.view(np.uint32))
    assert np.all(hi[outside] == PSENT) and np.all(lo[outside] == PSENT)
    sh, sl = CR.split_bf16(out[inside])
    assert np.array_equal(hi[inside], sh) and np.array_equal(lo[inside], sl)
    if alone:
        for b, (Tb, Pb) in enumerate(pairs):
            n = Tb + Pb
            q1 = np.full((-(-n // 8) * 8 + 8, qkv.shape[1]), np.nan, np.float32)
            q1[:n] = qkv[offs[b]:offs[b] + n]
            o1 = _attn(eng, [(Tb, Pb)], heads, q1)[0]
            assert np.array_equal(o1[:n].view(np.uint32), out[offs[b]:offs[b] + n].view(np.uint32)), b
    return out, res


# ------------------------------------------------------------------------------------------------ prefix attention
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("heads,dk", WIDTHS)
def test_prefix_attention(heads, dk, pattern):
    eng = _t2s("SMALL")[0].engine
    pairs = R.ragged_pairs(64, 100 + dk + heads)
    qkv = R.attn_qkv(pairs, heads, dk, pattern, 7 + dk)
    _check_attention(eng, pairs, heads, dk, qkv, "prefix attention", alone=pattern == "random")


@pytest.mark.parametrize("heads,dk,pattern", [(16, 32, "random"), (8, 128, "rising"), (2, 64, "large")])
def test_prefix_attention_near_the_position_table(heads, dk, pattern):
    """(200, 3700) in a ragged batch of 64 with every chunk-edge and real pair."""
    eng = _t2s("SMALL")[0].engine
    pairs = R.ragged_pairs(64, 500 + dk, extra=(R.LONG_PAIR,))
    qkv = R.attn_qkv(pairs, heads, dk, pattern, 11)
    _check_attention(eng, pairs, heads, dk, qkv, "prefix attention", alone=True)


@pytest.mark.parametrize("probe", [0, "first_prompt", "last"])
@pytest.mark.parametrize("heads,dk", [(16, 32), (1, 128)])
def test_prefix_attention_mask_probes(heads, dk, probe):
    eng = _t2s("SMALL")[0].engine
    pairs = R.ragged_pairs(64, 300 + dk)
    qkv, keys = R.attn_qkv(pairs, heads, dk, "random", 13, probe=probe)
    out, _ = _check_attention(eng, pairs, heads, dk, qkv, "prefix attention", alone=False)
    offs, _ = R.offsets(*_tp(pairs))
    for b, (Tb, Pb) in enumerate(pairs):
        t = np.arange(Tb + Pb)
        sees = (keys[b] < Tb) | (keys[b] <= t)
        marker = out[offs[b] + t][:, ::dk]                    # channel 0 of every head
        assert np.all(marker[sees] > 0.9e4), (b, Tb, Pb, keys[b])
        assert np.all(np.abs(marker[~sees]) < 1e2), (b, Tb, Pb, keys[b])


def test_prefix_attention_refusals():
    from vosk_tts_b200.engine import VttsError
    eng = _t2s("SMALL")[0].engine
    qkv = R.attn_qkv([(3, 2)], 2, 32, "random", 1)
    bad = [dict(heads=3), dict(heads=1, qkv=R.attn_qkv([(3, 2)], 1, 160, "random", 1)),
           dict(heads=4, qkv=R.attn_qkv([(3, 2)], 4, 16, "random", 1)), dict(T=[0]), dict(P=[-1]),
           dict(T=[40]), dict(launch_rows=4)]
    for kw in bad:
        a = dict(T=[3], P=[2], heads=2, qkv=qkv, launch_rows=0)
        a.update(kw)
        rows, H = a["qkv"].shape[0], a["qkv"].shape[1] // 3
        with pytest.raises(VttsError) as e:
            eng.debug_t2s_prefix_attn(a["T"], a["P"], a["heads"], a["qkv"], np.zeros((rows, H), np.float32), launch_rows=a["launch_rows"])
        assert e.value.code == -1, kw


# ------------------------------------------------------------------------------------------------ exact kernels
BLOCKS = ["SMALL", "D96", "D128", "UPSTREAM"]


def _tables(m):
    from vosk_tts_b200 import weights
    blob, man = weights.pack_t2s(m[1], m[2], tc=False)
    H = m[2]["cv_hidden"]
    tb = lambda n: A.blob_tensor(blob, man, n)
    at, aa = tb("t2s.alpha")
    return tb("t2s.temb").reshape(-1, H), tb("t2s.aemb").reshape(-1, H), tb("t2s.pe").reshape(-1, H), at, aa


@pytest.mark.parametrize("with_bert", [False, True])
@pytest.mark.parametrize("block", BLOCKS)
def test_embed(block, with_bert):
    m = _t2s(block)
    eng, sd, cfg = m
    eng = eng.engine
    H = cfg["cv_hidden"]
    temb, aemb, pe, at, aa = _tables(m)
    pairs = R.ragged_pairs(24, 5)[:20] + [(1, 0), (4, 4), (200, 600), (1, 7)]
    T, P = _tp(pairs)
    offs, tot = R.offsets(T, P)
    r = np.random.default_rng(9)
    ids = np.full(tot + 8, -1, np.int32)
    for b, (Tb, Pb) in enumerate(pairs):
        ids[offs[b]:offs[b] + Tb] = r.integers(0, temb.shape[0], Tb)
        ids[offs[b] + Tb:offs[b] + Tb + Pb] = r.integers(0, aemb.shape[0], Pb)
    ids[ids < 0] = 0
    bp = r.standard_normal((tot + 8, H)).astype(np.float32) if with_bert else None
    x0 = np.full((tot + 8, H), SENT, np.float32)
    p0 = np.full((tot + 8, H), PSENT, np.uint16)
    x, hi, lo = eng.debug_t2s_embed(T, P, ids, x0, bert_proj=bp, hi=p0, lo=p0)
    want = R.embed(ids, T, P, temb, aemb, pe, at, aa, x0, bp=bp, bp_bias=sd["bert_proj.bias"].numpy())
    assert np.array_equal(x.view(np.uint32), want.view(np.uint32))
    inside = R.rows_of(T, P)
    outside = np.setdiff1d(np.arange(tot + 8), inside)
    sh, sl = CR.split_bf16(x[inside])
    assert np.array_equal(hi[inside], sh) and np.array_equal(lo[inside], sl)
    assert np.all(hi[outside] == PSENT) and np.all(lo[outside] == PSENT)
    x2, _, _ = eng.debug_t2s_embed(T, P, ids, x0, bert_proj=bp)          # without planes: the same rows
    assert np.array_equal(x2.view(np.uint32), x.view(np.uint32))


def test_embed_refusals():
    from vosk_tts_b200.engine import VttsError
    eng, sd, cfg = _t2s("SMALL")
    eng = eng.engine
    PV, V, npos = cfg["t2s_phone_vocab"], cfg["t2s_vocab"], cfg["t2s_positions"]
    for T, P, bad_row, bad_id in [([2], [1], 0, PV), ([2], [1], 2, V), ([2], [1], 1, -1), ([npos + 1], [0], 0, 0), ([1], [npos + 1], 0, 0)]:
        _, tot = R.offsets(T, P)
        ids = np.zeros(tot, np.int32)
        ids[bad_row] = bad_id
        with pytest.raises(VttsError) as e:
            eng.debug_t2s_embed(T, P, ids, np.zeros((tot, cfg["cv_hidden"]), np.float32))
        assert e.value.code == -1


@pytest.mark.parametrize("block", BLOCKS)
def test_relu(block):
    eng, sd, cfg = _t2s(block)
    eng = eng.engine
    F = cfg["cv_ffn"]
    lens = [1, 7, 8, 9, 33, 600]
    offs = CR.offsets(lens)
    rows = offs[-1] + lens[-1] + 5
    y = np.random.default_rng(2).standard_normal((rows, F)).astype(np.float32)
    inside = np.concatenate([np.arange(o, o + n) for o, n in zip(offs, lens)])
    want = R.relu(y, inside)
    got, _, _ = eng.debug_act("relu", lens, y)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    p0 = np.full(y.shape, PSENT, np.uint16)
    same, hi, lo = eng.debug_act("relu", lens, y, hi=p0, lo=p0)
    assert np.array_equal(same.view(np.uint32), y.view(np.uint32))                # planes only: y untouched
    sh, sl = CR.split_bf16(want[inside])
    assert np.array_equal(hi[inside], sh) and np.array_equal(lo[inside], sl)
    outside = np.setdiff1d(np.arange(rows), inside)
    assert np.all(hi[outside] == PSENT) and np.all(lo[outside] == PSENT)


@pytest.mark.parametrize("block", BLOCKS)
def test_cache_and_state(block):
    eng, sd, cfg = _t2s(block)
    eng = eng.engine
    H, V = cfg["cv_hidden"], cfg["t2s_vocab"]
    nw = (V + 31) // 32
    pairs = [(5, 0), (1, 9), (17, 40), (8, 0), (3, 5), (30, 33), (2, 1), (12, 20), (1, 0), (64, 64), (7, 600), (9, 3)]
    T, P = _tp(pairs)
    B = len(pairs)
    offs, tot = R.offsets(T, P)
    r = np.random.default_rng(4)
    rows = tot + 8
    qkv = r.standard_normal((rows, 3 * H)).astype(np.float32)
    pre = r.standard_normal((rows, H)).astype(np.float32)
    prompts = []
    for b, Pb in enumerate(P):
        p = r.integers(0, V - 1, Pb)
        if Pb >= 6:                                   # repeats, both sides of a word edge, and the last token below EOS
            p[:6] = [31, 32, V - 2, 31, 0, V - 2]
        prompts.append(p)
    prompts = np.concatenate(prompts).astype(np.int32)
    # cache regions of T + P + 3 rows (room for decode steps) and token regions, neither in row order
    sizes = np.array([t + p + 3 for t, p in pairs])
    order = r.permutation(B)
    kv_off = np.zeros(B, np.int32)
    kv_off[order] = np.concatenate([[0], np.cumsum(sizes[order])[:-1]]) + 5
    kv_rows = int(sizes.sum()) + 11
    ysz = np.array(P) + 2
    order = r.permutation(B)
    y_off = np.zeros(B, np.int32)
    y_off[order] = np.concatenate([[0], np.cumsum(ysz[order])[:-1]]) + 3
    y_len = int(ysz.sum()) + 7
    kc0 = np.full((kv_rows, H), SENT, np.float32)
    vc0 = np.full((kv_rows, H), -SENT, np.float32)
    y0 = np.full(y_len, -5, np.int32)
    st0 = np.full((B, 8), 77, np.int32)
    seen0 = np.full(B * nw + 5, 0xDEADBEEF, np.uint32)      # five words behind the B rows, which must be kept
    hx0 = np.full((B, H), SENT, np.float32)
    got = eng.debug_t2s_state(T, P, qkv, pre, prompts, kv_off, kc0, vc0, y_off, y0, st0, seen0, hx0)
    kc, vc = R.kv_store(qkv, T, P, kv_off, kc0, vc0)
    st, y, seen, hx = R.init(T, P, kv_off, y_off, prompts, pre, V, y0, hx0)
    assert np.array_equal(got["kc"].view(np.uint32), kc.view(np.uint32))
    assert np.array_equal(got["vc"].view(np.uint32), vc.view(np.uint32))
    assert np.array_equal(got["state"], st)
    assert np.array_equal(got["y"], y)
    assert np.array_equal(got["seen"][:B * nw].reshape(B, nw), seen)
    assert np.all(got["seen"][B * nw:] == 0xDEADBEEF)
    assert np.array_equal(got["hx"].view(np.uint32), hx.view(np.uint32))
    if V % 32:                                        # no bit at or above V in the last word
        assert np.all(seen[:, -1] >> np.uint32(V % 32) == 0)
    # refusals: a prompt token at EOS, a cache region or a token region past its end or over another, a short seen
    from vosk_tts_b200.engine import VttsError
    bad_prompts = prompts.copy()
    bad_prompts[0] = V - 1
    bad_kv = kv_off.copy()
    bad_kv[0] = kv_rows - (T[0] + P[0]) + 1              # one row past the caches
    bad_y = y_off.copy()
    bad_y[1] = y_len - P[1] + 1                           # one slot past y
    over_kv = kv_off.copy()
    over_kv[2] = kv_off[5] + 1                      # utterance 2's 57 cache rows inside utterance 5's 66-row region
    over_y = y_off.copy()
    over_y[5] = y_off[2]                            # utterance 5's 33 token slots inside utterance 2's 42
    cases = [("prompt token", bad_prompts, kv_off, y_off, seen0), ("pass kv_rows", prompts, bad_kv, y_off, seen0),
             ("pass y_len", prompts, kv_off, bad_y, seen0), ("overlap", prompts, over_kv, y_off, seen0),
             ("overlap", prompts, kv_off, over_y, seen0), ("seen holds fewer", prompts, kv_off, y_off, seen0[:B * nw - 1])]
    for what, pr, ko, yo, sn in cases:
        try:
            eng.debug_t2s_state(T, P, qkv, pre, pr, ko, kc0, vc0, yo, y0, st0, sn, hx0)
        except VttsError as e:
            assert e.code == -1 and what in str(e), (what, str(e))
        else:
            pytest.fail("%s: accepted" % what)


# ------------------------------------------------------------------------------------------------ the composed prefill
def _composed(block, precision, pairs, seed):
    m, sd, cfg = _t2s(block, precision)
    eng = m.engine
    phs = [TI.phones(cfg, t, seed + b) for b, (t, p) in enumerate(pairs)]
    prs = [TI.prompt(cfg, p, seed + 500 + b) for b, (t, p) in enumerate(pairs)]
    q = np.stack([TI.q_draws(cfg, 2, seed + 900 + b) for b in range(len(pairs))])
    toks, idx, lg = eng.t2s_decode(phs, prs, q=q, step_cap=2, logits_steps=2)
    errs = []
    for b, (t, p) in enumerate(pairs):
        assert len(toks[b]) == p + 1
        assert np.all(np.isfinite(lg[b])), b
        ref = O.step_logits(sd, cfg, phs[b], toks[b], P=p).numpy()
        errs.append(np.abs(lg[b] - ref).max())
        t1, _, l1 = eng.t2s_decode([phs[b]], [prs[b]], q=q[b:b + 1], step_cap=2, logits_steps=2)
        assert np.array_equal(t1[0], toks[b]) and np.array_equal(l1[0].view(np.uint32), lg[b].view(np.uint32)), b
    err = float(np.max(errs))                                  # (a NaN stays NaN and fails below)
    print("composed prefill %s mode %d, %d utterances up to T + P = %d: max logit error %.3g (budget %g)" %
          (block, precision, len(pairs), max(t + p for t, p in pairs), err, BUDGET[precision]))
    assert err < BUDGET[precision], err


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("block", ["SMALL", "D128"])
def test_composed_prefill_at_real_lengths(block, precision):
    r = np.random.default_rng(21)
    pairs = [(512, 600), (1, 0), (150, 450), (33, 600), (500, 1), (7, 150)]
    while len(pairs) < 64:
        pairs.append((int(r.integers(1, 513)), int(r.integers(0, 601))))
    _composed(block, precision, pairs, 40)


@pytest.mark.parametrize("precision", [0, 1])
def test_composed_prefill_upstream_width(precision):
    _composed("UPSTREAM", precision, [(150, 450)], 70)


def test_engines_of_other_widths_coexist():
    """Binding an engine with a narrower FFN must not break the decode of a wider engine bound before it (t2s_ffn2_kernel's
    shared-memory attribute belongs to the kernel, not to an engine).  The wide engine's second call has a new shape, so its
    decode steps are captured after the narrow engine was bound."""
    from vosk_tts_b200.gpt_sovits import Text2Semantic
    m, sd, cfg = _t2s("D128")
    q = TI.q_draws(cfg, 3, 2)[None]
    m.engine.t2s_decode([TI.phones(cfg, 9, 1)], q=q, step_cap=3, logits_steps=2)
    narrow = Text2Semantic(TI.model(TI.SMALL), precision=0)
    try:
        ph = TI.phones(cfg, 14, 3)
        toks, idx, lg = m.engine.t2s_decode([ph], q=q, step_cap=3, logits_steps=2)
    finally:
        narrow.close()
    ref = O.step_logits(sd, cfg, ph, toks[0][:1]).numpy()
    assert np.all(np.isfinite(lg[0])) and np.abs(lg[0] - ref).max() < BUDGET[0]
