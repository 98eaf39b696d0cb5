"""The GPT-SoVITS text prefill's references on the CPU: attn_ref's prefix mode and t2s_prefill_ref's embedding rows restate
oracle/t2s_oracle.py (infer_panel in float64), an fp32 emulation of t2s_prefix_attn_kernel's chunked arithmetic meets the
bound, and planted defects on the inputs tests/test_gpu_t2s_prefill.py runs break the bound or exactness."""
import numpy as np
import pytest
import torch

import attn_ref as A
import t2s_inputs as TI
import t2s_prefill_ref as R
from oracle import t2s_oracle as O
from vosk_tts_b200 import weights

SMALL_PAIRS = R.EDGE_PAIRS + [(120, 450), (8, 0), (3, 13)]


def _offs(pairs):
    return R.offsets([p[0] for p in pairs], [p[1] for p in pairs])[0]


@pytest.mark.parametrize("heads,dk", [(2, 32), (1, 64), (2, 96), (1, 128)])
def test_prefix_reference_is_the_oracle(heads, dk):
    """attn_ref.reference(T=...) in float64 equals the oracle's masked attention on the same (pre-scaled) operands."""
    pairs = [(1, 0), (5, 27), (33, 0), (30, 3), (40, 70)]
    T = [p[0] for p in pairs]
    qkv = R.attn_qkv(pairs, heads, dk, "random", 1)
    lens = [t + p for t, p in pairs]
    res = A.reference(qkv, lens, heads, 0, None, "ffma", T=T, offs=_offs(pairs))
    H = heads * dk
    s32 = float(np.float32(np.sqrt(1.0 / dk)))
    for (rows, ref, bnd), Tb in zip(res, T):
        x = qkv[rows].astype(np.float64)
        # the kernel's q: fp32 q * fp32 sqrt(1 / dk); handed to the oracle so that its q * sqrt(1 / dk) is that product
        x[:, :H] = (qkv[rows, :H] * np.float32(s32)).astype(np.float64) / np.sqrt(1.0 / dk)
        o = O.prefix_attention(torch.from_numpy(x), Tb, heads).numpy()
        assert np.abs(o - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
        assert np.all(bnd > 0) and np.all(np.isfinite(bnd))


@pytest.mark.parametrize("with_bert", [False, True])
def test_embed_reference_is_the_oracle(with_bert):
    sd, cfg = TI.model(TI.SMALL)
    blob, man = weights.pack_t2s(sd, cfg, tc=False)
    tb = lambda n: A.blob_tensor(blob, man, n)
    H = cfg["cv_hidden"]
    temb, aemb, pe = tb("t2s.temb").reshape(-1, H), tb("t2s.aemb").reshape(-1, H), tb("t2s.pe").reshape(-1, H)
    at, aa = tb("t2s.alpha")
    pairs = [(7, 0), (12, 9), (1, 31)]
    T, P = [p[0] for p in pairs], [p[1] for p in pairs]
    offs, tot = R.offsets(T, P)
    r = np.random.default_rng(3)
    ids = np.zeros(tot, np.int32)
    bp = np.zeros((tot, H), np.float32)
    berts = []
    for b, (Tb, Pb) in enumerate(pairs):
        ids[offs[b]:offs[b] + Tb] = TI.phones(cfg, Tb, b)
        ids[offs[b] + Tb:offs[b] + Tb + Pb] = TI.prompt(cfg, Pb, 10 + b)
        bert = r.standard_normal((Tb, 1024)).astype(np.float32)
        berts.append(bert)
        bp[offs[b]:offs[b] + Tb] = (bert.astype(np.float64) @ sd["bert_proj.weight"].double().numpy().T + sd["bert_proj.bias"].double().numpy())
    x = R.embed(ids, T, P, temb, aemb, pe, at, aa, np.zeros((tot, H), np.float32), bp=bp if with_bert else None,
                bp_bias=sd["bert_proj.bias"].numpy())
    w = {k: v.double() for k, v in sd.items()}
    for b, (Tb, Pb) in enumerate(pairs):
        o = O.embed(w, cfg, ids[offs[b]:offs[b] + Tb], ids[offs[b] + Tb:offs[b] + Tb + Pb], berts[b] if with_bert else None).numpy()
        got = x[offs[b]:offs[b] + Tb + Pb].astype(np.float64)
        # three fp32 roundings of operands of the sizes below (and bp's own rounding to fp32)
        mag = np.abs(o) + np.abs(np.concatenate([temb[ids[offs[b]:offs[b] + Tb]], aemb[ids[offs[b] + Tb:offs[b] + Tb + Pb]]]))
        mag = mag + np.abs(np.concatenate([at * pe[:Tb], aa * pe[:Pb]]))
        assert np.all(np.abs(got - o) <= 4 * 2.0 ** -24 * (mag + np.abs(bp[offs[b]:offs[b] + Tb + Pb]).max())), b


def _emulation_ratio(pairs, heads, dk, pattern, corrupt=(), seed=2):
    T = [p[0] for p in pairs]
    lens = [t + p for t, p in pairs]
    offs = _offs(pairs)
    qkv = R.attn_qkv(pairs, heads, dk, pattern, seed)
    out, _ = A.f32_attention(qkv, lens, heads, 0, None, None, T=T, offs=offs, corrupt=corrupt)
    res = A.reference(qkv, lens, heads, 0, None, "ffma", T=T, offs=offs)
    return A.worst(out, res)


@pytest.mark.parametrize("pattern", ["random", "rising", "large", "equal"])
@pytest.mark.parametrize("heads,dk", [(2, 32), (1, 128)])
def test_fp32_emulation_meets_the_bound(pattern, heads, dk):
    w = _emulation_ratio(SMALL_PAIRS, heads, dk, pattern)
    print("prefix attention fp32 emulation %s dk %d: worst error / bound %.3f" % (pattern, dk, w))
    assert w <= 1.0


@pytest.mark.parametrize("corrupt,pattern", [("self", "random"), ("text_sees_prompt", "random"), ("no_rescale", "rising"),
                                             ("no_max", "large")])
def test_planted_attention_defects_break_the_bound(corrupt, pattern):
    w = _emulation_ratio(SMALL_PAIRS, 2, 32, pattern, corrupt=(corrupt,))
    print("prefix attention with %s: worst error / bound %.3g" % (corrupt, w))
    assert w > 1.0


def test_worst_reports_non_finite_outputs():
    """A NaN or inf output is never within the bound: worst() returns inf for it."""
    pairs = [(5, 27), (3, 0)]
    T = [p[0] for p in pairs]
    lens = [t + p for t, p in pairs]
    offs = _offs(pairs)
    qkv = R.attn_qkv(pairs, 1, 32, "random", 5)
    res = A.reference(qkv, lens, 1, 0, None, "ffma", T=T, offs=offs)
    out, _ = A.f32_attention(qkv, lens, 1, 0, None, None, T=T, offs=offs)
    assert A.worst(out, res) <= 1.0
    for bad in (np.nan, np.inf):
        o = out.copy()
        o[offs[1] + 2, 7] = bad
        assert A.worst(o, res) == float("inf")


def test_mask_probe_separates_the_planted_defects():
    """The GPU test's probe rows: with the marker at the first prompt position a prompt row that loses itself shows no marker
    where it must be dominated by it."""
    pairs = [(5, 27), (30, 3), (1, 1)]
    T = [p[0] for p in pairs]
    lens = [t + p for t, p in pairs]
    offs = _offs(pairs)
    qkv, keys = R.attn_qkv(pairs, 2, 32, "random", 4, probe="first_prompt")
    good, _ = A.f32_attention(qkv, lens, 2, 0, None, None, T=T, offs=offs)
    bad, _ = A.f32_attention(qkv, lens, 2, 0, None, None, T=T, offs=offs, corrupt=("self",))
    for b, (Tb, Pb) in enumerate(pairs):
        row = offs[b] + keys[b]
        assert good[row, 0] > 0.9e4 and bad[row, 0] < 1e3


def _embed_case():
    sd, cfg = TI.model(TI.SMALL)
    blob, man = weights.pack_t2s(sd, cfg, tc=False)
    tb = lambda n: A.blob_tensor(blob, man, n)
    H = cfg["cv_hidden"]
    tabs = dict(temb=tb("t2s.temb").reshape(-1, H), aemb=tb("t2s.aemb").reshape(-1, H), pe=tb("t2s.pe").reshape(-1, H))
    at, aa = tb("t2s.alpha")
    pairs = [(7, 0), (12, 9), (1, 31)]
    T, P = [p[0] for p in pairs], [p[1] for p in pairs]
    offs, tot = R.offsets(T, P)
    ids = np.zeros(tot, np.int32)
    for b, (Tb, Pb) in enumerate(pairs):
        ids[offs[b]:offs[b] + Tb] = TI.phones(cfg, Tb, b)
        ids[offs[b] + Tb:offs[b] + Tb + Pb] = TI.prompt(cfg, Pb, 10 + b)
    return ids, T, P, tabs, at, aa, np.zeros((tot, H), np.float32), sd["bert_proj.bias"].numpy()


@pytest.mark.parametrize("corrupt", ["swap_alpha", "prompt_pe_t"])
def test_planted_embed_defects_break_exactness(corrupt):
    ids, T, P, tabs, at, aa, x, bias = _embed_case()
    assert at != aa
    good = R.embed(ids, T, P, tabs["temb"], tabs["aemb"], tabs["pe"], at, aa, x, bp_bias=bias)
    bad = R.embed(ids, T, P, tabs["temb"], tabs["aemb"], tabs["pe"], at, aa, x, bp_bias=bias, corrupt=(corrupt,))
    assert not np.array_equal(good, bad)


def test_planted_hx_defect_breaks_exactness():
    T, P = [3, 4], [5, 0]
    offs, tot = R.offsets(T, P)
    pre = np.random.default_rng(0).standard_normal((tot, 8)).astype(np.float32)
    args = (T, P, [0, 8], [0, 5], np.arange(5), pre, 65, np.zeros(5, np.int32), np.zeros((2, 8), np.float32))
    good = R.init(*args)[3]
    bad = R.init(*args, corrupt=("hx_text",))[3]
    assert not np.array_equal(good[0], bad[0]) and np.array_equal(good[1], bad[1])     # P = 0: row T - 1 is row T + P - 1
