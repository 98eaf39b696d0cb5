"""GPU (-m gpu): the dense conv kernels in isolation -- conv_tc_kernel / conv_tc_persist_kernel (csrc/conv_tc.cuh) and the fp32
FFMA conv_kernel<G> (csrc/kernels.cuh) -- one grouped launch at a time through the engine's own launch code
(vtts_debug_conv), against the float64 reference and error bound of tests/conv_ref.py:
  tensor cores   operand-exact emulation of the products the kernel issues; bound = fp32 accumulation alone
  FFMA           exact conv of the fp32 operands; bound = fp32 accumulation of Cin*k products
Every case pins the launch shape it is meant to exercise with per-call overrides and asserts that the engine reports that
shape, so a change of the launch heuristics cannot quietly move it onto another path.  Every case also checks that output
rows outside each utterance (gap rows included) keep the sentinel written beforehand, that output planes equal the device
split of lrelu(y) bit for bit, and that a second launch is bit-identical (split-K and the FFMA reductions sum in a fixed
order).  The tensor-core input planes carry finite garbage in the gap rows between utterances: the engine's zero_tails pass,
not the test, must clear what a conv halo reads."""
import zlib

import numpy as np
import pytest
import torch

import conv_ref as cr
from vosk_tts_b200 import weights

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
PSENT = np.uint16(0x7E7E)


@pytest.fixture(scope="module")
def eng(packed, cfg):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    yield e
    e.close()


def _prob(**kw):
    q = dict(Cin=64, Cout=64, k=1, dil=1, pad=0, out_mul=1, out_add=0, in_extra=0, out_seq_extra=0, epi=0, alpha=1.0,
             pl_slope=1.0, y_on=1, ldy=None, yoff=0, res=0, ldr=None, roff=0, planes_on=0, ldp=None, poff=0, cond=False)
    q.update(kw)
    ncol = q["Cout"] // 2 if q["epi"] & cr.EPI_GATE else q["Cout"]
    q["ldy"] = q["ldy"] or q["yoff"] + ncol
    q["ldr"] = q["ldr"] or q["ldy"]
    q["ldp"] = q["ldp"] or q["poff"] + ncol
    return q


def _rows_needed(q, lens, rmul):
    offs = cr.offsets(lens)
    return max(offs[b] * rmul * q["out_mul"] + b * q["out_seq_extra"] + (n * rmul + q["in_extra"] - 1) * q["out_mul"]
               + q["out_add"] for b, n in enumerate(lens)) + 1


def run_case(eng, kind, lens, rmul, probs, expect, ov=None, n_planes=2, p_planes=2, seed=0, x_override=None):
    """One launch (twice, for determinism), checked against conv_ref.  Returns the launch report."""
    rng = np.random.default_rng(seed)
    B = len(lens)
    offs = cr.offsets(lens)
    Cin = probs[0]["Cin"]
    # ---- input
    if kind == "tc":
        extra = probs[0]["in_extra"]
        rows = offs[-1] * rmul + B * extra
        x = rng.uniform(-40.0, 40.0, (rows, Cin)).astype(np.float32)           # finite garbage: gap rows keep it
        for b, n in enumerate(lens):
            r0 = offs[b] * rmul + b * extra
            x[r0:r0 + n * rmul + extra] = rng.standard_normal((n * rmul + extra, Cin))
        if x_override is not None:
            x = x_override
        xin = cr.split_planes(x, n_planes)
        ins = cr.tc_inputs(xin, lens, rmul, extra)
    else:
        ldx = max(q.get("ldx", Cin) for q in probs)
        rows = offs[-1] * rmul + 2
        xin = rng.standard_normal(rows * ldx).astype(np.float32)
    # ---- weights, biases, cond
    specs, refw = [], []
    for q in probs:
        w = (rng.standard_normal((q["Cout"], q["Cin"], q["k"])) / np.sqrt(q["Cin"] * q["k"])).astype(np.float32)
        bias = (0.1 * rng.standard_normal(q["Cout"])).astype(np.float32)
        cond = (0.5 * rng.standard_normal((B, q["Cout"] + 3))).astype(np.float32) if q["cond"] else None
        s = {k: v for k, v in q.items() if k not in ("cond",)}
        s["cond"], s["cond_ld"] = cond, (q["Cout"] + 3 if cond is not None else 0)
        if kind == "tc":
            wp = weights.conv_tc_planes(w) if n_planes == 2 else weights.conv_tc3_planes(w)
            s["w_hi"], s["w_lo"] = wp[0], wp[-1]
            if n_planes == 3:
                s["w_mid"] = wp[1]
            s["bias"] = bias
            wpl = np.stack([cr.bf16_value(p).transpose(1, 2, 0) for p in wp])
        else:
            s["w"], s["bias"] = weights.conv_ffma_layout(w, bias)
            wpl = None
        specs.append(s)
        refw.append((w, bias, cond, wpl))
    # ---- output buffers: sentinels, residuals
    ny = max((_rows_needed(q, lens, rmul) + 3) * max(q["ldy"], q["ldr"]) for q in probs)
    y0 = np.full(ny, SENT, np.float32)
    res0 = None
    for i, q in enumerate(probs):
        if q["res"] == 1:
            res0 = rng.standard_normal(ny).astype(np.float32) if res0 is None else res0
        if q["res"] == 2:                                   # in place: the residual is what y holds in this problem's rows
            ncol = q["Cout"] // 2 if q["epi"] & cr.EPI_GATE else q["Cout"]
            for b, n in enumerate(lens):
                L = n * rmul + q["in_extra"]
                r = offs[b] * rmul * q["out_mul"] + b * q["out_seq_extra"] + np.arange(L) * q["out_mul"] + q["out_add"]
                idx = (r[:, None] * q["ldr"] + q["roff"] + np.arange(ncol)[None, :]).reshape(-1)
                y0[idx] = rng.standard_normal(idx.size)
    pn = max((_rows_needed(q, lens, rmul) + 3) * q["ldp"] for q in probs)
    any_planes = any(q["planes_on"] for q in probs)
    p0 = np.full((p_planes, pn), PSENT, np.uint16) if any_planes else None
    # ---- run twice
    outs = [eng.debug_conv(kind == "tc", lens, rmul, specs, xin, y=y0, res=res0, planes=p0, overrides=ov) for _ in range(2)]
    (y, pl, rep), (y2, pl2, rep2) = outs
    assert rep == rep2
    for key, v in expect.items():
        assert rep[key] == v, "launch shape: %s = %d, expected %d (report %s)" % (key, rep[key], v, rep)
    assert np.array_equal(y.view(np.uint32), y2.view(np.uint32)), "two launches differ"
    if any_planes:
        assert np.array_equal(pl, pl2), "two launches differ (planes)"
    # ---- reference
    ymask = np.zeros(ny, bool)
    pmask = np.zeros(pn, bool)
    for i, q in enumerate(probs):
        w, bias, cond, wpl = refw[i]
        qi = ins if kind == "tc" else cr.ffma_inputs(xin, lens, rmul, q)
        resbuf = y0 if q["res"] == 2 else res0
        res = cr.reference(kind, q, w, bias, lens, rmul, qi, n_planes, wpl, cond=cond, res_buf=resbuf)
        if q["y_on"]:
            exp, bnd, m = cr.scatter(res, ny, q["ldy"], q["yoff"])
            assert not (ymask & m).any()
            ymask |= m
            err = np.abs(y[m].astype(np.float64) - exp[m])
            bad = ~(err <= bnd[m])
            assert not bad.any(), "problem %d: %d of %d outputs outside the bound (max err %.3e, bound there %.3e)" % (
                i, bad.sum(), m.sum(), err.max(), bnd[m][np.argmax(err - bnd[m])])
        if q["planes_on"]:
            exp, bnd, m = cr.scatter(res, pn, q["ldp"], q["poff"])
            pmask |= m
            idx = np.flatnonzero(m)
            if q["y_on"]:                                    # planes are the device split of lrelu(y) bit for bit
                _, _, my = cr.scatter(res, ny, q["ldy"], q["yoff"])
                want = cr.split_planes(cr.lrelu32(y[my], q["pl_slope"]), p_planes)
                assert np.array_equal(pl[:, idx], want), "problem %d: output planes != split(lrelu(y))" % i
            else:
                got = sum(cr.bf16_value(pl[j, idx]) for j in range(p_planes))
                e = exp[m]
                want = np.where(e > 0, e, e * q["pl_slope"])
                tol = bnd[m] * max(1.0, abs(q["pl_slope"])) + 2.0 ** -15 * np.abs(want)
                assert np.all(np.abs(got - want) <= tol), "problem %d: output planes" % i
    assert np.array_equal(y[~ymask].view(np.uint32), y0[~ymask].view(np.uint32)), "rows outside the utterances were written"
    if any_planes:
        assert np.all(pl[:, ~pmask] == PSENT), "plane rows outside the utterances were written"
    return rep


TC_DEFAULT = dict(tc_bn=64, tc_split=1, tc_persist=0, tc_tall=-1, tc_mc=0, tc_wmc=0)


def _ov(**kw):
    o = dict(TC_DEFAULT)
    o.update(kw)
    return o


# ------------------------------------------------------------------------------------------------ tensor-core launch modes
TC_MODES = {
    # name: (overrides, expected report, lens, rmul, problems, n_planes)
    "bn64-one-tile-per-cta": (_ov(), dict(bn=64, split=1, tall=0, cn=1, persist=0, np=2, image=0, grid_y=3),
                              [300], 1, [_prob(Cin=192, Cout=192, k=5, pad=2, cond=True)], 2),
    "bn128-wn-in-gated": (_ov(tc_bn=128), dict(bn=128, split=1, persist=0, image=0, grid_y=3),
                          [300], 1, [_prob(Cin=192, Cout=384, k=5, pad=2, epi=cr.EPI_GATE, cond=True)], 2),
    "split2-bn64": (_ov(tc_split=2, tc_min_steps=1), dict(bn=64, split=2, cn=1, image=0, grid_z=2),
                    [200], 1, [_prob(Cin=512, Cout=96, k=3, pad=1)], 2),
    "split4-bn64": (_ov(tc_split=4, tc_min_steps=1), dict(bn=64, split=4, image=0, grid_z=4),
                    [130], 1, [_prob(Cin=192, Cout=192, k=3, pad=1, epi=cr.EPI_RELU, alpha=0.5)], 2),
    "split8-bn128-cout96": (_ov(tc_bn=128, tc_split=8, tc_min_steps=1), dict(bn=128, split=8, image=0, grid_z=8),
                            [200], 1, [_prob(Cin=512, Cout=96, k=3, pad=1, cond=True)], 2),
    "persistent-per-tap-ragged": (_ov(tc_persist=2), dict(persist=1, tall=0, wmc=1, image=2, grid_y=1, grid_z=1),
                                  [1, 5, 300, 64, 2], 1, [_prob(Cin=192, Cout=192, k=5, pad=2, epi=cr.EPI_GATE, cond=True)], 2),
    "persistent-tall-ragged": (_ov(tc_persist=2, tc_tall=1), dict(persist=1, tall=1, image=2, ast=2),
                               [1, 129, 3, 257], 1, [_prob(Cin=192, Cout=192, k=5, pad=2)], 2),
    "persistent-tall-mrf-group": (_ov(tc_persist=2, tc_tall=1), dict(persist=1, tall=1, image=2),
                                  [1, 7, 40], 4, [_prob(Cin=128, Cout=128, k=3, dil=1, pad=1, ldy=384, yoff=0),
                                                  _prob(Cin=128, Cout=128, k=7, dil=3, pad=9, ldy=384, yoff=128),
                                                  _prob(Cin=128, Cout=128, k=11, dil=5, pad=25, ldy=384, yoff=256)], 2),
    "persistent-wmc-odd-row-tiles": (_ov(tc_persist=2, tc_wmc=1), dict(persist=1, wmc=2, image=2),
                                     [300, 40], 1, [_prob(Cin=192, Cout=384, k=5, pad=2, epi=cr.EPI_GATE, cond=True)], 2),
    "persistent-wmc-tall": (_ov(tc_persist=2, tc_wmc=1, tc_tall=1), dict(persist=1, wmc=2, tall=1, image=2),
                            [129, 1, 385], 1, [_prob(Cin=192, Cout=192, k=3, pad=1)], 2),
    "multicast-cn2": (_ov(tc_mc=1), dict(cn=2, split=1, persist=0, image=0),
                      [200, 3, 129], 1, [_prob(Cin=192, Cout=384, k=3, pad=1, cond=True)], 2),
    "multicast-cn4": (_ov(tc_mc=1), dict(cn=4, split=1, persist=0, image=0),
                      [200, 3, 129], 1, [_prob(Cin=192, Cout=256, k=3, pad=1, epi=cr.EPI_RELU)], 2),
    "np3-single-wave": (_ov(), dict(np=3, image=1, persist=0, split=1, ast=2),
                        [1, 150], 1, [_prob(Cin=192, Cout=576, k=1)], 3),
    "np3-split2": (_ov(tc_split=2, tc_min_steps=1), dict(np=3, image=1, split=2),
                   [150], 1, [_prob(Cin=192, Cout=192, k=3, pad=1, epi=cr.EPI_RELU)], 3),
    "np3-persistent": (_ov(tc_persist=2, tc_tall=1), dict(np=3, image=2, persist=1, tall=0),
                       [5, 200, 1], 1, [_prob(Cin=192, Cout=192, k=3, pad=1, epi=cr.EPI_RELU)], 3),
    "tall-fallback-wide-halo": (_ov(tc_persist=2, tc_tall=1), dict(persist=1, tall=0, image=2),
                                [300], 1, [_prob(Cin=64, Cout=64, k=11, dil=7, pad=35)], 2),
}


@pytest.mark.parametrize("name", list(TC_MODES))
def test_tc_launch_modes(eng, name):
    ov, expect, lens, rmul, probs, n_planes = TC_MODES[name]
    run_case(eng, "tc", lens, rmul, probs, expect, ov=ov, n_planes=n_planes, seed=zlib.crc32(name.encode()))


@pytest.mark.parametrize("L", [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000])
@pytest.mark.parametrize("mode", ["one-tile-per-cta", "persistent-tall"])
def test_tc_lengths(eng, L, mode):
    ov = _ov() if mode == "one-tile-per-cta" else _ov(tc_persist=2, tc_tall=1)
    expect = dict(persist=0, image=0) if mode == "one-tile-per-cta" else dict(persist=1, tall=1, image=2)
    run_case(eng, "tc", [L], 1, [_prob(Cin=64, Cout=72, k=7, pad=3)], expect, ov=ov, seed=L)


@pytest.mark.parametrize("rmul", [1, 4, 16])
def test_tc_ragged_batches_and_rmul(eng, rmul):
    lens = [1, 3, 17, 64, 129, 2, 40, 1][: 8 if rmul == 1 else 5]
    run_case(eng, "tc", lens, rmul, [_prob(Cin=64, Cout=96, k=5, pad=2, cond=True, epi=cr.EPI_RELU)],
             dict(persist=1, tall=1), ov=_ov(tc_persist=2, tc_tall=1), seed=rmul)


def test_tc_polyphase_convtranspose_group(eng):
    """The four polyphase branches of a ConvTranspose1d(stride 4) in one launch: output row t*4 + r, planes for the next conv."""
    probs = [_prob(Cin=128, Cout=64, k=4, pad=p, out_mul=4, out_add=r, ldy=64, planes_on=1, ldp=64, pl_slope=0.1)
             for r, p in enumerate([2, 2, 1, 1])]
    run_case(eng, "tc", [2, 9, 1], 4, probs, dict(persist=0, image=0), ov=_ov(), seed=7)


def test_tc_wn_residual_pair_in_place(eng):
    """The WaveNet layer's res/skip pair: rsx adds into the residual stream, rss into the skip sum, both in place."""
    probs = [_prob(Cin=192, Cout=192, ldy=384, yoff=0, res=2, ldr=384, roff=0, planes_on=1, ldp=192),
             _prob(Cin=192, Cout=192, ldy=384, yoff=192, res=2, ldr=384, roff=192)]
    run_case(eng, "tc", [17, 1, 60], 1, probs, dict(persist=1, tall=1), ov=_ov(tc_persist=2, tc_tall=1), seed=8)


def test_tc_flow_post_in_place_negative_alpha(eng):
    """The flow's post conv: y = res = z with yoff = roff = half and alpha = -1 (reverse coupling)."""
    probs = [_prob(Cin=192, Cout=96, ldy=192, yoff=96, res=2, ldr=192, roff=96, alpha=-1.0)]
    run_case(eng, "tc", [33, 1, 128], 1, probs, dict(split=1, persist=0), ov=_ov(), seed=9)


@pytest.mark.parametrize("p_planes", [2, 3])
def test_tc_epilogues_scalar_store_and_planes(eng, p_planes):
    """Odd ldy / yoff (scalar stores), a separate residual, ReLU and alpha, planes of lrelu(out, 0.1) at an odd offset."""
    probs = [_prob(Cin=64, Cout=65, k=3, pad=1, ldy=67, yoff=1, res=1, ldr=69, roff=3, epi=cr.EPI_RELU, alpha=0.75, cond=True,
                   planes_on=1, ldp=67, poff=1, pl_slope=0.1)]
    run_case(eng, "tc", [5, 70], 1, probs, dict(persist=0), ov=_ov(), p_planes=p_planes, seed=10 + p_planes)
    probs = [_prob(Cin=64, Cout=128, k=3, pad=1, epi=cr.EPI_GATE, y_on=0, planes_on=1, ldp=64, pl_slope=0.2)]
    run_case(eng, "tc", [5, 70], 1, probs, dict(persist=1), ov=_ov(tc_persist=2), p_planes=p_planes, seed=20 + p_planes)


def test_tc_reflect_row_and_sequence_extra(eng):
    """conv_post-like: one extra logical input row per utterance (the reflection pad's) and one extra output row."""
    probs = [_prob(Cin=64, Cout=72, k=7, pad=3, in_extra=1, out_seq_extra=1)]
    run_case(eng, "tc", [3, 1, 20], 16, probs, dict(persist=0), ov=_ov(), seed=12)


def test_tc_stale_gap_rows_are_cleared(eng):
    """A long dense launch fills the input plane slot; a ragged launch through the same slot has garbage in its gap rows
    and must still see zeros in every halo (zero_tails_kernel under buffer reuse)."""
    q = [_prob(Cin=192, Cout=192, k=5, pad=2)]
    run_case(eng, "tc", [1000], 1, q, dict(persist=1), ov=_ov(tc_persist=2), seed=13)
    run_case(eng, "tc", [5, 300, 2, 1], 1, q, dict(persist=1), ov=_ov(tc_persist=2), seed=14)


@pytest.mark.parametrize("Cin,Cout,k,dil", [(64, 192, 3, 1), (192, 192, 5, 1), (512, 72, 7, 1), (192, 576, 1, 1),
                                            (128, 128, 11, 5), (64, 96, 3, 3)])
def test_tc_model_shapes_auto_launch(eng, Cin, Cout, k, dil):
    """Model shapes under the engine's own heuristics (no overrides): whatever shape they pick must be right."""
    run_case(eng, "tc", [1, 90, 300], 4 if (k - 1) * dil // 2 > 8 else 1,
             [_prob(Cin=Cin, Cout=Cout, k=k, dil=dil, pad=(k - 1) * dil // 2, cond=True)], {}, seed=Cin + Cout + k)


# ------------------------------------------------------------------------------------------------ FFMA kernel
@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("S", [1, 2, 4, 8])
def test_ffma_groups_and_split(eng, G, S):
    ov = dict(conv_min_g=G, conv_max_g=G, conv_big_g=G, conv_max_s=S)
    q = _prob(Cin=192, Cout=192, k=3, pad=1, ldx=192, cond=True, epi=cr.EPI_RELU)
    run_case(eng, "ffma", [100], 1, [q], dict(S=S, G=G), ov=ov, seed=G * 10 + S)


@pytest.mark.parametrize("Cin,Cout,k", [(16, 1, 3), (32, 2, 7), (192, 65, 3), (528, 192, 1), (16, 384, 5)])
def test_ffma_channel_counts(eng, Cin, Cout, k):
    q = _prob(Cin=Cin, Cout=Cout, k=k, pad=(k - 1) // 2, ldx=Cin)
    run_case(eng, "ffma", [1, 70, 3], 1, [q], {}, seed=Cin + Cout)


def test_ffma_reflect_prologue_and_tanh(eng):
    """conv_post of the HiFi-GAN decoder on the FFMA kernel: lrelu prologue, ReflectionPad1d((1,0)) row map, tanh."""
    q = _prob(Cin=32, Cout=4, k=7, pad=0, in_extra=1, reflect=1, pro=1, slope=0.01, ldx=32, epi=cr.EPI_TANH)
    run_case(eng, "ffma", [5, 20, 1], 16, [q], {}, seed=21)


def test_ffma_input_slices_gate_and_planes(eng):
    """ldx / xoff column slices of a wider input, gate with cond, planes (2 and 3) of the output, a grouped launch."""
    probs = [_prob(Cin=64, Cout=128, k=5, pad=2, ldx=256, xoff=64, ldy=128, epi=cr.EPI_GATE, cond=True, planes_on=1, ldp=64,
                   pl_slope=0.1),
             _prob(Cin=128, Cout=64, k=3, pad=1, ldx=256, xoff=128, ldy=128, yoff=64, res=2, ldr=128, roff=64, alpha=-1.0)]
    for p_planes in (2, 3):
        run_case(eng, "ffma", [2, 130, 1], 1, probs, {}, p_planes=p_planes, seed=22 + p_planes)


# ------------------------------------------------------------------------------------------------ refusals
def test_malformed_specs_are_refused_on_the_host(eng):
    from vosk_tts_b200.engine import VttsError
    x = cr.split_planes(np.ones((10, 64), np.float32), 2)
    w = weights.conv_tc_planes(np.ones((64, 64, 1), np.float32))
    ok = dict(_prob(), w_hi=w[0], w_lo=w[1], bias=np.zeros(64, np.float32), cond=None)
    y = np.zeros(10 * 64, np.float32)
    eng.debug_conv(True, [10], 1, [ok], x, y=y)                                 # the well-formed launch runs
    bad = [
        ("tc Cin % 64", True, [dict(ok, Cin=48)], x, y),
        ("5 problems", True, [ok] * 5, x, y),
        ("mixed plane counts", True, [ok, dict(ok, w_mid=w[0])], x, y),
        ("y too small", True, [ok], x, y[:-1]),
        ("x rows", True, [ok], x[:, :9], y),
        ("halo wider than the gap", True, [dict(ok, k=21, pad=10, w_hi=np.ones((21, 64, 64), np.uint16),
                                                w_lo=np.ones((21, 64, 64), np.uint16))], x, y),
    ]
    fw, fb = weights.conv_ffma_layout(np.ones((64, 24, 1), np.float32))
    fok = dict(_prob(Cin=24, Cout=64), w=fw, bias=fb, ldx=24, cond=None)
    bad += [("ffma Cin % 16", False, [fok], np.ones(240, np.float32), y),
            ("ffma halo", False, [dict(fok, Cin=16, k=33, dil=3, pad=48, ldx=16, w=np.ones((33, 16, 64), np.float32))],
             np.ones(160, np.float32), y)]
    for name, tc, probs, xx, yy in bad:
        lens = [10]
        if name == "halo wider than the gap":               # two utterances 8 gap rows apart, a 10-row halo
            lens, xx, yy = [4, 1], cr.split_planes(np.ones((13, 64), np.float32), 2), np.zeros(13 * 64, np.float32)
        with pytest.raises(VttsError) as ei:
            eng.debug_conv(tc, lens, 1, probs, xx, y=yy)
        assert ei.value.code == -1, name
