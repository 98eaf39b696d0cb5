"""CPU: the float64 references of tests/duration_ref.py against the repository's oracles (oracle/vits_oracle.py: dds_conv,
rq_spline_inverse, durations, frame_to_token; oracle/stabletts_oracle.py: duration_rule), on the edge inputs the GPU test
(test_gpu_durations.py) feeds the kernels, so that a wrong reference cannot make a GPU test pass.  Where an fp32 oracle runs
the same op sequence as a kernel, its output must also lie within the reference's bound."""
import math

import numpy as np
import pytest
import torch

import duration_ref as dr
from oracle import stabletts_oracle as sto
from oracle import vits_oracle as vo
from vosk_tts_b200 import config as C, synthetic, weights


_SD = {}


def _variant(v):
    """Float32 numpy weights of the DDS variant v of the GPU test (synthetic seed 4321, its dp_filter_channels, the depthwise
    weights scaled where the variant scales them)."""
    if v not in _SD:
        D = dr.DDS_VARIANTS[v]
        sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(dict(C.DEFAULT_CONFIG, dp_filter_channels=D), 4321))
        sc = dr.DDS_SEP_SCALE.get(v)
        _SD[v] = {k: (t * sc if sc and ".convs_sep." in k else t).float().numpy() for k, t in sd.items()}
    return _SD[v]


def _oracle_dds(sd, prefix, k, lens, x=None, x0=None, cond=None):
    """vits_oracle.dds_conv in float64 (with the ConvFlow front: conv(x0, pre) and g = cond) per utterance."""
    w = {n: torch.as_tensor(v, dtype=torch.float64) for n, v in sd.items()}
    offs = dr.offsets(lens)
    out = []
    for b, L in enumerate(lens):
        r = slice(offs[b], offs[b] + L)
        mask = torch.ones(1, 1, L, dtype=torch.float64)
        if x0 is not None:
            h = vo.conv(torch.as_tensor(x0[r], dtype=torch.float64)[None, None], w, prefix[:-len(".convs")] + ".pre")
            y = vo.dds_conv(h, mask, w, prefix, k, 3, g=torch.as_tensor(cond[r], dtype=torch.float64).T[None])
        else:
            y = vo.dds_conv(torch.as_tensor(x[r], dtype=torch.float64).T[None], mask, w, prefix, k, 3)
        out.append(y[0].T.numpy())
    return out


@pytest.mark.parametrize("case", dr.dds_cases(), ids=lambda c: "%s-%s-%s-%s" % (c[0], c[1], "x".join(map(str, c[2])), c[3]))
def test_dds_reference(case):
    """Every DDS case of the GPU test: the float64 layers chained agree with the oracle's dds_conv, and each layer's bound
    rejects a 1e-3 relative error and a skipped layer (output = input), so a wrong layer cannot pass."""
    v, stack, lens, kind, seed = case
    sd, D = _variant(v), dr.DDS_VARIANTS[v]
    x, x0, cond = dr.dds_inputs(kind, lens, D, seed=seed)
    if stack == "dp.convs":
        kw = dict(x=x)
    else:
        kw = dict(x0=x0, cond=cond, pre=(sd[stack[:-6] + ".pre.weight"][:, 0, 0], sd[stack[:-6] + ".pre.bias"]))
    oracle = _oracle_dds(sd, stack, 3, lens, **{n: a for n, a in kw.items() if n != "pre"})
    for a, o in zip(dr.dds_chain(sd, stack, 3, lens, **kw), oracle):
        assert np.allclose(a, o, rtol=1e-10, atol=1e-10 * (1 + np.abs(o).max()))
    layers = dr.dds_layers(sd, stack, 3, lens, **kw)
    for i in range(3):
        for b, (r, y, bnd) in enumerate(layers[i]):
            assert np.any(1e-3 * np.abs(y) > bnd), "layer %d of utterance %d: a 1e-3 relative error passes" % (i, b)
            if i > 0:
                prev = layers[i - 1][b][1].astype(np.float32).astype(np.float64)
                assert np.any(np.abs(prev - y) > bnd), "layer %d of utterance %d: skipping the layer passes" % (i, b)


@pytest.mark.parametrize("nb", [1, 2, 10, 16])
def test_spline_reference_matches_oracle(nb):
    """On the GPU test's rows (its seed and bound, den = sqrt(256) of every bin-count variant)."""
    bound, den = 5.0, 16.0
    h, x = dr.spline_rows(nb, bound, den, seed=nb)
    y, bnd, _, _ = dr.spline_inverse(h, x, nb, bound, den)
    t = lambda a, d: torch.as_tensor(np.asarray(a), dtype=d)

    def oracle(d, hh=h, xx=x):
        hh = t(hh, d)
        return vo.rq_spline_inverse(t(xx, d), hh[:, :nb] / math.sqrt(256), hh[:, nb:2 * nb] / math.sqrt(256),
                                    hh[:, 2 * nb:3 * nb - 1], bound=bound).numpy()
    o64 = oracle(torch.float64)
    inside = np.abs(x.astype(np.float64)) <= bound
    # at a knot the float64 oracle may take the other bin: the spline is continuous there, so both agree to rounding
    assert np.allclose(y, o64, rtol=0, atol=1e-9)
    assert np.array_equal(y[~inside], x[~inside].astype(np.float64)) and np.all(bnd[~inside] == 0)
    # the fp32 oracle and the float32 emulation of the kernel lie within the float64 bound (either bin at a knot)
    for name, out in (("fp32 oracle", oracle(torch.float32)), ("emulation", dr.spline_emulate(h, x, nb, bound, den))):
        r = dr.spline_check(h, x, out, nb, bound, den)
        assert np.all(r <= 1.0), "%s %.3g x the bound" % (name, r.max())
    # away from ill-conditioned points the fp32 oracle is within the oracle budget of the emulation, which stands in for
    # the kernel here
    ok = dr.oracle_points(h, x, nb, bound, den)
    assert ok.sum() > 20
    _, bo, _, _ = dr.spline_inverse(h[ok], x[ok], nb, bound, den, err=dr.SPLINE_ERR_ORACLE)
    emu = dr.spline_emulate(h[ok], x[ok], nb, bound, den).astype(np.float64)
    assert np.all(np.abs(oracle(torch.float32, h[ok], x[ok]) - emu) <= bo)
    # rows where no expf / log1pf result reaches the output, on which the GPU test compares bit for bit: for nb >= 3 the
    # rows of equal widths and heights whose x lies in an interior bin
    ex = dr.emulation_exact(h, x, nb, bound, den)
    if nb >= 3:
        assert ex.sum() >= 15
        _, be, _, _ = dr.spline_inverse(h[ex], x[ex], nb, bound, den, err=dr.SPLINE_ERR_EMU)
        assert np.all(be == 0)                    # (the tape agrees: no expf / log1pf op has a derivative there)
    assert np.all(dr.emulation_check(h, x, dr.spline_emulate(h, x, nb, bound, den), nb, bound, den) == 0)


@pytest.mark.parametrize("kind", ["plain", "under", "some_zero", "near", "nan"])
def test_vits_durations_match_oracle(kind):
    m, logs, ls = 0.15, -0.3, 1.1
    lens = [1, 255, 256, 257, 513]
    offs = dr.offsets(lens)
    z = np.zeros(offs[-1], np.float32)
    for b, n in enumerate(lens):
        z[offs[b]:offs[b] + n] = dr.z_of_logw(dr.vits_logw(kind, n, seed=b), m, logs)
    w, bw = dr.vits_w(z, m, logs, ls)
    wc = np.zeros(len(z), np.int64)
    for b, n in enumerate(lens):
        r = slice(offs[b], offs[b] + n)
        if kind == "nan":                      # the oracle propagates NaN; the kernel's ceil gives 0 frames (fmaxf)
            assert dr.ceil_ok(np.where(np.isnan(w[r]), 0, np.ceil(np.nan_to_num(w[r]))), w[r], bw[r]).all()
            continue
        # the fp32 oracle (the kernel's op sequence: exp underflows to 0 in fp32) is one result the bound must accept
        logw = (torch.as_tensor(z[r]) - torch.tensor(m, dtype=torch.float32)) * torch.exp(-torch.tensor(logs, dtype=torch.float32))
        wce, yl = vo.durations(logw[None, None], torch.ones(1, 1, n), ls)
        wc[r] = wce[0, 0].numpy().astype(np.int64)
        assert dr.ceil_ok(wc[r], w[r], bw[r]).all()
        if kind != "under":                    # and the float64 oracle's ceil, away from fp32 underflow
            w64, _ = vo.durations(((torch.as_tensor(z[r], dtype=torch.float64) - m) * math.exp(-logs))[None, None],
                                  torch.ones(1, 1, n, dtype=torch.float64), ls)
            assert dr.ceil_ok(w64[0, 0].numpy(), w[r], bw[r]).all()
        cum, real, capped, foff, host = dr.vits_layout(wc[r], [n])
        assert real[0] == int(yl[0]) and capped == real
        idx = vo.frame_to_token(wce, yl)[0].numpy()
        assert np.array_equal(dr.frame_tokens(cum, real[0]), idx)
    if kind == "under":
        assert dr.vits_layout(wc, lens)[1] == [1] * len(lens)       # no frames at all: y_len 1, the frame takes token T
        assert dr.frame_tokens(np.zeros(3, np.int64), 1)[0] == 3


def test_vits_layout_cap_and_offsets():
    wc = np.array([3, 0, 4, 0, 0, 0, 0, 0, 0, 0, 0, 7, 1], np.int64)      # utterances of 3 and 2 tokens (8 gap rows)
    cum, real, capped, foff, host = dr.vits_layout(wc, [3, 2], cap=5)
    assert real == [7, 8] and capped == [5, 5] and foff == [0, 13, 18] and host == [0, 15, 23]
    assert list(cum[[0, 1, 2, 11, 12]]) == [3, 3, 7, 7, 8]


@pytest.mark.parametrize("ls", [1.0, 0.9])
def test_stt_rule_matches_oracle(ls):
    rng = np.random.default_rng(5)
    n = len(dr.STT_PAUSES) * 3
    mu = rng.standard_normal((n, 50)).astype(np.float32)
    pause = np.zeros(n, np.float32)
    pause[::3] = dr.STT_PAUSES
    a, bnd = dr.stt_pre_round(mu, pause, ls)
    logw32 = torch.sigmoid(torch.as_tensor(mu, dtype=torch.float64)).sum(1).numpy().astype(np.float32)
    d_or, pre = sto.duration_rule(logw32, pause, ls)
    ours = dr.stt_rule(a, 1e9)
    # the oracle rounds the fp32 value: equal wherever the float64 value is not within its bound of a half-integer, and
    # exactly equal on the pause tokens (half to even: 0.5 -> 1 (minimum), 1.5 -> 2, 2.5 -> 2, 3.5 -> 4; negative -> 1)
    assert dr.rint_ok(d_or, a, bnd, 1e9).all()
    p = pause != 0
    assert np.array_equal(ours[p], d_or[p]) and np.array_equal(a[p], pre[p].astype(np.float64))
    if ls == 1.0:
        assert list(ours[::3][:6]) == [1, 2, 2, 4, 1, 1]
    assert list(dr.stt_rule(np.array([5000.0, 4096.5, 4095.5]), 4096)) == [4096, 4096, 4096]


def test_stt_expand_and_pause_fill_emulation():
    x = np.arange(12, dtype=np.float32).reshape(6, 2)
    mu_mel = np.arange(6, dtype=np.float32)[:, None] + np.float32(0.25)
    pause = np.array([0, 2, 0, 0, 0, 1], np.float32)
    dur = np.array([1, 2, 0, 0, 0, 1], np.int64)                       # utterances [2, 1] (tokens at rows 0-1 and 10)
    lens = [2, 1]
    x = np.concatenate([x[:2], np.zeros((8, 2), np.float32), x[2:3]])
    mu_mel = np.concatenate([mu_mel[:2], np.zeros((8, 1), np.float32), mu_mel[2:3]])
    pause = np.concatenate([pause[:2], np.zeros(8, np.float32), [1]]).astype(np.float32)
    dur = np.concatenate([dur[:2], np.zeros(8, np.int64), [1]])
    mu, pau, pr, mask = dr.stt_expand(x, mu_mel, pause, dur, lens, [3, 1], denorm=(1.5, 2.0))
    assert mask.sum() == 4 and list(pau[mask]) == [0, 2, 2, 1]
    assert np.array_equal(mu[[0, 1, 2, 11]], x[[0, 1, 1, 10]]) and pr[0, 0] == np.float32(0.25 * 2 + 1.5)
    mel = np.arange(12, dtype=np.float32).reshape(12, 1)
    filled = dr.pause_fill(mel, pau, [3, 1])
    assert list(filled[:, 0][[0, 1, 2, 11]]) == [0, 0, 0, 11]     # frames 1, 2 take frame 0; frame 0 of each keeps its own
