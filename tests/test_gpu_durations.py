"""GPU (-m gpu): the kernels that produce the durations, one stage at a time through the engine's own launch code, against
the float64 references and error bounds of tests/duration_ref.py:
  vtts_debug_dds            dds_layer_kernel<DDS_TT> x 3 (a DDSConv stack, with the ConvFlow front)
  vtts_debug_spline         spline_inverse_kernel (also against the fp32 oracle, op order for op order)
  vtts_debug_durations      duration_kernel, then sample_prior_kernel
  vtts_debug_stt_durations  stt_dur_kernel, stt_expand_kernel, stt_pause_fill_kernel (StableTTS)
Every case writes finite garbage (or a sentinel) into the gap rows and the rows behind the last utterance and checks that
rows outside the utterances keep it, and that a second run is bit-identical.  Engines are built from synthetic checkpoints,
with config variants for other dp_filter_channels (32 .. 256: 1 to 8 warps, 1 to 8 weight chunks around the ring depth 4)
and bin counts (1, 2, 10, 16)."""
import json
import math

import numpy as np
import pytest
import torch

import duration_ref as dr
import stabletts_inputs as SI
from oracle import vits_oracle as vo
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine, VttsError

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
ISENT = -7
VARIANTS = dict({v: dict(dp_filter_channels=D) for v, D in dr.DDS_VARIANTS.items()}, b1=dict(dp_num_bins=1), b2=dict(dp_num_bins=2),
                b16=dict(dp_num_bins=16))
WORST = {}                   # largest error / bound seen per kernel


@pytest.fixture(scope="module")
def engines():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    made = {}

    def get(name):
        if name not in made:
            c = dict(C.DEFAULT_CONFIG, **VARIANTS[name])
            scale = dr.DDS_SEP_SCALE.get(name)
            sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(c, 4321))
            if scale:
                sd = {k: v * scale if ".convs_sep." in k else v for k, v in sd.items()}
            blob, man = weights.pack(sd, c)
            made[name] = (Engine(c, blob, man, device=0, precision=0), {k: v.float() for k, v in sd.items()}, c)
        return made[name]
    yield get
    for e, _, _ in made.values():
        e.close()
    print("\nduration path error / bound, largest per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


def _note(kernel, r):
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(r))


def _inside(lens, rows):
    m = np.zeros(rows, bool)
    for b, n in enumerate(lens):
        m[dr.offsets(lens)[b]:dr.offsets(lens)[b] + n] = True
    return m


# ---------------------------------------------------------------------------------------------------- DDSConv
def run_dds(ent, stack, lens, kind, seed=0):
    """The three layers; each layer's output against the float64 layer on the kernel's own input (the previous layer's
    output), within that layer's bound."""
    e, sd, c = ent
    D, k = c["dp_filter_channels"], c["dp_kernel_size"]
    x, x0, cond = dr.dds_inputs(kind, lens, D, seed=seed)
    rows = x.shape[0]
    y0 = np.full((3, rows, D), SENT, np.float32)
    if stack == "dp.convs":
        args, kw = dict(x=x), dict(x=x)
    else:
        p = stack[:-len(".convs")]
        args = dict(x0=x0, cond=cond)
        kw = dict(args, pre=(sd[p + ".pre.weight"][:, 0, 0].numpy(), sd[p + ".pre.bias"].numpy()))
    y = e.debug_dds(stack, lens, y0, **args)
    y2 = e.debug_dds(stack, lens, y0, **args)
    assert np.array_equal(y.view(np.uint32), y2.view(np.uint32)), "two launches differ"
    assert np.all(y[:, ~_inside(lens, rows)].view(np.uint32) == SENT.view(np.uint32)), "rows outside the utterances written"
    worst = 0.0
    for i, layer in enumerate(dr.dds_layers({n: t.numpy() for n, t in sd.items()}, stack, k, lens, ys=y, **kw)):
        for r, v, bnd in layer:
            assert np.isfinite(y[i, r]).all()
            ratio = float(np.max(np.abs(y[i, r].astype(np.float64) - v) / bnd))
            assert ratio <= 1.0, "%s %s %s layer %d: error %.3g x the bound" % (stack, lens[:6], kind, i, ratio)
            worst = max(worst, ratio)
    _note("dds_layer_kernel", worst)
    return y


@pytest.mark.parametrize("case", dr.dds_cases(), ids=lambda c: "%s-%s-%s-%s" % (c[0], c[1], "x".join(map(str, c[2])), c[3]))
def test_dds(engines, case):
    v, stack, lens, kind, seed = case
    run_dds(engines(v), stack, lens, kind, seed=seed)


# ---------------------------------------------------------------------------------------------------- spline
def _pack_rows(h, x, nparts, rng):
    """Split N rows into nparts utterances packed with gaps; gap and tail rows hold garbage parameters and the sentinel x."""
    N = len(x)
    cuts = np.sort(rng.choice(np.arange(1, N), nparts - 1, replace=False)) if nparts > 1 else []
    lens = list(np.diff(np.concatenate([[0], cuts, [N]])).astype(int))
    offs = dr.offsets(lens)
    rows = offs[-1] + 5
    hp = rng.uniform(-50, 50, (rows, h.shape[1] + 3)).astype(np.float32)
    xp = np.full(rows, SENT, np.float32)
    src = 0
    for b, n in enumerate(lens):
        hp[offs[b]:offs[b] + n, :h.shape[1]] = h[src:src + n]
        xp[offs[b]:offs[b] + n] = x[src:src + n]
        src += n
    return lens, hp, xp, _inside(lens, rows)


@pytest.mark.parametrize("variant", ["b1", "b2", "c256", "b16"])
def test_spline_inverse(engines, variant):
    e, sd, c = engines(variant)
    nb, bound, D = c["dp_num_bins"], float(c["dp_tail_bound"]), c["dp_filter_channels"]
    den = float(np.float32(math.sqrt(D)))
    h, x = dr.spline_rows(nb, bound, den, seed=nb)
    lens, hp, xp, inside = _pack_rows(h, x, 3, np.random.default_rng(nb))
    out = e.debug_spline(lens, hp, xp)
    assert np.array_equal(out.view(np.uint32), e.debug_spline(lens, hp, xp).view(np.uint32)), "two launches differ"
    assert np.all(out[~inside].view(np.uint32) == SENT.view(np.uint32)), "rows outside the utterances written"
    y = out[inside]
    outside = np.abs(x.astype(np.float64)) > bound
    assert np.array_equal(y[outside].view(np.uint32), x[outside].view(np.uint32)), "linear tails are not the identity"
    r = dr.spline_check(h, x, y, nb, bound, den)
    _note("spline_inverse_kernel", r.max())
    assert np.all(r <= 1.0), "spline: error %.3g x the bound at rows %s" % (r.max(), np.nonzero(r > 1)[0][:8])
    # the fp32 oracle, away from ill-conditioned points: the budget of exp / log1p / softmax differences only
    ok = dr.oracle_points(h, x, nb, bound, den)
    hh = torch.as_tensor(h[ok])
    o32 = vo.rq_spline_inverse(torch.as_tensor(x[ok]), hh[:, :nb] / math.sqrt(D), hh[:, nb:2 * nb] / math.sqrt(D),
                               hh[:, 2 * nb:3 * nb - 1], bound=bound).numpy().astype(np.float64)
    _, bo, _, _ = dr.spline_inverse(h[ok], x[ok], nb, bound, den, err=dr.SPLINE_ERR_ORACLE)
    ro = np.abs(y[ok] - o32) / bo
    _note("spline_vs_fp32_oracle", ro.max())
    i = int(np.argmax(ro))
    assert np.all(ro <= 1.0), "spline vs fp32 oracle: %.3g x the budget (x %r, kernel %r, oracle %r, budget %.3g, h %s)" % (
        ro.max(), float(x[ok][i]), float(y[ok][i]), float(o32[i]), bo[i], h[ok][i].tolist())
    # the op order itself: against the kernel's op sequence in NumPy float32, bit for bit where no expf / log1pf result
    # reaches the output (the rows of equal widths and heights), within SPLINE_ERR_FLIP elsewhere
    re = dr.emulation_check(h, x, y, nb, bound, den)
    _note("spline_vs_emulation", re.max())
    assert np.all(re <= 1.0), "spline vs float32 emulation: %.3g x the expf / log1pf budget at rows %s" % (
        re.max(), np.nonzero(re > 1)[0][:8])


# ---------------------------------------------------------------------------------------------------- VITS durations
def run_durations(ent, lens, kinds, cap=0, seed=0, ls=1.1, ns=0.667):
    e, sd, c = ent
    I = c["inter_channels"]
    m, logs = float(sd["dp.flows.0.m"][0, 0]), float(sd["dp.flows.0.logs"][0, 0])
    rng = np.random.default_rng(seed)
    offs = dr.offsets(lens)
    rows = offs[-1] + 9
    z = rng.uniform(-1e3, 1e3, rows).astype(np.float32)
    for b, n in enumerate(lens):
        z[offs[b]:offs[b] + n] = dr.z_of_logw(dr.vits_logw(kinds[b % len(kinds)], n, seed=seed + b), m, logs)
    stats = rng.uniform(-1e3, 1e3, (rows, 2 * I)).astype(np.float32)
    for b, n in enumerate(lens):
        stats[offs[b]:offs[b] + n] = rng.standard_normal((n, 2 * I))
        stats[offs[b]:offs[b] + n, I:] *= 0.3
    w, bw = dr.vits_w(z, m, logs, ls)
    hi = np.where(np.isnan(w), 0, np.clip(np.ceil(w + bw), 0, dr.CEIL_CAP))
    frames = [max(int(hi[offs[b]:offs[b] + n].sum()), 1) for b, n in enumerate(lens)]
    capped = [min(f, cap) if cap else f for f in frames]
    frame_rows = dr.offsets(capped)[-1] + 16
    eps = rng.standard_normal((len(lens), I, max(capped))).astype(np.float32)
    init = dict(wceil=np.full(rows, ISENT, np.int32), cum=np.full(rows, ISENT, np.int32), z_p=np.full((frame_rows, I), SENT, np.float32),
                frame_token=np.full(frame_rows, ISENT, np.int32))
    o = e.debug_durations(lens, z, ls, stats, eps, ns, frame_rows, frame_cap=cap, **init)
    o2 = e.debug_durations(lens, z, ls, stats, eps, ns, frame_rows, frame_cap=cap, **init)   # the ticket counter is back at 0
    for k in o:
        assert np.array_equal(o[k].view(np.uint32) if o[k].dtype == np.float32 else o[k], o2[k].view(np.uint32) if o2[k].dtype == np.float32 else o2[k]), k
    inside = _inside(lens, rows)
    assert np.all(o["wceil"][~inside] == ISENT) and np.all(o["cum"][~inside] == ISENT), "token rows outside the utterances written"
    wc = o["wceil"].astype(np.int64)
    ok = dr.ceil_ok(wc[inside], w[inside], bw[inside])
    assert ok.all(), "ceil durations differ at %s" % np.nonzero(~ok)[0][:8]
    cum, real, cl, foff, host = dr.vits_layout(np.where(inside, wc, 0), lens, cap)
    assert np.array_equal(o["cum"][inside], cum[inside])
    assert list(o["ylen_real"]) == real and list(o["ylen"]) == cl and list(o["frm_off"]) == foff
    assert list(o["published"]) == real + host
    fin = _inside(cl, frame_rows)
    assert np.all(o["frame_token"][~fin] == ISENT) and np.all(o["z_p"][~fin].view(np.uint32) == SENT.view(np.uint32))
    worst = 0.0
    for b, n in enumerate(lens):
        tok = dr.frame_tokens(cum[offs[b]:offs[b] + n], cl[b])
        fr = slice(foff[b], foff[b] + cl[b])
        assert np.array_equal(o["frame_token"][fr], tok), "frame -> token map of utterance %d" % b
        v, bnd = dr.prior(stats[offs[b]:offs[b] + n], tok, eps[b, :, :cl[b]], ns, I)
        err = np.abs(o["z_p"][fr].astype(np.float64) - v)
        worst = max(worst, float(np.max(np.where(bnd > 0, err / np.maximum(bnd, 1e-300), np.where(err == 0, 0, np.inf)))))
    _note("sample_prior_kernel", worst)
    assert worst <= 1.0, "z_p: error %.3g x the bound" % worst
    return o


@pytest.mark.parametrize("T", [1, 255, 256, 257, 511, 512, 513, 2000])
def test_durations_lengths(engines, T):
    run_durations(engines("c256"), [T], ["plain"], seed=T)


@pytest.mark.parametrize("B", [2, 37, 128])
def test_durations_batches(engines, B):
    lens = [int(v) for v in np.random.default_rng(B).integers(1, 300, B)]
    lens[0] = 257
    run_durations(engines("c256"), lens, ["plain", "some_zero", "near"], seed=B)


@pytest.mark.parametrize("kinds", [["under"], ["some_zero"], ["near"], ["nan"], ["plain", "under", "nan"]], ids="-".join)
def test_durations_edges(engines, kinds):
    o = run_durations(engines("c256"), [300, 1, 40][:len(kinds)] if len(kinds) > 1 else [300], kinds, seed=7)
    if kinds[0] == "under":                  # every token underflows to 0 frames: y_len 1, its one frame takes token T
        assert o["ylen"][0] == 1 and np.all(o["wceil"][:300] == 0) and o["frame_token"][0] == 300


def test_durations_ceil_cap_and_length_cap(engines):
    """logw past the 1e6 cap, and a speculative frame cap: ylen clamped on the device, ylen_real and the published offsets not."""
    o = run_durations(engines("c256"), [6, 40, 3], ["cap", "plain"], cap=256, seed=3)
    assert o["wceil"].max() == 1000000 and o["ylen_real"][0] >= 3 * 1000000 and o["ylen"][0] == 256


def test_durations_past_int32_refused(engines):
    """2148 tokens of 1e6 frames sum past INT32_MAX: refused, as one utterance and as a batch, by the hook and by vtts_durations."""
    e, sd, c = engines("c256")
    m, logs = float(sd["dp.flows.0.m"][0, 0]), float(sd["dp.flows.0.logs"][0, 0])
    I = c["inter_channels"]
    for lens, what in (([2148], "utterance"), ([1074, 1074], "batch")):
        rows = dr.offsets(lens)[-1]
        z = np.full(rows, dr.z_of_logw(np.array([20.0]), m, logs)[0], np.float32)
        with pytest.raises(VttsError, match="INT32_MAX") as ei:
            e.debug_durations(lens, z, 1.0, np.zeros((rows, 2 * I), np.float32), np.zeros((len(lens), I, 1), np.float32), 1.0, 64)
        assert ei.value.code == -1 and what in str(ei.value)
    # the same through the engine: a huge length_scale caps every token at 1e6 frames
    ids = np.random.default_rng(0).integers(0, c["n_vocab"], (1, 2148))
    with pytest.raises(VttsError, match="INT32_MAX"):
        e.durations(ids, [2148], [0], (0.667, 1e30, 0.8))
    ylen = e.durations(ids[:, :40], [40], [0], (0.667, 1.0, 0.8))                 # and the engine still serves the next call
    assert 1 <= int(ylen[0]) < 10000


# ---------------------------------------------------------------------------------------------------- StableTTS
@pytest.fixture(scope="module")
def stt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.stabletts import StableTTS
    cfg = SI.config()
    sd = SI.model(cfg)
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=0)
    yield t
    t.engine.close()


@pytest.mark.parametrize("denorm", [False, True])
@pytest.mark.parametrize("lens", [[256], [257], [5, 256, 3, 40]], ids=lambda v: "x".join(map(str, v)))
def test_stt_durations(stt, lens, denorm):
    e, cfg = stt.engine, stt.cfg
    DC, MC, NC = cfg["dur_channels"], cfg["cond_channels"], cfg["noise_channels"]
    rng = np.random.default_rng(len(lens) * 100 + lens[0])
    offs = dr.offsets(lens)
    rows = offs[-1] + 7
    inside = _inside(lens, rows)
    mu_dp = rng.uniform(-1e3, 1e3, (rows, DC)).astype(np.float32)
    mu_dp[inside] = (rng.standard_normal((inside.sum(), DC)) * 2 - 3.2).astype(np.float32)
    pause = rng.uniform(-1e3, 1e3, rows).astype(np.float32)
    pause[inside] = 0
    tok = np.nonzero(inside)[0]
    pause[tok[::5]] = np.resize(np.float32(dr.STT_PAUSES), len(tok[::5]))
    x = rng.standard_normal((rows, MC)).astype(np.float32)
    mu_mel = rng.standard_normal((rows, NC)).astype(np.float32)
    ls = 1.0
    a, bnd = dr.stt_pre_round(mu_dp, pause, ls)
    frame_rows = dr.offsets([int(np.clip(np.rint(a[offs[b]:offs[b] + n] + bnd[offs[b]:offs[b] + n] + 1), 1, 4096).sum())
                             for b, n in enumerate(lens)])[-1] + 11
    init = dict(dur=np.full(rows, ISENT, np.int32), first=np.full(rows, ISENT, np.int32), logw=np.full(rows, SENT, np.float32),
                mu=np.full((frame_rows, MC), SENT, np.float32), pau=np.full(frame_rows, SENT, np.float32),
                prior=np.full((frame_rows, NC), SENT, np.float32), mel=rng.standard_normal((frame_rows, NC)).astype(np.float32))
    o = e.debug_stt_durations(lens, mu_dp, pause, ls, x, frame_rows, mu_mel=mu_mel, denormalise=denorm, init=init)
    o2 = e.debug_stt_durations(lens, mu_dp, pause, ls, x, frame_rows, mu_mel=mu_mel, denormalise=denorm, init=init)
    for k in o:
        assert np.array_equal(o[k], o2[k]), k
    for k in ("dur", "first"):
        assert np.all(o[k][~inside] == ISENT)
    assert np.all(o["logw"][~inside].view(np.uint32) == SENT.view(np.uint32))
    d = o["dur"][inside].astype(np.int64)
    err = np.abs(o["logw"][inside].astype(np.float64) - a[inside])
    r = float(np.max(np.where(bnd[inside] > 0, err / np.maximum(bnd[inside], 1e-300), np.where(err == 0, 0, np.inf))))
    _note("stt_dur_kernel", r)
    assert r <= 1.0, "pre-rounding values: %.3g x the bound" % r
    assert dr.rint_ok(d, a[inside], bnd[inside], 4096).all()
    p = pause[inside] != 0
    assert np.array_equal(d[p], dr.stt_rule(a[inside][p], 4096)), "pause tokens (half to even, minimum 1, at most 4096)"
    flens = []
    for b, n in enumerate(lens):
        db = o["dur"][offs[b]:offs[b] + n].astype(np.int64)
        assert np.array_equal(o["first"][offs[b]:offs[b] + n], np.cumsum(db) - db)
        flens.append(int(db.sum()))
    assert list(o["ylen"]) == flens
    dur_full = np.where(inside, o["dur"], 0)
    mu, pau, pr, fmask = dr.stt_expand(x, mu_mel, pause, dur_full, lens, flens,
                                       denorm=(stt.mel_mean, stt.mel_std) if denorm else None, frame_rows=frame_rows)
    assert np.array_equal(o["mu"][fmask].view(np.uint32), mu[fmask].view(np.uint32))
    assert np.array_equal(o["pau"][fmask].view(np.uint32), pau[fmask].view(np.uint32))
    assert np.array_equal(o["prior"][fmask].view(np.uint32), pr[fmask].view(np.uint32))
    assert np.all(o["mu"][~fmask].view(np.uint32) == SENT.view(np.uint32)) and np.all(o["pau"][~fmask].view(np.uint32) == SENT.view(np.uint32))
    assert np.array_equal(o["mel"].view(np.uint32), dr.pause_fill(init["mel"], np.where(fmask, pau, 0), flens).view(np.uint32))


# ---------------------------------------------------------------------------------------------------- refusals
def test_hook_refusals(engines, stt):
    e, sd, c = engines("c96")
    x = np.zeros((20, 96), np.float32)
    y = np.zeros((3, 20, 96), np.float32)
    for stack, kw in (("dp.flows.2.convs", dict(x0=x[:, 0], cond=x)), ("dp.flows.9.convs", dict(x0=x[:, 0], cond=x)),
                      ("dp.flows.3x.convs", dict(x0=x[:, 0], cond=x)), ("dp.flows.+3.convs", dict(x0=x[:, 0], cond=x)),
                      ("dp.proj", dict(x=x)), ("dp.convs", dict(x0=x[:, 0], cond=x)), ("dp.flows.3.convs", dict(x=x))):
        with pytest.raises(VttsError) as ei:
            e.debug_dds(stack, [5], y, **kw)
        assert ei.value.code == -1
    for lens in ([0], [15, 5], []):
        with pytest.raises(VttsError) as ei:
            e.debug_dds("dp.convs", lens, y, x=x)
        assert ei.value.code == -1
    with pytest.raises(VttsError) as ei:
        e.debug_spline([5], np.zeros((20, 28), np.float32), np.zeros(20, np.float32))       # 3 * 10 - 1 = 29 parameters
    assert ei.value.code == -1
    with pytest.raises(VttsError) as ei:
        e.debug_durations([30], np.zeros(20, np.float32), 1.0, np.zeros((20, 384), np.float32), np.zeros((1, 192, 4), np.float32),
                          1.0, 64)
    assert ei.value.code == -1
    # a StableTTS hook on a VITS engine (refused by the library before it reads any pointer) and the other way round
    lens = np.array([5], np.int32)
    assert e.lib.vtts_debug_stt_durations(e.h, 1, lens.ctypes.data, 20, *([None] * 2), 1.0, None, None, 0, *([None] * 4), 64,
                                          *([None] * 4)) == -1
    # mis-shaped arrays are refused by the wrappers before they reach the library
    for call in (lambda: e.debug_dds("dp.convs", [5], y, x=np.zeros((20, 95), np.float32)),
                 lambda: e.debug_dds("dp.flows.3.convs", [5], y, x0=np.zeros(19, np.float32), cond=x),
                 lambda: e.debug_dds("dp.convs", [5], y[0], x=x),
                 lambda: e.debug_spline([5], np.zeros((20, 32), np.float32), np.zeros(19, np.float32)),
                 lambda: e.debug_durations([5], np.zeros(20, np.float32), 1.0, np.zeros((20, 383), np.float32),
                                           np.zeros((1, 192, 4), np.float32), 1.0, 64),
                 lambda: e.debug_durations([5], np.zeros(20, np.float32), 1.0, np.zeros((20, 384), np.float32),
                                           np.zeros((2, 192, 4), np.float32), 1.0, 64),
                 lambda: e.debug_stt_durations([5], np.zeros((20, 50), np.float32), np.zeros(20, np.float32), 1.0,
                                               np.zeros((20, 8), np.float32), 64),
                 lambda: stt.engine.debug_stt_durations([5], np.zeros((20, 49), np.float32), np.zeros(20, np.float32), 1.0,
                                                        np.zeros((20, stt.cfg["cond_channels"]), np.float32), 64)):
        with pytest.raises(ValueError):
            call()
    with pytest.raises(VttsError) as ei:
        stt.engine.debug_spline([5], np.zeros((20, 32), np.float32), np.zeros(20, np.float32))
    assert ei.value.code == -1


@pytest.mark.parametrize("nb", [0, 17])
def test_bin_counts_refused_at_create(nb):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = dict(C.DEFAULT_CONFIG, dp_num_bins=nb)
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(dict(c, dp_num_bins=max(nb, 1)), 1)), c)
    with pytest.raises(VttsError, match="dp_num_bins") as ei:
        Engine(c, blob, man, device=0, precision=0)
    assert ei.value.code == -1


@pytest.mark.parametrize("variant", ["b1", "b2", "b16"])
def test_durations_call_with_bin_count(engines, variant):
    """Spline parameter rows are sized from dp_num_bins: 1, 2 and 16 bins (16 did not fit the former fixed pitch of 32)
    run the whole duration predictor, with the oracle's durations except where its fp32 w is within 1e-3 of an integer."""
    e, sd, c = engines(variant)
    g = torch.Generator().manual_seed(5)
    T = 60
    tok = torch.randint(0, c["n_vocab"], (1, T), generator=g)
    eps_dp = torch.randn(1, 2, T, generator=g)
    scales = (0.667, 1.0, 0.8)
    ylen, dur = e.durations(tok.numpy(), [T], [2], scales, eps_dp.numpy(), want_durations=True)
    with torch.no_grad():
        o = vo.infer(sd, c, tok, torch.tensor([T]), torch.tensor([2]), scales, eps_dp, eps_z=lambda shape: torch.zeros(shape),
                     decode=False)
    wref = o["w_ceil"][0, 0].numpy()
    logw = o["logw"][0, 0].numpy().astype(np.float64)
    w = np.exp(logw) * scales[1]
    near = np.abs(w - np.rint(w)) < 1e-3 * np.maximum(1, w)
    assert np.array_equal(dur[0][~near], wref[~near].astype(np.int32)) and np.all(np.abs(dur[0] - wref) <= 1)
    assert int(ylen[0]) == max(int(dur[0].sum()), 1)
