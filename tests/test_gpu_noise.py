"""GPU (-m gpu): the four kernels that draw the engine's Gaussian noise when the caller gives none.  Each runs alone through
the engine's own launch helper (vtts_debug_noise) and is compared with the float64 restatement and bounds of
tests/noise_ref.py:
  dp_noise_kernel          (dp_noise: VITS durations)                    stream 1
  sample_prior_kernel      (sample_prior: VITS prior sample, phase 2)    stream 2
  posterior_sample_kernel  (posterior_sample: VITS and QuickVC convert, align)   stream 3
  dit_init_kernel          (dit_init: StableTTS flow matching)           stream 7
Every element written must lie within its bound, over ragged batches, at B = 64 and at lengths up to 3001.  Rows outside the
utterances must keep a sentinel, and two launches must give the same bits.  The seeds include the ends of the 64-bit range
and halves whose bits are a float NaN, infinity, a denormal or -0, because the seed travels through the call's float scalar
block.

Then each family's entry point is pinned to its caller-noise path: a call with seed S must give the same bits as the same
call given, as caller noise, the draws the hook returns for S.  That checks the seed plumbing and the (b, t, c) keying of
real calls.  An utterance's draws depend on its index b in the batch and on the call's one seed.  There is no per-utterance
seed, unlike the GPT-SoVITS sampler's per-sentence seeds: the same utterance at another index draws other noise."""
import json

import numpy as np
import pytest
import torch

import noise_ref as R
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
import stabletts_cfm_inputs as SI
import vc_inputs as VI
import golden_ref as GR
from vosk_tts_b200 import config as CF, synthetic, weights
from vosk_tts_b200.engine import Engine

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
WORST = {}                                   # largest error / bound per kernel
S = 0x0123456789ABCDEF
BATCHES = {
    "ragged": [1, 2, 7, 64, 65, 130, 3001],
    "b64": [int(n) for n in np.random.default_rng(64).integers(1, 160, 64)],
}
SEEDS = [0, 1, 2 ** 32, 2 ** 63, 2 ** 64 - 1,   # 1 and 2^32: a denormal half (low / high); 2^63: -0 in the high half
         0x7FC00000, 0x7FC00000 << 32,         # quiet NaN in the low / high half
         0x7F800001, 0x7F800001 << 32,         # signalling NaN
         0x7F800000, 0x7F800000 << 32,         # infinity
         0x80000000,                           # -0 in the low half
         0x7FC000007F800001]
_ENGINES = {}


def _engine(kind):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if kind not in _ENGINES:
        if kind == "vits":         # the tiny linear-spectrogram model: text, durations, prior, posterior
            cfg = CF.from_training_json(VI.training_json("lin"), n_vocab=GR.N_VOCAB)
            sd = synthetic.make_random_checkpoint(cfg, VI.SEEDS["lin"], posterior=True)
            blob, man = weights.pack(weights.fold_weight_norm(sd), cfg, posterior=True)
        elif kind == "quickvc":
            cfg = QI.config()
            blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), cfg)
        else:
            cfg = SI.config()
            blob, man = weights.pack_stabletts_cfm(SI.model(cfg), cfg)
        _ENGINES[kind] = Engine(cfg, blob, man, device=0, precision=0)
    return _ENGINES[kind]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()
    print("\nnoise kernels error / bound, largest per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


def _within(kernel, dev, ref, bound):
    dev = np.asarray(dev, np.float64)
    assert np.all(np.isfinite(dev))
    r = np.abs(dev - ref) / np.maximum(bound, 1e-300)
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(r.max()))
    bad = np.nonzero(~(np.abs(dev - ref) <= bound))[0]
    assert bad.size == 0, "%s: %d elements outside the bound, first %s: %r vs %r (bound %r)" % (
        kernel, bad.size, bad[0], dev[bad[0]], ref[bad[0]], bound[bad[0]])


def _outside(lens, rows):
    off = R.offsets(lens)
    inside = np.zeros(rows, bool)
    for b, n in enumerate(lens):
        inside[off[b]:off[b] + n] = True
    return ~inside


def _stats(lens, C, seed):
    """stats rows [rows, 2C] = [m | logs], NaN outside the utterances so that a stray read shows."""
    rows = int(R.offsets(lens)[-1])
    rng = np.random.default_rng(seed)
    st = np.concatenate([rng.normal(0, 2, (rows, C)), rng.uniform(-3, 1.5, (rows, C))], 1).astype(np.float32)
    st[_outside(lens, rows)] = np.nan
    return st


def _run_twice(fn):
    a, b = fn(), fn()
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), "two launches differ"
    return a


def _check_dp(e, lens, seed, scale=0.667):
    rows = int(R.offsets(lens)[-1])
    out = _run_twice(lambda: e.debug_noise("dp", seed, lens, np.full((2, rows), SENT, np.float32), scale=scale))
    ref, row = R.draws("dp", seed, lens)
    for k in range(2):
        _within("dp_noise_kernel", out[k, row], ref[k] * float(np.float32(scale)), R.scaled_bound(ref[k], scale))
    assert np.all(out[:, _outside(lens, rows)] == SENT)


def _check_sampler(e, kernel, lens, C, seed, scale=0.8):
    rows = int(R.offsets(lens)[-1])
    st = _stats(lens, C, len(lens) + C)
    out = _run_twice(lambda: e.debug_noise(kernel, seed, lens, np.full((rows, C), SENT, np.float32), scale=scale, stats=st))
    ref_e, (row, c) = R.draws(kernel, seed, lens, C)
    ref, bound = R.sample_ref(ref_e, st[row, c], st[row, C + c], scale)
    _within({"prior": "sample_prior_kernel", "posterior": "posterior_sample_kernel"}[kernel], out[row, c], ref, bound)
    assert np.all(out[_outside(lens, rows)] == SENT)


def _check_dit(e, lens, NC, seed, temperature=0.9, MC=24, HC=16):
    B = len(lens)
    exts = [n + (b % 4) * 3 for b, n in enumerate(lens)]        # padded extents, lens == exts for every fourth utterance
    off = R.offsets(exts)
    rows = int(off[-1])
    fake = np.random.default_rng(NC).normal(size=MC).astype(np.float32)
    xc, mu, skx = _run_twice(lambda: e.debug_noise(
        "dit", seed, lens, np.full((2 * rows, NC + HC), SENT, np.float32), scale=temperature, exts=exts, fake_content=fake,
        mu=np.full((2 * rows, MC), SENT, np.float32), skx=np.full((2 * rows, 2 * HC), SENT, np.float32)))
    ref_e, (row, c) = R.draws("dit", seed, exts, NC)
    _within("dit_init_kernel", xc[row, c], ref_e * float(np.float32(temperature)), R.scaled_bound(ref_e, temperature))
    cond, unc = xc[:rows], xc[rows:]
    # the unconditional sequences carry their conditional twin's noise, bit for bit
    assert np.array_equal(cond[:, :NC].view(np.uint32), unc[:, :NC].view(np.uint32))
    out = _outside(exts, rows)
    assert np.all(cond[out] == SENT) and np.all(unc[out] == SENT) and np.all(xc[:, NC:] == SENT)
    for b in range(B):
        o, n, x = int(off[b]), lens[b], exts[b]
        assert np.all(mu[o:o + n] == SENT)                                   # conditional mu rows are the caller's
        assert np.all(mu[o + n:o + x] == 0) and np.all(skx[o + n:o + x, :HC] == 0)
        assert np.all(mu[rows + o:rows + o + x] == fake[None, :])            # unconditional mu rows are fake_content
        assert np.all(skx[rows + o + n:rows + o + x, :HC] == 0)
        assert np.all(skx[o:o + n] == SENT) and np.all(skx[rows + o:rows + o + n] == SENT)
    assert np.all(skx[:, HC:] == SENT)
    for a in (mu[:rows], mu[rows:], skx[:rows], skx[rows:]):
        assert np.all(a[out] == SENT)


@pytest.mark.parametrize("batch", sorted(BATCHES))
def test_dp_noise(batch):
    _check_dp(_engine("vits"), BATCHES[batch], S)


@pytest.mark.parametrize("kernel", ["prior", "posterior"])
@pytest.mark.parametrize("batch,C", [("ragged", 192), ("b64", 192), ("ragged", 37), ("b64", 2)])
def test_samplers(kernel, batch, C):
    _check_sampler(_engine("vits"), kernel, BATCHES[batch], C, S)


@pytest.mark.parametrize("batch,NC", [("ragged", 80), ("b64", 80), ("ragged", 100)])
def test_dit_init(batch, NC):
    _check_dit(_engine("vits"), BATCHES[batch], NC, S)


@pytest.mark.parametrize("seed", SEEDS, ids=[hex(s) for s in SEEDS])
def test_seeds(seed):
    """Every seed's restated stream comes out of every kernel: the seed's bits survive the float scalar block."""
    e, lens = _engine("vits"), [1, 5, 130]
    _check_dp(e, lens, seed)
    _check_sampler(e, "prior", lens, 192, seed)
    _check_sampler(e, "posterior", lens, 192, seed)
    _check_dit(e, lens, 80, seed)


def test_scale_one_is_the_draw():
    """With scale 1 and stats m = 0, logs = 0 the outputs are the draws themselves (the caller noise the family tests pass)."""
    e, lens = _engine("vits"), [3, 40]
    rows = int(R.offsets(lens)[-1])
    z = e.debug_noise("posterior", S, lens, np.zeros((rows, 8), np.float32), stats=np.zeros((rows, 16), np.float32))
    ref, (row, c) = R.draws("posterior", S, lens, 8)
    _within("posterior_sample_kernel", z[row, c], ref, R.normal_bound(ref))


# ---------------------------------------------------------------------------------------------- each family's entry point
def _hook_noise(e, kernel, lens, C):
    """The draws the hook makes for seed S at utterances of `lens` rows as caller noise [B, C, max len]."""
    lens = [int(n) for n in lens]
    rows = int(R.offsets(lens)[-1])
    out = e.debug_noise(kernel, S, lens, np.zeros((rows, C), np.float32), stats=np.zeros((rows, 2 * C), np.float32))
    off = R.offsets(lens)
    eps = np.zeros((len(lens), C, max(lens)), np.float32)
    for b, n in enumerate(lens):
        eps[b, :, :n] = out[off[b]:off[b] + n].T
    return eps


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _vits_inputs(e):
    rng = np.random.default_rng(3)
    lens = np.array([11, 5, 23], np.int64)
    ids = rng.integers(1, int(e.cfg["n_vocab"]), (3, 23)).astype(np.int64)
    return ids, lens, np.array([1, 0, 2], np.int64)


@pytest.mark.parametrize("fused", [False, True], ids=["two-phase", "vtts_infer"])
def test_infer_seed_is_the_hooks_noise(fused):
    """infer with seed S == infer given the hook's dp noise (stream 1) and prior noise (stream 2) for S."""
    e = _engine("vits")
    ids, lens, sid = _vits_inputs(e)
    scales = np.array([0.667, 1.0, 0.8], np.float32)
    hint = 4096 if fused else None
    wav, y = e.infer(ids, lens, sid, scales, seed=S, frames_hint=hint)
    rows = int(R.offsets(lens)[-1])
    dp = e.debug_noise("dp", S, lens, np.zeros((2, rows), np.float32), scale=1.0)
    off = R.offsets(lens)
    noise_dp = np.zeros((3, 2, ids.shape[1]), np.float32)
    for b, n in enumerate(lens):
        noise_dp[b, :, :n] = dp[:, off[b]:off[b] + n]
    noise_z = _hook_noise(e, "prior", y, int(e.cfg["inter_channels"]))
    wav2, y2 = e.infer(ids, lens, sid, scales, noise_dp=noise_dp, noise_z=noise_z, seed=S ^ 1, frames_hint=hint)
    _same(y, y2)
    _same(wav, wav2)


def _clips(e):
    rng = np.random.default_rng(4)
    hop = int(e.cfg.get("hop_length", 256))
    lengths = np.array([61 * hop + 17, 23 * hop + 5], np.int64)
    wav = (0.1 * rng.standard_normal((2, int(lengths.max())))).astype(np.float32)
    return wav, lengths


def test_convert_seed_is_the_hooks_noise():
    """convert with seed S == convert given the hook's posterior noise (stream 3) for S."""
    e = _engine("vits")
    wav, lengths = _clips(e)
    out, frames = e.convert(wav, np.array([1, 2]), np.array([2, 0]), lengths, noise_scale=0.7, seed=S)
    eps = _hook_noise(e, "posterior", frames, int(e.cfg["inter_channels"]))
    out2, frames2 = e.convert(wav, np.array([1, 2]), np.array([2, 0]), lengths, noise_scale=0.7, noise=eps, seed=S ^ 1)
    _same(frames, frames2)
    _same(out, out2)


def test_align_seed_is_the_hooks_noise():
    """align with seed S == align given the hook's posterior noise for S (durations, token of frame and score)."""
    e = _engine("vits")
    wav, lengths = _clips(e)
    rng = np.random.default_rng(5)
    ids = rng.integers(1, int(e.cfg["n_vocab"]), (2, 20)).astype(np.int64)
    ids[:, 1::2] = 0
    tl = np.array([20, 15], np.int64)
    r1 = e.align(ids, tl, np.array([1, 2]), wav, lengths, seed=S)
    eps = _hook_noise(e, "posterior", r1[1], int(e.cfg["inter_channels"]))
    r2 = e.align(ids, tl, np.array([1, 2]), wav, lengths, noise=eps, seed=S ^ 1)
    for a, b in zip(r1, r2):
        _same(a, b)


def test_quickvc_convert_seed_is_the_hooks_noise():
    """quickvc_convert with seed S == quickvc_convert given the hook's posterior noise for S."""
    e = _engine("quickvc")
    rng = np.random.default_rng(6)
    units = [rng.standard_normal((n, 768)).astype(np.float32) for n in (37, 12, 64)]
    g = rng.standard_normal((3, int(e.cfg["gin_channels"]))).astype(np.float32)
    wav, frames = e.quickvc_convert(units, g, seed=S)
    eps = _hook_noise(e, "posterior", frames, int(e.cfg["inter_channels"]))
    wav2, frames2 = e.quickvc_convert(units, g, noise=eps, seed=S ^ 1)
    _same(frames, frames2)
    _same(wav, wav2)


def test_cfm_decode_seed_is_the_hooks_noise():
    """cfm_decode (guided: both branches) with seed S == cfm_decode given the hook's dit_init noise (stream 7) for S."""
    e = _engine("stabletts")
    NC, MC = int(e.cfg["noise_channels"]), int(e.cfg["cond_channels"])
    rng = np.random.default_rng(7)
    lens = [40, 7, 65]
    mu = [rng.standard_normal((n, MC)).astype(np.float32) for n in lens]
    kw = dict(sid=[0, 1, 0], n_timesteps=2, temperature=0.9, guidance_scale=0.5)
    mel, ml = e.cfm_decode(mu, seed=S, **kw)
    off = R.offsets(lens)
    rows = int(off[-1])
    xc, _, _ = e.debug_noise("dit", S, lens, np.zeros((2 * rows, NC + 1), np.float32), exts=lens, fake_content=np.zeros(1, np.float32),
                             mu=np.zeros((2 * rows, 1), np.float32), skx=np.zeros((2 * rows, 2), np.float32))
    noise = [xc[off[b]:off[b] + n, :NC] for b, n in enumerate(lens)]
    mel2, ml2 = e.cfm_decode(mu, noise=noise, seed=S ^ 1, **kw)
    _same(ml, ml2)
    _same(mel, mel2)
