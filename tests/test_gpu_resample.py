"""Resampling and trimming on the GPU (vtts_resample) against the float64 restatement (oracle/resample_oracle.py): every rate
pair of the CPU grid, ragged batches of up to 64 clips from 1 sample to 60 s, batch invariance, rows left untouched past each
clip, trim bounds, refusals, the front ends end to end, and the handle's memory after close()."""
import json
import wave

import numpy as np
import pytest

import contentvec_inputs as CI
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
import vc_inputs as VI
from oracle import resample_oracle as R
from vosk_tts_b200 import engine as E, quickvc, synthetic, weights

pytestmark = pytest.mark.gpu

RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000]
PAIRS = sorted({(a, b) for a in RATES for b in (16000, 22050) if a != b} | {(b, a) for a in RATES for b in (16000, 22050) if a != b})
# taps of every phase beyond shared memory (read through L2), the largest rate ratio, an equal-rate copy
EXTRA = [(384000, 44100), (384000, 4000), (4000, 384000), (16000, 16000)]
_ENG = {}


def _engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if "q" not in _ENG:
        blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
        _ENG["q"] = E.Engine(dict(QI.config(), contentvec=CI.cv()), blob, man, device=0, precision=1)
    return _ENG["q"]


def teardown_module(module):
    for e in _ENG.values():
        e.close()
    _ENG.clear()


def _raw(e, clips, fr, to, top_db=0.0, fill=np.nan):
    """vtts_resample on a padded batch whose output rows start as `fill`: (out rows, lengths, bounds)."""
    lens = np.array([c.size for c in clips], np.int64)
    x = np.zeros((len(clips), int(lens.max())), np.float32)
    for b, c in enumerate(clips):
        x[b, :c.size] = c
    ld = int(R.out_length(int(lens.max()), fr, to))
    out = np.full((len(clips), ld + 5), fill, np.float32)
    n = np.zeros(len(clips), np.int64)
    bnd = np.zeros((len(clips), 2), np.int64)
    e._check(e.lib.vtts_resample(e.h, E._ptr(x), E._ptr(lens), len(clips), x.shape[1], fr, to, float(top_db), E._ptr(out),
                                 out.shape[1], E._ptr(n), E._ptr(bnd)))
    return out, n, bnd


def _speechlike(n, rate, seed):
    """Band-limited noise bursts at speech levels (the kernels see every sample value; spectra only matter for the bound)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) * 0.2
    env = 0.5 + 0.5 * np.sin(2 * np.pi * np.arange(n) * 3.0 / rate)
    return (x * env).astype(np.float32)


def _check_batch(e, clips, fr, to):
    out, n, _ = _raw(e, clips, fr, to)
    worst = 0.0
    for b, c in enumerate(clips):
        m = R.out_length(c.size, fr, to)
        assert n[b] == m
        y = out[b, :m].astype(np.float64)
        err = np.abs(y - R.resample(c, fr, to))
        bnd = R.bound(c, fr, to)
        assert np.all(err <= bnd), (fr, to, c.size, float((err - bnd).max()))
        worst = max(worst, float((err / np.maximum(bnd, 1e-300)).max()))
        assert np.all(np.isnan(out[b, m:])), "row written past the clip"
        alone, n1, _ = _raw(e, [c], fr, to)
        assert n1[0] == m and np.array_equal(alone[0, :m], out[b, :m]), "clip differs alone and in the batch"
    return worst


@pytest.mark.parametrize("pair", PAIRS + EXTRA, ids=["%d-%d" % p for p in PAIRS + EXTRA])
def test_kernel_against_oracle(pair):
    """|engine - oracle| <= (K + 8) 2^-23 sum|h x| + 2^-24 sum|h||x| sample by sample (R.bound derives it: a K-term fp32 FMA
    chain over taps rounded to fp32 once); equal rates are exact."""
    e = _engine()
    fr, to = pair
    up, down = R.ratio(fr, to)
    half = 10 * max(up, down)
    lens = [1, 2, 3, max(4, half // up // 3), 101, 997, 7919, fr // 3, 2 * fr + 13]
    clips = [_speechlike(n, fr, 10 * i + fr % 97) for i, n in enumerate(lens)]
    worst = _check_batch(e, clips, fr, to)
    print("%d -> %d Hz: worst error / bound %.3f" % (fr, to, worst))


@pytest.mark.parametrize("pair", [(44100, 16000), (48000, 16000)])
def test_ragged_batch_of_64(pair):
    e = _engine()
    fr, to = pair
    rng = np.random.default_rng(fr)
    lens = list(rng.integers(2 * fr, 10 * fr, 62)) + [1, 60 * fr]
    clips = [_speechlike(int(n), fr, i) for i, n in enumerate(lens)]
    _check_batch(e, clips, fr, to)


def _tone(n, a, b, amp=0.5, period=16):
    y = np.zeros(n, np.float32)
    y[a:b] = amp * np.sin(2 * np.pi * np.arange(a, b) / period + 0.3)
    return y


CONSTRUCTED = [(_tone(16384, 4096, 8192), (3584, 9216)), (_tone(16384, 4000, 8300), (3072, 9728)),
               (_tone(16384, 4090, 8192), (3584, 9216)), (_tone(10000, 0, 10000), (0, 10000)),
               (_tone(16384, 0, 8192) + _tone(16384, 8192, 16384, amp=0.5 * 10 ** (-30 / 20)), (0, 9216))]


def test_trim_bounds_constructed():
    """At equal rates the clip is copied exactly, so the GPU's fp64 energies must give the hand-computed bounds."""
    e = _engine()
    clips = [c for c, _ in CONSTRUCTED]
    out, bounds = e.resample(clips, 16000, 16000, trim_top_db=20, return_bounds=True)
    for (c, want), y, bd in zip(CONSTRUCTED, out, bounds):
        assert tuple(bd) == want and np.array_equal(y, c[want[0]:want[1]])


def _speech_padded(rate):
    d = np.load(QI.GOLDEN + "/vc_speech.npz")
    out = []
    for k, (pre, post) in zip(("a", "b"), ((9000, 20000), (31337, 777))):
        s = R.resample(d[k].astype(np.float64) / 32768.0, 22050, rate)
        out.append(np.concatenate([np.zeros(pre), s, np.zeros(post)]).astype(np.float32))
    return out


@pytest.mark.parametrize("pair", [(44100, 16000), (48000, 22050), (16000, 16000)])
def test_trim_bounds_speech(pair):
    """Trim bounds from the GPU energies equal the float64 restatement's on the GPU's own resampled clip, and the kept part is
    that clip's [start, end)."""
    e = _engine()
    fr, to = pair
    clips = _speech_padded(fr)
    full = e.resample(clips, fr, to)
    out, bounds = e.resample(clips, fr, to, trim_top_db=20, return_bounds=True)
    for y, t, bd in zip(full, out, bounds):
        want = R.trim_bounds(R.frame_energies(y), y.size)
        assert tuple(bd) == want and 0 < want[0] < want[1] <= y.size
        assert np.array_equal(t, y[want[0]:want[1]])


def _code(fn):
    with pytest.raises(E.VttsError) as ex:
        fn()
    return ex.value.code, str(ex.value)


def test_refusals():
    e = _engine()
    x = _speechlike(1000, 16000, 0)
    for fr, to in [(3999, 16000), (16000, 384001), (0, 16000)]:
        if fr <= 0:
            with pytest.raises(ValueError):
                e.resample(x, fr, to)
            continue
        code, msg = _code(lambda: e.resample(x, fr, to))
        assert code == -1 and "sample rates" in msg
    code, msg = _code(lambda: e.resample(x, 22050, 32001))                  # up / down = 10667 / 7350: 213 341 taps
    assert code == -1 and "taps" in msg
    code, msg = _code(lambda: e.resample([x, np.zeros(3000, np.float32)], 16000, 16000, trim_top_db=20))
    assert code == -1 and "clip 1 is silent" in msg
    lens = np.array([1000], np.int64)
    out = np.zeros(100, np.float32)
    n = np.zeros(1, np.int64)
    assert e.lib.vtts_resample(e.h, E._ptr(x), E._ptr(lens), 1, 1000, 16000, 22050, 0.0, E._ptr(out), 100, E._ptr(n), None) == -4
    out, n, _ = _raw(e, [x], 16000, 22050)                                 # the handle still works
    assert n[0] == 1379


def test_works_on_a_vits2_engine(cfg):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 3)), cfg)
    e = E.Engine(cfg, blob, man, device=0, precision=0)
    try:
        x = _speechlike(4410, 44100, 1)
        y = e.resample(x, 44100, 22050)[0]
        assert np.all(np.abs(y - R.resample(x, 44100, 22050)) <= R.bound(x, 44100, 22050))
    finally:
        e.close()


def test_close_gives_back_everything():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    base = E.live_bytes()
    e = E.Engine(dict(QI.config(), contentvec=CI.cv()), blob, man, device=0, precision=1)
    for fr, to in [(44100, 16000), (48000, 16000), (16000, 22050), (384000, 44100), (22050, 22050)]:
        e.resample(_speech_padded(fr), fr, to, trim_top_db=20)
    now = E.live_bytes()
    assert now[0] > base[0] and now[1] > base[1]
    e.close()
    assert E.live_bytes() == base


# ---- end to end.  Each front end compares its resampled path with the same path fed the oracle's resampled clip.  The
# resampler's measured error `err` (max |engine - oracle| over the clip) is the only difference between the two inputs.  The
# model's sensitivity to such a difference is measured, not assumed: one probe run feeds the oracle's clip plus a seeded
# perturbation uniform in [-err, err] in every sample, and its output moves by d_probe.  The resampler's error is at most err
# per sample and mostly far below it, so it should move the output by no more than the probe does; the tolerance is
# PROBE_MARGIN * d_probe, the margin covering a direction the model amplifies more than the probe's.

PROBE_MARGIN = 4.0


def _probe(f, x, err, seed=0):
    """max |f(x + delta) - f(x)| for delta uniform in [-err, err]: the output change an input error of size err causes."""
    delta = np.random.default_rng(seed).uniform(-err, err, x.size)
    y0 = np.asarray(f(np.asarray(x, np.float32)), np.float64)
    y1 = np.asarray(f((np.asarray(x, np.float64) + delta).astype(np.float32)), np.float64)
    assert y0.shape == y1.shape
    return float(np.abs(y1 - y0).max())


def _resample_err(e, x, fr, to):
    y = e.resample(x, fr, to)[0]
    err = float(np.abs(y - R.resample(x, fr, to)).max())
    assert err <= 1e-5
    return max(err, 1e-7)


def _qvc():
    vc = quickvc.QuickVC.__new__(quickvc.QuickVC)
    vc.engine, vc.sampling_rate = _engine(), 16000
    return vc


def test_quickvc_embed_resampled_and_trimmed():
    vc = _qvc()
    x44 = _speech_padded(44100)[0]
    err = _resample_err(vc.engine, x44, 44100, 16000)
    g = vc.embed(x44, sampling_rate=44100, trim=True)
    ref_clip = R.trim(R.resample(x44, 44100, 16000))
    _, bnd = vc.engine.resample(x44, 44100, 16000, trim_top_db=20, return_bounds=True)
    assert int(bnd[0, 1] - bnd[0, 0]) == ref_clip.size
    g_ref = vc.engine.speaker_embedding(ref_clip.astype(np.float32))[0]
    d = float(np.abs(g - g_ref).max())
    probe = _probe(lambda c: vc.engine.speaker_embedding(c)[0], ref_clip, err)
    print("embed: resampler err %.2e, |g - g_oracle| %.2e, probe %.2e" % (err, d, probe))
    assert d <= PROBE_MARGIN * probe
    assert np.array_equal(vc.embed(x44, sampling_rate=44100, trim=True), g)


def test_quickvc_convert_48k_source():
    vc = _qvc()
    src = _speech_padded(48000)[1]
    err = _resample_err(vc.engine, src, 48000, 16000)
    g = vc.embed(_speech_padded(16000)[0])
    out = vc.convert(src, g=g, noise_scale=0.0, sampling_rate=48000)
    ref_src = R.resample(src, 48000, 16000)
    ref = vc.convert(ref_src.astype(np.float32), g=g, noise_scale=0.0)
    d = float(np.abs(out - ref).max())
    probe = _probe(lambda c: vc.convert(c, g=g, noise_scale=0.0), ref_src, err)
    print("convert: resampler err %.2e, |wav - wav_oracle| %.2e, probe %.2e" % (err, d, probe))
    assert out.shape == ref.shape and d <= PROBE_MARGIN * probe


def _synth(tmp_path):
    from vosk_tts_b200 import config as CF
    from vosk_tts_b200.model import Model
    from vosk_tts_b200.session import VitsSession
    from vosk_tts_b200.synth import Synth
    cfg = CF.from_training_json(VI.training_json("mel"), n_vocab=62)
    sd = synthetic.make_random_checkpoint(cfg, VI.SEEDS["mel"], posterior=True)
    sess = VitsSession(sd, cfg, precision=1, voice_conversion=True)
    ids = {p: i % 62 for i, p in enumerate(["_", "^", "$", " ", ",", "a", "b", "c", "d", "e", "h", "l", "o", "w", "r"])}
    (tmp_path / "config.json").write_text(json.dumps({"phoneme_id_map": ids}), encoding="utf-8")
    model = Model(str(tmp_path), session=sess)
    model.dic = {"hello": "h e l l o", "world": "w o r l d"}
    return Synth(model), sess


def _write(path, x, sr):
    with wave.open(str(path), "w") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.asarray(x, np.int16).tobytes())


def test_synth_convert_and_align_resampled(tmp_path):
    """A 44.1 kHz file with resample=True against the 22 050 Hz clip the oracle makes of it (noise_scale 0: the posterior
    mean, so both paths are deterministic)."""
    s, sess = _synth(tmp_path)
    try:
        x16 = np.clip(np.round(_speech_padded(44100)[0] * 32767), -32768, 32767).astype(np.int16)
        _write(tmp_path / "in44.wav", x16, 44100)
        xf = x16.astype(np.float32) / 32768.0
        err = _resample_err(sess.engine, xf, 44100, 22050)
        ref_in = np.clip(R.resample(xf, 44100, 22050), -1, 1).astype(np.float32)
        s.convert(str(tmp_path / "in44.wav"), str(tmp_path / "o.wav"), 0, 1, noise_scale=0.0, resample=True)
        with wave.open(str(tmp_path / "o.wav")) as f:
            assert f.getframerate() == 22050
            out = np.frombuffer(f.readframes(f.getnframes()), np.int16).astype(np.float64)
        ref = s.convert_audio(ref_in, 0, 1, noise_scale=0.0).astype(np.float64)
        d = float(np.abs(out - ref).max()) / 32767.0
        probe = _probe(lambda c: s.convert_audio(np.clip(c, -1, 1), 0, 1, noise_scale=0.0), ref_in, err) / 32767.0
        print("Synth.convert: resampler err %.2e, |out - out_oracle| %.2e, probe %.2e" % (err, d, probe))
        assert out.shape == ref.shape and d <= PROBE_MARGIN * probe + 1.0 / 32767.0    # + one LSB of the int16 rounding
        a = s.align(str(tmp_path / "in44.wav"), "hello, world", 0, noise_scale=0.0, resample=True)
        b = s.align_audio("hello, world", ref_in, 0, noise_scale=0.0)
        assert a == b, "alignment paths differ"
    finally:
        sess.close()
