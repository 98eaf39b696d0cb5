"""CPU: the resampler's float64 restatement against scipy.signal.resample_poly, the trim restatement on constructed clips
with hand-computed bounds, the opt-in resampling of the Synth / QuickVC front ends and CLIs with stub sessions in place of
the GPU engine (their defaults still refuse a wrong-rate file), and the C entry point."""
import ctypes
import json
import os
import wave

import numpy as np
import pytest
import scipy.signal

import quickvc_inputs as QI
from oracle import resample_oracle as R
from vosk_tts_b200 import cli, engine as E, quickvc
from vosk_tts_b200.model import Model
from vosk_tts_b200.synth import Synth

RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000]
PAIRS = sorted({(a, b) for a in RATES for b in (16000, 22050) if a != b} | {(b, a) for a in RATES for b in (16000, 22050) if a != b})


def _lengths(from_rate, to_rate):
    up, down = R.ratio(from_rate, to_rate)
    half = 10 * max(up, down)
    return [1, 2, max(3, half // 3), 101, 997, 7919, 10 * from_rate]


@pytest.mark.parametrize("pair", PAIRS, ids=["%d-%d" % p for p in PAIRS])
def test_oracle_is_resample_poly(pair):
    fr, to = pair
    up, down = R.ratio(fr, to)
    rng = np.random.default_rng(fr * 7 + to)
    for n in _lengths(fr, to):
        x = rng.standard_normal(n)
        ref = scipy.signal.resample_poly(x, up, down)
        y = R.resample(x, fr, to)
        assert y.shape == ref.shape == (R.out_length(n, fr, to),)
        assert float(np.abs(y - ref).max()) <= 1e-12, (n, float(np.abs(y - ref).max()))


def test_taps_are_firwin():
    for up, down in [(160, 441), (441, 160), (1, 2), (147, 640)]:
        M = max(up, down)
        ref = scipy.signal.firwin(2 * 10 * M + 1, 1.0 / M, window=("kaiser", 5.0)) * up
        assert float(np.abs(R.taps(up, down) - ref).max()) <= 1e-15 * up
        P = R.polyphase(up, down)
        assert P.shape == (up, -(-(20 * M + 1) // up)) and np.array_equal(P.T.reshape(-1)[:20 * M + 1], R.taps(up, down))
    assert R.taps(160, 441).size == 8821 and R.polyphase(160, 441).size * 4 == 35840        # 44.1 -> 16 kHz: 35 KB of taps


def _tone(n, a, b, amp=0.5, period=16):
    y = np.zeros(n)
    t = np.arange(a, b)
    y[a:b] = amp * np.sin(2 * np.pi * t / period + 0.3)
    return y


@pytest.mark.parametrize("clip,bounds", [
    (_tone(16384, 4096, 8192), (3584, 9216)),       # edges on frame boundaries: the frames overlapping by 512 are at -6 dB
    (_tone(16384, 4000, 8300), (3072, 9728)),       # off the boundaries: 96 and 108 samples of overlap are at -13 dB
    (_tone(16384, 4090, 8192), (3584, 9216)),       # 6 samples of overlap (-25 dB) do not keep frame 6
    (_tone(10000, 0, 10000), (0, 10000)),           # no silence: the last frame's end is clipped to the clip
    (_tone(16384, 0, 8192) + _tone(16384, 8192, 16384, amp=0.5 * 10 ** (-30 / 20)), (0, 9216)),   # a tail 30 dB down is cut
])
def test_trim_bounds(clip, bounds):
    e = R.frame_energies(clip)
    assert e.size == 1 + clip.size // 512
    assert R.trim_bounds(e, clip.size) == bounds
    assert np.array_equal(R.trim(clip), clip[bounds[0]:bounds[1]])


def test_trim_refuses_digital_silence():
    assert R.trim(np.zeros(5000)) is None
    assert R.trim(np.full(5000, 1e-6)) is None                       # mean square 1e-12 <= 1e-10
    assert R.trim(np.full(5000, 1e-4)) is not None


def test_frame_energies_are_centred_frames():
    y = np.random.default_rng(3).standard_normal(5000)
    pad = np.pad(y, 1024)
    ref = [np.sum(pad[512 * f:512 * f + 2048] ** 2) for f in range(1 + 5000 // 512)]
    assert np.allclose(R.frame_energies(y), ref, rtol=1e-13, atol=0)


# ---- front ends with stub sessions

class _StubSession:
    def __init__(self):
        self.calls, self.resampled = [], []
        self.cfg = {"sampling_rate": 22050}

    def resample(self, wav, from_rate, to_rate):
        self.resampled.append((np.array(wav), from_rate, to_rate))
        return np.asarray(wav, np.float32)[: R.out_length(wav.size, from_rate, to_rate)] * 0.5

    def convert(self, wav, src, tgt, noise=None, noise_scale=1.0):
        self.calls.append(("convert", wav))
        return np.zeros(256 * (wav.size // 256), np.float32)

    def align(self, ids, wav, sid=0, noise=None, noise_scale=1.0):
        self.calls.append(("align", wav))
        dur = np.ones(len(ids), np.int32)
        return dur, np.arange(len(ids), dtype=np.int32), -1.0


def _model(tmp_path):
    (tmp_path / "config.json").write_text(json.dumps({"phoneme_id_map": {"^": 1, "$": 2, "_": 0}}), encoding="utf-8")
    sess = _StubSession()
    return Model(str(tmp_path), session=sess), sess


def _write(path, x, sr, channels=1):
    with wave.open(str(path), "w") as f:
        f.setnchannels(channels)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.asarray(x, np.int16).tobytes())


def test_synth_defaults_still_refuse_other_rates(tmp_path):
    model, sess = _model(tmp_path)
    s = Synth(model)
    _write(tmp_path / "a.wav", np.zeros(3000), 44100)
    with pytest.raises(ValueError, match="resample it first"):
        s.convert(str(tmp_path / "a.wav"), str(tmp_path / "o.wav"), 0, 1)
    with pytest.raises(ValueError, match="resample it first"):
        s.align(str(tmp_path / "a.wav"), "", 0)
    _write(tmp_path / "st.wav", np.zeros(6000), 22050, channels=2)
    with pytest.raises(ValueError, match="mono"):
        s.convert(str(tmp_path / "st.wav"), str(tmp_path / "o.wav"), 0, 1)
    assert sess.resampled == []
    s.convert_audio(np.zeros(3000, np.int16), 0, 1)
    s.convert_audio(np.zeros(3000, np.int16), 0, 1, sampling_rate=22050)       # the model's rate: nothing to do
    assert sess.resampled == []


def test_synth_resample_opt_in(tmp_path):
    model, sess = _model(tmp_path)
    s = Synth(model)
    rng = np.random.default_rng(0)
    st = rng.integers(-20000, 20000, size=(4410, 2)).astype(np.int16)
    _write(tmp_path / "st.wav", st.reshape(-1), 44100, channels=2)
    mono = (st.astype(np.float64) / 32768.0).mean(axis=1).astype(np.float32)       # librosa.load(mono=True)
    s.convert(str(tmp_path / "st.wav"), str(tmp_path / "o.wav"), 0, 1, resample=True)
    wav, fr, to = sess.resampled[-1]
    assert (fr, to) == (44100, 22050) and np.array_equal(wav, mono)
    assert np.array_equal(sess.calls[-1][1], mono[:2205] * 0.5)                   # the session's resampled clip is converted
    with wave.open(str(tmp_path / "o.wav")) as f:
        assert f.getframerate() == 22050
    s.align(str(tmp_path / "st.wav"), "", 0, resample=True)
    assert sess.resampled[-1][1:] == (44100, 22050) and np.array_equal(sess.calls[-1][1], mono[:2205] * 0.5)
    a = rng.integers(-300, 300, 1600).astype(np.int16)
    s.align_audio("", a, sampling_rate=16000)
    assert sess.resampled[-1][1:] == (16000, 22050) and np.array_equal(sess.resampled[-1][0], a / np.float32(32768.0))
    s.convert_audio(a, 0, 1, sampling_rate=48000)
    assert sess.resampled[-1][1:] == (48000, 22050)


class _StubEngine:
    def __init__(self):
        self.resampled = []
        self.hop = 320

    def resample(self, clips, from_rate, to_rate, trim_top_db=None):
        self.resampled.append(([np.array(c) for c in clips], from_rate, to_rate, trim_top_db))
        return [np.asarray(c, np.float32)[::2] for c in clips]

    def speaker_embedding(self, wav):
        self.embedded = np.array(wav)
        return np.ones((1, 256), np.float32)

    def content_units(self, clips):
        self.unit_clips = [np.array(c) for c in clips]
        return np.zeros((len(clips), 3, 768), np.float32), np.full(len(clips), 3)

    def quickvc_convert_wav(self, clips, g, noise_scale=1.0, seed=0):
        self.conv_clips = [np.array(c) for c in clips]
        return np.zeros((len(clips), 960), np.float32), np.full(len(clips), 3)


def _qvc():
    vc = quickvc.QuickVC.__new__(quickvc.QuickVC)
    vc.engine, vc.sampling_rate = _StubEngine(), 16000
    return vc


def test_quickvc_opt_in():
    vc = _qvc()
    x = np.linspace(-0.5, 0.5, 4410).astype(np.float32)
    vc.embed(x)
    assert vc.engine.resampled == [] and np.array_equal(vc.engine.embedded, x)        # default: as before
    vc.embed(np.stack([x, x]))
    assert vc.engine.resampled == [] and vc.engine.embedded.shape == (2, 4410)          # a batch reaches the engine as one
    vc.embed(x, trim=True)
    assert vc.engine.resampled[-1][1:] == (16000, 16000, 20.0)                      # trim alone: convert.py's top_db=20
    vc.embed(x, sampling_rate=44100, trim=True)
    clips, fr, to, top = vc.engine.resampled[-1]
    assert (fr, to, top) == (44100, 16000, 20.0) and np.array_equal(clips[0], x) and np.array_equal(vc.engine.embedded, x[::2])
    vc.embed(x, sampling_rate=44100)
    assert vc.engine.resampled[-1][1:] == (44100, 16000, None)
    n = len(vc.engine.resampled)
    vc.units([x, x[:3000]])
    vc.convert(x, g=np.ones(256, np.float32))
    assert len(vc.engine.resampled) == n
    vc.units([x, x[:3000]], sampling_rate=48000)
    assert vc.engine.resampled[-1][1:] == (48000, 16000, None) and [c.size for c in vc.engine.unit_clips] == [2205, 1500]
    vc.convert([x], target_wav=x, sampling_rate=22050)
    assert [r[1:] for r in vc.engine.resampled[-2:]] == [(22050, 16000, None)] * 2 and vc.engine.conv_clips[0].size == 2205


def test_quickvc_cli_flags(tmp_path, monkeypatch, capsys):
    cfgp = tmp_path / "quickvc.json"
    cfgp.write_text(json.dumps(QI.QUICKVC_JSON))
    _write(tmp_path / "t44.wav", np.arange(4410) % 100, 44100, channels=2)
    _write(tmp_path / "s48.wav", np.arange(4800) % 100, 48000)
    _write(tmp_path / "s22.wav", np.arange(2205) % 100, 22050)
    _write(tmp_path / "t48.wav", np.arange(3000) % 100, 48000)
    base = ["--config", str(cfgp), "--checkpoint", str(tmp_path / "G.pth"), "--out-dir", str(tmp_path / "o"),
            "--target", str(tmp_path / "t44.wav")]
    units = tmp_path / "u.npy"
    np.save(units, np.zeros((5, 768), np.float32))
    with pytest.raises(SystemExit):
        quickvc.main(base + ["--units", str(units)])                                 # no --resample: refused as before
    assert "44100 Hz" in capsys.readouterr().err
    seen = {}

    class _QVC:
        sampling_rate = 16000

        def __init__(self, *a, **k):
            pass

        def embed(self, wav, sampling_rate=None, trim=False):
            seen["embed"] = (wav.size, sampling_rate, trim)
            return np.zeros(256, np.float32)

        def resample(self, clips, rate):
            seen.setdefault("sources", []).append(([c.size for c in clips], rate))
            return [c[::3] for c in clips]

        def convert(self, units, g=None, seed=0):
            seen["convert"] = [u.shape for u in units]
            return [np.zeros(10, np.float32) for _ in units]

        def close(self):
            pass

    monkeypatch.setattr(quickvc, "QuickVC", _QVC)
    assert quickvc.main(base + ["--units", str(units), "--resample", "--trim-target"]) == 0
    assert seen["embed"] == (2205, 44100, True) and seen["convert"] == [(5, 768)] and "sources" not in seen
    srcs = [str(tmp_path / n) for n in ("s48.wav", "s22.wav", "t48.wav")]
    assert quickvc.main(base + ["--source"] + srcs + ["--contentvec", "cv", "--resample"]) == 0
    # one ragged call per rate, and the converted clips keep the order of --source
    assert seen["embed"] == (2205, 44100, False) and seen["sources"] == [([2205], 22050), ([4800, 3000], 48000)]
    assert seen["convert"] == [(1600,), (735,), (1000,)]


def test_vosk_cli_resample_flag(monkeypatch):
    seen = {}

    class _M:
        def __init__(self, *a, **k):
            pass

    class _S:
        def __init__(self, m):
            pass

        def convert(self, i, o, src, tgt, **k):
            seen["convert"] = k

        def align(self, wav, text, speaker_id=None, **k):
            seen["align"] = k
            return []

    monkeypatch.setattr(cli, "Model", _M)
    monkeypatch.setattr(cli, "Synth", _S)
    cli.main(["-m", "x", "--convert-from", "in.wav", "--source-speaker", "3", "-s", "7"])
    cli.main(["-m", "x", "--align", "in.wav", "-i", "hello"])
    assert seen == {"convert": {}, "align": {}}
    cli.main(["-m", "x", "--convert-from", "in.wav", "--source-speaker", "3", "-s", "7", "--resample"])
    cli.main(["-m", "x", "--align", "in.wav", "-i", "hello", "--resample"])
    assert seen == {"convert": {"resample": True}, "align": {"resample": True}}


def test_c_abi_declares_and_exports_resample():
    with open(os.path.join(os.path.dirname(E._build.CSRC), "..", "include", "vtts.h")) as f:
        h = f.read()
    assert ("int vtts_resample(vtts_handle h, const float* wav, const int64_t* lengths, int B, int64_t ld, int from_rate, "
            "int to_rate,\n                  float trim_top_db, float* out, int64_t out_ld, int64_t* out_lengths, "
            "int64_t* trim_bounds);") in h
    assert "vtts_resample" in E.EXPORTS
    assert hasattr(ctypes.CDLL(E.lib_path()), "vtts_resample")
