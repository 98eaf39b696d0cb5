"""CPU: voice conversion host side -- the oracle restatement against the reference's stored outputs
(tests/golden/ref_voice_conversion.npz, oracle/make_golden_vc.py), the mel filter bank, configuration, enc_q packing, and the
Synth / CLI front end with a stub session in place of the GPU engine."""
import json
import os
import wave

import numpy as np
import pytest
import torch

import golden_ref as GR
import vc_inputs as VI
from oracle import vc_oracle as vo
from vosk_tts_b200 import cli, config as CF, synthetic, weights
from vosk_tts_b200.model import Model
from vosk_tts_b200.synth import Synth

CASES = {c[0]: c for c in VI.CASES}


def _cfg(model):
    return CF.from_training_json(VI.training_json(model), n_vocab=62 if model == "mel" else GR.N_VOCAB)


@pytest.mark.parametrize("case", ["c0", "c1", "c2"])
def test_oracle_front_end_matches_reference(case):
    ref = GR.load("ref_voice_conversion.npz")
    _, clip, _, _, model = CASES[case]
    d = VI.training_json(model)["data"]
    y = torch.from_numpy(VI.wav_float(VI.speech()[clip]))[None]
    lin = vo.spectrogram(y, d["filter_length"], d["hop_length"], d["win_length"])
    assert tuple(lin.shape) == tuple(ref[case + "/lin_shape"]) and lin.shape[2] == y.shape[1] // 256
    flat = lin.reshape(-1).numpy()
    assert float(np.abs(flat[ref[case + "/lin_idx"]] - ref[case + "/lin"]).max()) <= 1e-5 * float(np.abs(ref[case + "/lin"]).max())
    if model == "mel":
        mel = vo.mel_spectrogram(y, d["filter_length"], d["n_mel_channels"], d["sampling_rate"], d["hop_length"], d["win_length"],
                                 d["mel_fmin"], d["mel_fmax"])
        assert float(np.abs(mel[0].numpy() - ref[case + "/spec"]).max()) <= 1e-5


@pytest.mark.parametrize("case", ["c0", "c1", "c2"])
def test_oracle_voice_conversion_matches_reference(case):
    ref = GR.load("ref_voice_conversion.npz")
    _, clip, s, t, model = CASES[case]
    cfg = _cfg(model)
    w = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, VI.SEEDS[model], posterior=True))
    spec = torch.from_numpy(ref[case + "/spec"])[None]
    T = spec.shape[2]
    with torch.no_grad():
        r = vo.voice_conversion(w, cfg, spec, torch.tensor([T]), torch.tensor([s]), torch.tensor([t]),
                                VI.eps_q(case, cfg["inter_channels"], T))
    for nm, key in (("z", "z"), ("z_p", "z_p"), ("z_hat", "z_hat"), ("o_hat", "o_hat")):
        v = r[key].reshape(-1).numpy()
        assert tuple(r[key].shape) == tuple(ref[case + "/" + nm + "_shape"])
        err = float(np.abs(v[ref[case + "/" + nm + "_idx"]] - ref[case + "/" + nm]).max())
        assert err <= 1e-5, (nm, err)
    assert tuple(r["o_hat"].shape)[-1] == 256 * T


@pytest.mark.parametrize("sr,n_fft,n_mels,fmin,fmax", [(22050, 1024, 80, 0.0, None), (16000, 512, 40, 50.0, 7000.0)])
def test_mel_basis_matches_torchaudio(sr, n_fft, n_mels, fmin, fmax):
    torchaudio = pytest.importorskip("torchaudio")
    fb = torchaudio.functional.melscale_fbanks(n_fft // 2 + 1, fmin, sr / 2.0 if fmax is None else fmax, n_mels, sr,
                                               norm="slaney", mel_scale="slaney").T.numpy()
    for m in (weights.mel_basis(sr, n_fft, n_mels, fmin, fmax), vo.mel_basis(sr, n_fft, n_mels, fmin, fmax)):
        assert m.shape == (n_mels, n_fft // 2 + 1) and m.dtype == np.float32
        assert float(np.abs(m - fb).max()) <= 1e-5 * float(np.abs(fb).max())     # (torchaudio computes in float32)


def test_stft_basis_is_the_windowed_dft():
    n = 64
    b = weights.stft_basis(n).astype(np.float64)
    x = np.random.RandomState(0).randn(n)
    X = np.fft.rfft(x * (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)))
    y = x @ b
    assert np.allclose(y[0::2][1:], X.real[1:n // 2], atol=1e-5) and np.allclose(y[1::2][1:], X.imag[1:n // 2], atol=1e-5)
    assert abs(y[0] - X.real[0]) < 1e-5 and abs(y[1] - X.real[n // 2]) < 1e-5


def test_config_keys_and_defaults():
    d = CF.DEFAULT_CONFIG
    assert (d["filter_length"], d["hop_length"], d["win_length"], d["n_mel_channels"], d["mel_fmin"], d["mel_fmax"]) == \
        (1024, 256, 1024, 80, 0.0, None)
    assert d["use_mel_posterior_encoder"] and d["spec_channels"] == 80
    mel = _cfg("mel")
    assert mel["use_mel_posterior_encoder"] and mel["spec_channels"] == 80 and mel["mel_fmax"] is None
    lin = _cfg("lin")
    assert not lin["use_mel_posterior_encoder"] and lin["spec_channels"] == 513
    j = VI.training_json("mel")
    j["model"].pop("use_mel_posterior_encoder")          # onnx_export.py:38-45: the model block decides, data's flag is ignored
    assert not CF.from_training_json(j)["use_mel_posterior_encoder"]
    j["data"]["filter_length"], j["data"]["hop_length"] = 2048, 512
    c = CF.from_training_json(j)
    assert c["spec_channels"] == 1025 and c["hop_length"] == 512


@pytest.mark.parametrize("model", ["mel", "lin"])
def test_synthetic_enc_q_matches_reference_names_and_shapes(model):
    ref = GR.load("ref_voice_conversion.npz")
    cfg = _cfg(model)
    sd = synthetic.make_random_checkpoint(cfg, VI.SEEDS[model], posterior=True)
    names = sorted(k for k in sd if k.startswith("enc_q."))
    assert names == list(ref[model + "/encq_names"])
    assert [",".join(map(str, sd[k].shape)) for k in names] == list(ref[model + "/encq_shapes"])
    base = synthetic.make_random_checkpoint(cfg, VI.SEEDS[model])
    assert set(base) == set(sd) - set(names) and all(torch.equal(base[k], sd[k]) for k in base)


def test_default_pack_ignores_enc_q_and_posterior_pack_appends():
    cfg = _cfg("lin")
    w0 = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 5))
    w1 = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 5, posterior=True))
    b0, m0 = weights.pack(w0, cfg)
    b1, m1 = weights.pack(w1, cfg)
    assert m0 == m1 and np.array_equal(b0, b1)
    bp, mp = weights.pack(w1, cfg, posterior=True)
    assert mp.startswith(m0) and np.array_equal(bp[: b0.size], b0)
    names = [l.split()[0] for l in mp[len(m0):].splitlines()]
    assert "encq.pre.w" in names and "encq.in15.b" in names and "vc.stft" in names and "vc.mel" not in names
    pre = dict((l.split()[0], (int(l.split()[1]), int(l.split()[2]))) for l in mp.splitlines())["encq.pre.w"]
    assert pre[1] == 528 * cfg["hidden_channels"]                   # 513 input channels zero-padded to 528
    with pytest.raises(ValueError, match="enc_q"):
        weights.pack(w0, cfg, posterior=True)
    odd = dict(cfg, flow_n_flows=3)
    with pytest.raises(ValueError, match="flow_n_flows"):
        weights.pack(w1, odd, posterior=True)


class _StubSession:
    def __init__(self):
        self.calls = []
        self.cfg = {"sampling_rate": 22050}

    def convert(self, wav, src, tgt, noise=None, noise_scale=1.0):
        self.calls.append((wav, src, tgt, noise_scale))
        n = 256 * (wav.size // 256)
        return np.linspace(-1.5, 1.5, n, dtype=np.float32)


def _model(tmp_path):
    (tmp_path / "config.json").write_text(json.dumps({"phoneme_id_map": {"_": [0]}, "inference": {"scale": 0.5}}), encoding="utf-8")
    sess = _StubSession()
    return Model(str(tmp_path), session=sess), sess


def _write_wav(path, x, sr=22050):
    with wave.open(str(path), "w") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.asarray(x, np.int16).tobytes())


def test_convert_audio_scales_int16_and_checks_inputs(tmp_path):
    model, sess = _model(tmp_path)
    s = Synth(model)
    a = (np.arange(1000) % 200 - 100).astype(np.int16) * 300
    out = s.convert_audio(a, 3, 7)
    wav, src, tgt, ns = sess.calls[-1]
    assert np.array_equal(wav, a.astype(np.float32) / 32768.0) and (src, tgt, ns) == (3, 7, 1.0)
    assert out.dtype == np.int16 and out.size == 768 and out.max() == int(0.75 * 32767)      # config scale 0.5
    s.convert_audio(a.astype(np.float32) / 40000.0, 0, 1, noise_scale=0.3)
    assert sess.calls[-1][3] == 0.3
    with pytest.raises(ValueError):
        s.convert_audio(np.array([0.5, 1.5], np.float32), 0, 1)
    with pytest.raises(ValueError):
        s.convert_audio(np.zeros((2, 100), np.int16), 0, 1)
    with pytest.raises(ValueError):
        s.convert_audio(np.zeros(100, np.int32), 0, 1)
    with pytest.raises(ValueError):
        s.convert_audio(np.zeros(1000, np.int16), None, 1)


def test_convert_wav_files_and_sample_rate_check(tmp_path):
    model, sess = _model(tmp_path)
    s = Synth(model)
    _write_wav(tmp_path / "in.wav", np.arange(1000) % 50)
    s.convert(str(tmp_path / "in.wav"), str(tmp_path / "out.wav"), 2, 5)
    with wave.open(str(tmp_path / "out.wav")) as f:
        assert (f.getframerate(), f.getnchannels(), f.getsampwidth(), f.getnframes()) == (22050, 1, 2, 768)
    _write_wav(tmp_path / "in16k.wav", np.zeros(1000), sr=16000)
    with pytest.raises(ValueError, match="resample"):
        s.convert(str(tmp_path / "in16k.wav"), str(tmp_path / "o.wav"), 2, 5)


def test_cli_convert_arguments(tmp_path, monkeypatch):
    seen = {}

    class _M:
        def __init__(self, *a, **k):
            seen["model"] = k

    class _S:
        def __init__(self, m):
            pass

        def convert(self, i, o, src, tgt):
            seen["convert"] = (i, o, src, tgt)

    monkeypatch.setattr(cli, "Model", _M)
    monkeypatch.setattr(cli, "Synth", _S)
    assert cli.main(["-m", "x", "--convert-from", "in.wav", "--source-speaker", "3", "-s", "7", "-o", "out.wav"]) == 0
    assert seen["convert"] == ("in.wav", "out.wav", 3, 7) and seen["model"]["voice_conversion"] is True
    with pytest.raises(SystemExit):
        cli.main(["-m", "x", "--convert-from", "in.wav", "-s", "7"])


def test_onnx_model_directory_refuses_voice_conversion(tmp_path):
    import shutil
    shutil.copyfile(os.path.join(GR.GOLDEN, "tiny_model.onnx"), tmp_path / "model.onnx")
    (tmp_path / "config.json").write_text(json.dumps({"phoneme_id_map": {"_": [0]}}), encoding="utf-8")
    with pytest.raises(ValueError, match="enc_q"):
        Model(str(tmp_path), voice_conversion=True)
