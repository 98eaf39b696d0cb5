"""Stores the reference's voice conversion (SynthesizerTrn.voice_conversion, training/vits2/models.py:1710-1718) for the
GPU and CPU tests, so that they run without the reference tree.

Run where the reference tree is present (``python oracle/make_golden_vc.py``); writes ONLY these new files under
tests/golden/:
  vc_speech.npz              int16 slices of two LJSpeech clips of the reference tree (vc/test_data, public domain)
  ref_voice_conversion.npz   per case of tests/vc_inputs.CASES: the reference spectrogram_torch / mel_spectrogram_torch
                             output, z / z_p / z_hat and o_hat (sampled with golden_ref.sample_index), and the sorted enc_q.*
                             names and shapes of the reference model.
librosa is not installed: ``librosa.filters.mel`` is replaced, inside this script only, by the restatement
``vosk_tts_b200.weights.mel_basis`` (pinned against torchaudio by tests/test_voice_conversion_host.py).
"""
import contextlib
import io
import os
import sys
import types
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as rh  # noqa: E402
from vosk_tts_b200 import config as C, synthetic, weights  # noqa: E402
import golden_ref as GR  # noqa: E402
import vc_inputs as VI  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SPEECH = [("a", "LJ001-0001.wav", 22050, 2 * 22050 + 57), ("b", "LJ032-0032.wav", 11025, 28665 + 33)]


def write_speech():
    out, names = {}, []
    for key, fn, start, n in SPEECH:
        with wave.open(os.path.join(rh.REF_ROOT, "vc", "test_data", fn)) as f:
            assert f.getframerate() == 22050 and f.getnchannels() == 1 and f.getsampwidth() == 2
            x = np.frombuffer(f.readframes(f.getnframes()), np.int16)
        out[key] = x[start:start + n].copy()
        assert n % 256 != 0
        names.append("%s=%s[%d:%d]" % (key, fn, start, start + n))
    out["sources"] = np.array(names)
    np.savez_compressed(os.path.join(GOLDEN, "vc_speech.npz"), **out)


def reference_mel_processing():
    filters = types.ModuleType("librosa.filters")
    filters.mel = lambda sr, n_fft, n_mels, fmin, fmax: weights.mel_basis(sr, n_fft, n_mels, fmin, fmax)
    rh._install_shims()
    sys.modules["librosa"].filters = filters
    sys.modules["librosa.filters"] = filters
    rh.import_reference()
    import mel_processing            # the reference's module (training/vits2/mel_processing.py)
    return mel_processing


def build_reference_model(state_dict, cfg, n_vocab, spec_channels):
    """ref_harness.build_reference_model with the posterior encoder's input width as a parameter (that builder fixes it at
    80 mel channels; the linear-spectrogram case needs filter_length // 2 + 1): SynthesizerTrn as the exporter builds it
    (onnx_export.py:47-55,78-79), checkpoint loaded, weight norm removed on dec and flow, eval()."""
    models = rh.import_reference()
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(1234)
        net = models.SynthesizerTrn(n_vocab, spec_channels, cfg["train"]["segment_size"] // cfg["data"]["hop_length"],
                                    n_speakers=cfg["data"]["n_speakers"], is_onnx=True, **cfg["model"])
        missing, unexpected = net.load_state_dict(state_dict, strict=False)
        assert not unexpected, unexpected
        net.eval()
        net.dec.remove_weight_norm()
        net.flow.remove_weight_norm()
    return net


def main():
    assert rh.available(), "needs the reference tree"
    torch.set_num_threads(4)
    write_speech()
    mp = reference_mel_processing()
    clips = VI.speech()
    out = {}
    nets = {}
    for case, clip, s_src, s_tgt, model in VI.CASES:
        tj = VI.training_json(model)
        n_vocab = 62 if model == "mel" else GR.N_VOCAB
        cfg = C.from_training_json(tj, n_vocab=n_vocab)
        if model not in nets:
            sd = synthetic.make_random_checkpoint(cfg, VI.SEEDS[model], posterior=True)
            net = build_reference_model(sd, tj, n_vocab, cfg["spec_channels"])
            keys = sorted(k for k in net.state_dict() if k.startswith("enc_q."))
            out[model + "/encq_names"] = np.array(keys)
            out[model + "/encq_shapes"] = np.array([",".join(map(str, net.state_dict()[k].shape)) for k in keys])
            net.enc_q.enc.remove_weight_norm()           # modules.py:178-184
            nets[model] = net
        net = nets[model]
        d = tj["data"]
        y = torch.from_numpy(VI.wav_float(clips[clip]))[None]
        lin = mp.spectrogram_torch(y, d["filter_length"], d["sampling_rate"], d["hop_length"], d["win_length"], center=False)
        if cfg["use_mel_posterior_encoder"]:
            spec = mp.mel_spectrogram_torch(y, d["filter_length"], d["n_mel_channels"], d["sampling_rate"], d["hop_length"],
                                            d["win_length"], d["mel_fmin"], d["mel_fmax"], center=False)
        else:
            spec = lin
        T = spec.shape[2]
        eps = VI.eps_q(case, cfg["inter_channels"], T)
        calls = {"n": 0}
        orig = torch.randn_like

        def randn_like(x, **kw):
            calls["n"] += 1
            assert calls["n"] == 1 and tuple(x.shape) == tuple(eps.shape)
            return eps.clone()

        torch.randn_like = randn_like
        try:
            with torch.no_grad():
                o_hat, _, y_mask, (z, z_p, z_hat) = net.voice_conversion(spec, torch.tensor([T]), torch.tensor([s_src]),
                                                                         torch.tensor([s_tgt]))
        finally:
            torch.randn_like = orig
        out[case + "/spec"] = spec[0].numpy().astype(np.float32)
        l = lin.reshape(-1).numpy().astype(np.float32)
        out[case + "/lin_shape"] = np.array(lin.shape)
        out[case + "/lin_idx"] = GR.sample_index(l.size, case + "lin")
        out[case + "/lin"] = l[out[case + "/lin_idx"]]
        for nm, t in (("z", z), ("z_p", z_p), ("z_hat", z_hat), ("o_hat", o_hat)):
            v = t.reshape(-1).numpy().astype(np.float32)
            out[case + "/" + nm + "_shape"] = np.array(t.shape)
            out[case + "/" + nm + "_idx"] = GR.sample_index(v.size, case + nm)
            out[case + "/" + nm] = v[out[case + "/" + nm + "_idx"]]
            out[case + "/" + nm + "_absmax"] = np.float32(np.abs(v).max())
    np.savez_compressed(os.path.join(GOLDEN, "ref_voice_conversion.npz"), **out)


if __name__ == "__main__":
    main()
