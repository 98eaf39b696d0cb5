"""Stores the reference QuickVC speaker embedding (SpeakerEncoder.embed_utterance on mel_spectrogram_torch of the target, as
SynthesizerTrn.infer computes g, vc/models.py:862-865) for the GPU and CPU tests, so that they run without the reference tree.

Run where the reference tree is present (``python oracle/make_golden_quickvc.py``); writes ONLY these new files under
tests/golden/:
  quickvc_targets.npz   int16 16 kHz slices of three clips of the reference tree (vc/test_data), tests/quickvc_inputs.TARGETS
  ref_quickvc.npz       per target: the reference log-mel and g; the sorted enc_spk.* names and shapes of the reference model
The model classes come from the unmodified vc/models.py.  librosa is not installed: ``librosa.util`` is the shim of
ref_harness and ``librosa.filters.mel`` the restatement ``vosk_tts_b200.weights.mel_basis``; current SciPy has ``kaiser``
only as ``scipy.signal.windows.kaiser`` (vc/pqmf.py imports ``scipy.signal.kaiser``).
"""
import contextlib
import io
import os
import sys
import types
import wave

import numpy as np
import scipy.signal
import scipy.signal.windows
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as rh  # noqa: E402
from vosk_tts_b200 import weights  # noqa: E402
import quickvc_inputs as QI  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_VC = os.path.join(rh.REF_ROOT, "vc")


def import_reference_vc():
    rh._install_shims()
    filters = types.ModuleType("librosa.filters")
    filters.mel = lambda sr, n_fft, n_mels, fmin, fmax: weights.mel_basis(sr, n_fft, n_mels, fmin, fmax)
    sys.modules["librosa"].filters = filters
    sys.modules["librosa.filters"] = filters
    scipy.signal.kaiser = scipy.signal.windows.kaiser
    sys.path.insert(0, REF_VC)
    import models            # the reference's vc/models.py
    import mel_processing    # vc/mel_processing.py
    return models, mel_processing


def write_targets():
    out, names = {}, []
    for key, fn, start, n in QI.TARGETS:
        with wave.open(os.path.join(REF_VC, "test_data", fn)) as f:
            assert f.getframerate() == 16000 and f.getnchannels() == 1 and f.getsampwidth() == 2
            x = np.frombuffer(f.readframes(f.getnframes()), np.int16)
        assert start + n <= x.size
        out[key] = x[start:start + n].copy()
        names.append("%s=%s[%d:%d]" % (key, fn, start, start + n))
    out["sources"] = np.array(names)
    np.savez_compressed(os.path.join(GOLDEN, "quickvc_targets.npz"), **out)


def main():
    assert os.path.isfile(os.path.join(REF_VC, "models.py")), "needs the reference tree"
    torch.set_num_threads(4)
    write_targets()
    models, mp = import_reference_vc()
    hps = QI.QUICKVC_JSON
    d = hps["data"]
    with contextlib.redirect_stdout(io.StringIO()):
        net = models.SynthesizerTrn(d["filter_length"] // 2 + 1, 10240 // d["hop_length"], **hps["model"]).eval()
    keys = sorted(k for k in net.state_dict() if k.startswith("enc_spk."))
    out = {"enc_spk_names": np.array(keys),
           "enc_spk_shapes": np.array([",".join(map(str, net.state_dict()[k].shape)) for k in keys])}
    sd = QI.speaker_encoder()
    missing, unexpected = net.load_state_dict(sd, strict=False)
    assert not unexpected and not [k for k in missing if k.startswith("enc_spk.")]
    for key, wav in QI.targets().items():
        y = torch.from_numpy(QI.wav_float(wav))[None]
        mel = mp.mel_spectrogram_torch(y, d["filter_length"], d["n_mel_channels"], d["sampling_rate"], d["hop_length"],
                                       d["win_length"], d["mel_fmin"], d["mel_fmax"])
        with torch.no_grad():
            g = net.enc_spk.embed_utterance(mel.transpose(1, 2))
        out[key + "/mel"] = mel[0].numpy().astype(np.float32)
        out[key + "/g"] = g[0].numpy().astype(np.float32)
    np.savez_compressed(os.path.join(GOLDEN, "ref_quickvc.npz"), **out)


if __name__ == "__main__":
    main()
