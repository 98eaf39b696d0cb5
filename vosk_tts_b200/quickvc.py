"""QuickVC any-to-any voice conversion (vc/ of the reference: SynthesizerTrn.infer, vc/models.py:862-872, as vc/convert.py
runs it) on the GPU: content units of a source recording and a target voice in, a 16 kHz waveform out.

    vc = QuickVC("quickvc.json", "G_quickvc.pth")
    g = vc.embed(target_wav)                       # once per target voice
    wav = vc.convert(units, g=g)                    # units: ContentVec last_hidden_state [T, 768] (vc/encode.py's .npy)

ContentVec itself is not part of this package: the units come from vc/encode.py.  Unlike convert.py, the target recording
is not trimmed of silence (librosa.effects.trim(top_db=20)); trim it before embedding for the same g.

CLI:  python -m vosk_tts_b200.quickvc --config quickvc.json --checkpoint G.pth --units a.npy b.npy --target tgt.wav --out-dir out
writes out/<units file name>.wav, 16 kHz int16, clipped to the int16 range (convert.py's astype(int16) wraps instead).
"""
import argparse
import os
import sys
import wave

import numpy as np

from . import config as _config, weights as _weights


def read_wav(path, sampling_rate=16000):
    """Mono 16-bit PCM WAV -> float32 in [-1, 1]; refuses any other rate (the model is trained at `sampling_rate`)."""
    with wave.open(path, "rb") as f:
        sr, ch, sw = f.getframerate(), f.getnchannels(), f.getsampwidth()
        if sr != sampling_rate:
            raise ValueError("%s is sampled at %d Hz; the model needs %d Hz (resample it first)" % (path, sr, sampling_rate))
        if ch != 1 or sw != 2:
            raise ValueError("%s: only mono 16-bit PCM WAV files are read" % path)
        x = np.frombuffer(f.readframes(f.getnframes()), np.int16)
    return (x.astype(np.float32) / 32768.0).astype(np.float32)


def write_wav(path, wav, sampling_rate=16000):
    """float waveform -> 16-bit PCM WAV: wav * 32768 as convert.py scales it, clipped to the int16 range."""
    x = np.clip(np.round(np.asarray(wav, np.float64) * 32768.0), -32768, 32767).astype(np.int16)
    with wave.open(path, "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sampling_rate)
        f.writeframes(x.tobytes())


class QuickVC:
    """A QuickVC checkpoint on one GPU: the speaker encoder for targets and the conversion of content units."""

    def __init__(self, config, checkpoint, device=0, precision=1):
        from .engine import Engine
        self.cfg = _config.from_quickvc_json(config)
        sd = _weights.load_checkpoint(checkpoint)
        blob, man = _weights.pack_quickvc(sd, self.cfg, precision=precision)
        self.engine = Engine(self.cfg, blob, man, device=device, precision=precision)
        self.sampling_rate = int(self.cfg["sampling_rate"])

    def embed(self, target_wav):
        """The target voice g [256] of a recording (float [-1, 1] at the model's rate)."""
        return self.engine.speaker_embedding(np.asarray(target_wav, np.float32))[0]

    def convert(self, units, target_wav=None, g=None, noise_scale=1.0, seed=0):
        """Units [T, 768] (or a list of them) in the voice of g, or of target_wav's g: float32 waveform(s) at the model's rate."""
        if g is None:
            if target_wav is None:
                raise ValueError("convert needs a target: target_wav or g")
            g = self.embed(target_wav)
        single = not isinstance(units, (list, tuple))
        clips = [units] if single else list(units)
        wav, frames = self.engine.quickvc_convert(clips, g, noise_scale=noise_scale, seed=seed)
        out = [wav[b, :int(frames[b]) * self.engine.hop] for b in range(len(clips))]
        return out[0] if single else out

    def close(self):
        self.engine.close()


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m vosk_tts_b200.quickvc", description="QuickVC voice conversion on the GPU")
    ap.add_argument("--config", required=True, help="QuickVC config json (vc/configs/quickvc.json)")
    ap.add_argument("--checkpoint", required=True, help="QuickVC generator checkpoint (G_*.pth)")
    ap.add_argument("--units", required=True, nargs="+", help="content units of each source, [T, 768] .npy (vc/encode.py)")
    ap.add_argument("--target", required=True, help="recording of the target voice, 16 kHz mono 16-bit WAV")
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--precision", type=int, default=1, choices=[0, 1])
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args(argv)
    cfg = _config.from_quickvc_json(a.config)
    try:
        target = read_wav(a.target, int(cfg["sampling_rate"]))
    except ValueError as ex:
        ap.error(str(ex))
    units = []
    for p in a.units:
        u = np.load(p)
        if u.ndim != 2 or u.shape[1] != cfg["unit_channels"] or u.shape[0] < 1:
            ap.error("%s holds %s; expected content units [T, %d]" % (p, u.shape, cfg["unit_channels"]))
        units.append(u.astype(np.float32))
    vc = QuickVC(a.config, a.checkpoint, device=a.device, precision=a.precision)
    try:
        g = vc.embed(target)
        os.makedirs(a.out_dir, exist_ok=True)
        for p, w in zip(a.units, vc.convert(units, g=g, seed=a.seed)):
            out = os.path.join(a.out_dir, os.path.splitext(os.path.basename(p))[0] + ".wav")
            write_wav(out, w, vc.sampling_rate)
            print(out)
    finally:
        vc.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
