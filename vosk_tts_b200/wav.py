"""Reading 16-bit PCM WAV files at any sample rate, for the front ends' opt-in resampling (`resample=True`, `--resample`)."""
import wave

import numpy as np


def read_pcm16(path):
    """A 16-bit PCM WAV, mono or multichannel -> (float32 [n] in [-1, 1], sample rate).  Channels are averaged to mono as
    librosa.load(mono=True) does (the mean of the float samples, int16 / 32768)."""
    with wave.open(path, "rb") as f:
        sr, ch, sw = f.getframerate(), f.getnchannels(), f.getsampwidth()
        if sw != 2:
            raise ValueError("%s: only 16-bit PCM WAV files are read" % path)
        x = np.frombuffer(f.readframes(f.getnframes()), "<i2").astype(np.float64) / 32768.0
    return x.reshape(-1, ch).mean(axis=1).astype(np.float32), int(sr)
