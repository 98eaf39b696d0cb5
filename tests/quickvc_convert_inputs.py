"""Inputs of the QuickVC conversion tests: the whole seeded checkpoint, stand-in content units, the posterior noise and the
cases of tests/golden/ref_quickvc_convert.npz.  The configuration, the seed and the target clips are quickvc_inputs'."""
import numpy as np

from vosk_tts_b200 import synthetic
from quickvc_inputs import GOLDEN, config, SEED  # noqa: F401

# (T content frames, target whose g conditions the case)
CASES = [(1, "short"), (2, "t129"), (37, "long"), (250, "short")]
# frames of the T = 250 case whose latents (m_p, logs_p, z_p, z) the fixture keeps: both ends, where the convs' zero padding
# and the decoder's edges act, and enough of the interior; its waveform is kept whole
LONG_FRAMES = np.r_[0:24, 113:137, 226:250]


def model():
    """The whole seeded QuickVC checkpoint (its enc_spk is quickvc_inputs.speaker_encoder()'s)."""
    return synthetic.make_random_quickvc(config(), SEED)


def kept_frames(T):
    """Frames of a case whose latents the fixture stores."""
    return LONG_FRAMES if T == 250 else np.arange(T)


def units(T, seed):
    """Stand-in for ContentVec's last_hidden_state of one clip, float32 [T][768]: every channel an AR(1) process with
    coefficient 0.9 (neighbouring 20 ms frames are strongly correlated, as speech features are) and its own scale, drawn
    log-normally around 0.3 (about the spread of ContentVec's hidden units), plus a per-channel offset."""
    rng = np.random.RandomState(1000 + seed)
    scale = np.exp(rng.randn(768) * 0.5) * 0.3
    offset = rng.randn(768) * 0.1
    x = np.zeros((T, 768))
    s = rng.randn(768)
    for t in range(T):
        s = 0.9 * s + np.sqrt(1 - 0.81) * rng.randn(768)
        x[t] = s
    return (x * scale + offset).astype(np.float32)


def eps(T, seed):
    """The standard normal noise of enc_p's sample (models.py:270), float32 [inter_channels][T]."""
    return np.random.RandomState(2000 + seed).randn(192, T).astype(np.float32)
