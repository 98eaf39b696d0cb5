"""Inputs of the ContentVec tests: the seeded checkpoint, the source clips, and the unmodified reference model
(vc/contentvec.py on transformers) where the reference tree and transformers are present."""
import os

import numpy as np

from oracle import contentvec_ref
from vosk_tts_b200 import config as C, synthetic, weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 4242
LENGTHS = (400, 719, 720, 16000)          # the shortest clip, the frame-count edge at 720, one second
LONG = 160000                              # 10 s: 499 frames
LONG_KEEP = 48                             # frames kept at each end and in the middle of the 10 s clip
# end-to-end cases (source samples, target of tests/golden/ref_quickvc.npz): reference ContentVec, then reference QuickVC
E2E = [(16000, "short"), (40000, "long")]


def cv():
    return C.contentvec_config()


_SD = {}


def model(seed=SEED):
    if seed not in _SD:
        _SD[seed] = synthetic.make_random_contentvec(seed)
    return _SD[seed]


def folded(seed=SEED):
    return weights.fold_contentvec_pos_conv(model(seed))


def speech(n, seed):
    """A speech-like 16 kHz clip in [-1, 1]: harmonic bursts with a moving pitch under an envelope, plus a little noise."""
    r = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    f0 = 110 + 40 * np.sin(2 * np.pi * 0.7 * t + r.uniform(0, 6))
    ph = 2 * np.pi * np.cumsum(f0) / 16000.0
    x = sum(np.sin(k * ph + r.uniform(0, 6)) / k for k in range(1, 12))
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 3.1 * t + r.uniform(0, 6)) ** 2
    x = 0.3 * x * env + 0.01 * r.standard_normal(n)
    return np.clip(x, -1, 1).astype(np.float32)


def dc_offset(n, seed):
    """0.5 + 0.01 * signal: the clip on which a one-pass variance loses its digits."""
    return (0.5 + 0.01 * speech(n, seed)).astype(np.float32)


def kept_frames(T):
    if T <= 3 * LONG_KEEP:
        return np.arange(T)
    m = T // 2 - LONG_KEEP // 2
    return np.concatenate([np.arange(LONG_KEEP), np.arange(m, m + LONG_KEEP), np.arange(T - LONG_KEEP, T)])


def reference_available():
    return contentvec_ref.available()


def build_reference(sd):
    return contentvec_ref.build(sd)
