"""Seeded vocoder and mels of the StableTTS vocoder tests, shared by oracle/make_golden_hifigan.py (which runs the reference's
Generator on them) and the tests (which run the oracle and the engine on them and compare with the stored waveforms)."""
import hashlib
import os

import numpy as np
import torch

from vosk_tts_b200 import config as C, synthetic, weights

SEED = 4242
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_hifigan.npz")
# (name, frame counts of the utterances); each utterance goes through the reference alone
CASES = [("f1", [1]), ("f2", [2]), ("f7", [7]), ("f37", [37]), ("f300", [300]), ("ragged3", [23, 5, 61])]
# text-to-waveform: utterances of tests/golden/ref_stabletts.npz whose reference mel the fixture also vocodes
TEXT_CASES = ["short.mel0", "ragged3.mel2"]


def config():
    return C.hifigan_config()


def checkpoint():
    """The seeded `generator` state dict, weight-normed (weight_g / weight_v) as a training checkpoint holds it."""
    return synthetic.make_random_hifigan(SEED, config())


def folded():
    return weights.fold_weight_norm(checkpoint())


def mel(name, b, T):
    """A seeded denormalised mel [80, T] of the scale StableTTS's synthetic models produce (mel_mean -5.5, mel_std 2.1)."""
    g = torch.Generator().manual_seed(sum(map(ord, name)) * 100 + b)
    return (-5.5 + 2.1 * torch.randn(80, T, generator=g)).numpy()


def case_mels(case):
    return [mel(case[0], b, T) for b, T in enumerate(case[1])]


def sha1_state(sd):
    h = hashlib.sha1()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(np.ascontiguousarray(sd[k].detach().cpu().float().numpy() if hasattr(sd[k], "detach") else sd[k], np.float32).tobytes())
    return h.hexdigest()
