"""Seeded inputs of the voice-conversion fixtures, shared by oracle/make_golden_vc.py (which stores the reference's outputs
for them in tests/golden/ref_voice_conversion.npz) and the tests that compare against those stored outputs."""
import copy

import numpy as np
import torch

import golden_ref as GR

# (case, clip, sid_src, sid_tgt, model): the mel model is the reference architecture with synthetic weights (seed 1234),
# the linear one the tiny configuration with a linear-spectrogram posterior encoder (seed 11)
CASES = [("c0", "a", 3, 7, "mel"), ("c1", "b", 5, 5, "mel"), ("c2", "b", 1, 2, "lin")]
SEEDS = {"mel": 1234, "lin": 11}


def speech():
    """int16 clips of public-domain LJSpeech recordings (22 050 Hz), lengths not multiples of 256."""
    d = GR.load("vc_speech.npz")
    return {"a": d["a"], "b": d["b"]}


def wav_float(x):
    return np.asarray(x, np.float32) / 32768.0          # data_utils.py:77 (max_wav_value)


def training_json(model):
    if model == "mel":
        return GR.ref_config()
    j = copy.deepcopy(GR.tiny_training_json())
    j["model"]["use_mel_posterior_encoder"] = False
    j["data"]["use_mel_posterior_encoder"] = False
    return j


def eps_q(case, inter, frames):
    g = torch.Generator().manual_seed({"c0": 21, "c1": 22, "c2": 23}[case])
    return torch.randn(1, inter, frames, generator=g)
