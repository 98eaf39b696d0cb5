"""Seeded inputs of the forced-alignment fixtures, shared by oracle/make_golden_align.py (which stores the reference's
SynthesizerTrn.forward alignment for them in tests/golden/ref_alignment.npz) and the tests that compare against it."""
import copy

import numpy as np
import torch

import golden_ref as GR
import vc_inputs as VI

# (case, clip, model, sid, tokens): "mel" is the reference architecture with synthetic weights, "lin" the tiny configuration
# with a linear-spectrogram posterior encoder, "single" the same without speakers (n_speakers 0, g = None).  Clip "a" has
# 172 frames, "b" 112.  tokens None: as many tokens as frames (the path is forced).
CASES = [("a0", "a", "mel", 3, 1), ("a1", "b", "mel", 5, 45), ("a2", "b", "mel", 2, None), ("a3", "b", "lin", 1, 71),
         ("a4", "b", "single", 0, 41)]
# the reference's spectrogram of (clip, front end) is stored with the voice-conversion fixture (ref_voice_conversion.npz)
SPEC_CASE = {("a", "mel"): "c0", ("b", "mel"): "c1", ("b", "lin"): "c2", ("b", "single"): "c2"}
SEEDS = {"mel": 1234, "lin": 11, "single": 13}


def training_json(model):
    j = VI.training_json("mel" if model == "mel" else "lin")
    if model == "single":
        j = copy.deepcopy(j)
        j["data"]["n_speakers"] = 0
    return j


def n_vocab(model):
    return 62 if model == "mel" else GR.N_VOCAB


def frames(clip):
    return len(VI.speech()[clip]) // 256


def ids(case):
    """Phoneme ids with the blank 0 interspersed (synth.py:244-251): odd positions are blanks."""
    _, clip, model, _, n = next(c for c in CASES if c[0] == case)
    n = frames(clip) if n is None else n
    rng = np.random.RandomState(sum(map(ord, case)))
    out = rng.randint(1, n_vocab(model), size=n).astype(np.int64)
    out[1::2] = 0
    return out


def ref_spec(case):
    _, clip, model, _, _ = next(c for c in CASES if c[0] == case)
    return GR.load("ref_voice_conversion.npz")[SPEC_CASE[(clip, model)] + "/spec"]


def eps_q(case, inter, t_y):
    g = torch.Generator().manual_seed(100 + sum(map(ord, case)))
    return torch.randn(1, inter, t_y, generator=g)
