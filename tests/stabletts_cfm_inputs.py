"""Seeded model and inputs of the StableTTS flow-matching tests, shared by oracle/make_golden_stabletts_cfm.py (which runs
the reference on them) and the tests (which run the oracle and the engine on them and compare with the stored mel)."""
import os

import numpy as np
import torch

from vosk_tts_b200 import config as C, synthetic

SEED = 4321
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_stabletts_cfm.npz")
# (name, frame counts of the batch's utterances, n_timesteps, guidance scale, temperature, speaker ids)
CASES = [
    ("t1", [1], 10, 0.5, 1.0, [0]),
    ("short", [23], 10, 0.5, 1.0, [1]),
    ("short_n1", [23], 1, 0.5, 1.0, [1]),
    ("short_s0", [23], 10, 0.0, 0.8, [0]),
    ("long", [301], 10, 0.5, 0.667, [1]),
    ("ragged3", [40, 7, 65], 10, 0.5, 1.0, [0, 1, 0]),
    ("ragged3_n1_s0", [40, 7, 65], 1, 0.0, 1.0, [1, 1, 0]),
]


def config():
    return C.stabletts_cfm_config()


def model(cfg=None):
    return synthetic.make_random_stabletts_cfm(cfg or config(), SEED)


def inputs(name, T, cfg=None):
    """Seeded mu [cond, T] and noise [noise, T] of one utterance (float32 numpy)."""
    cfg = cfg or config()
    g = torch.Generator().manual_seed(sum(map(ord, name)) * 1000 + T)
    return (torch.randn(cfg["cond_channels"], T, generator=g).numpy(), torch.randn(cfg["noise_channels"], T, generator=g).numpy())


def case_inputs(case):
    """[(mu, noise)] of a CASES entry's utterances."""
    name, lens = case[0], case[1]
    return [inputs(name + str(b), T) for b, T in enumerate(lens)]
