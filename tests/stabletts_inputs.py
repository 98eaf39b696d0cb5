"""Seeded model and inputs of the StableTTS text-to-mel tests, shared by oracle/make_golden_stabletts.py (which runs the
reference's synthesise on them) and the tests (which run the oracle and the engine on them and compare with the stored
durations and mel)."""
import hashlib
import os

import numpy as np
import torch

from vosk_tts_b200 import config as C, synthetic

SEED = 9753
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_stabletts.npz")
MAX_FRAMES = 1280      # columns of the seeded noise; a case reads its first ceil4(frames)
# (name, token counts of the batch's utterances, speaker ids, n_timesteps, temperature, length_scale, {utterance: {token: pause}})
CASES = [
    ("t1", [1], [0], 10, 1.0, 1.0, {}),
    ("short", [9], [1], 10, 1.0, 1.0, {}),
    ("short_n1", [9], [1], 1, 0.8, 1.0, {}),
    ("pause", [12], [0], 10, 1.0, 1.0, {0: {0: 3.0, 5: 7.0, 9: 2.0}}),
    ("slow", [11], [1], 10, 0.667, 1.3, {0: {4: 2.5}}),
    # one text, the pause of one token growing by a frame: the four residues of the frame count mod 4
    ("mod_a", [7], [0], 10, 1.0, 1.0, {0: {3: 2.0}}),
    ("mod_b", [7], [0], 10, 1.0, 1.0, {0: {3: 3.0}}),
    ("mod_c", [7], [0], 10, 1.0, 1.0, {0: {3: 4.0}}),
    ("mod_d", [7], [0], 10, 1.0, 1.0, {0: {3: 5.0}}),
    ("long", [150], [1], 10, 1.0, 1.0, {0: {0: 4.0, 71: 9.0}}),
    ("ragged3", [14, 5, 22], [0, 1, 0], 10, 1.0, 1.0, {1: {0: 2.0}, 2: {7: 6.0, 21: 3.0}}),
]


def config():
    return C.stabletts_config({"n_vocab": 120})


def model(cfg=None):
    return synthetic.make_random_stabletts(cfg or config(), SEED)


def inputs(name, T, pauses=None, cfg=None):
    """Seeded ids [streams, T], bert [bert_dim, T], pause [T] (zeros but for `pauses`) and noise [noise, MAX_FRAMES] of one
    utterance (numpy).  "mod_*" share one text."""
    cfg = cfg or config()
    key = "mod" if name.startswith("mod_") else name
    g = torch.Generator().manual_seed(sum(map(ord, key)) * 1000 + T)
    ids = torch.randint(0, int(cfg["n_vocab"]), (int(cfg["n_streams"]), T), generator=g).numpy()
    bert = torch.randn(int(cfg["bert_dim"]), T, generator=g).numpy()
    noise = torch.randn(int(cfg["noise_channels"]), MAX_FRAMES, generator=g).numpy()
    pause = np.zeros(T, np.float32)
    for i, v in (pauses or {}).items():
        pause[i] = v
    return ids, bert, pause, noise


def case_inputs(case):
    """[(ids, bert, pause, noise)] of a CASES entry's utterances; the utterance's key in the fixture is name + index."""
    name, lens, pauses = case[0], case[1], case[6]
    return [inputs(name if name.startswith("mod_") else name + str(b), T, pauses.get(b)) for b, T in enumerate(lens)]


def sha1(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def denormalise(mel, mean, std):
    """matcha.utils.model.denormalize in fp32: one rounded product, one rounded sum."""
    return mel * np.float32(std) + np.float32(mean)


def load_golden():
    """The fixture as a dict, with what it leaves out because it follows exactly from what it holds (the maker checks each
    identity bit for bit against the reference's own tensors): "<case>.mel<b>" = decoder_outputs * mel_std + mel_mean, and
    "<case>.encoder_outputs<b>" = one stored column per token repeated w_round times."""
    g = dict(np.load(GOLDEN))
    for k in [k for k in g if ".decoder_outputs" in k]:
        g[k.replace("decoder_outputs", "mel")] = denormalise(g[k], g["mel_mean"], g["mel_std"])
        g[k.replace("decoder_outputs", "encoder_outputs")] = np.repeat(g[k.replace("decoder_outputs", "encoder_tokens")],
                                                                       g[k.replace("decoder_outputs", "w_round")], 1)
    return g
