"""Seeded inputs shared by oracle/make_golden_ref.py (which stores the reference's outputs for them under tests/golden/) and
the tests that compare against those stored outputs."""
import copy
import json
import os
import zlib

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
INFER_CASES = [(24, 101), (77, 102)]
N_VOCAB = 40
DECODER_VARIANTS = [("ms_istft_vits", "ms_istft"), ("istft_vits", "istft"), ("mb_istft_vits", "mb_istft")]
SAMPLE = 4096          # values kept of a large stored output (a fixed, name-seeded choice of positions)


SD_SAMPLE = 64         # values kept per checkpoint tensor


def sample_index(n, name, k=SAMPLE):
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.RandomState(zlib.crc32(name.encode()) & 0x7FFFFFFF).choice(n, k, replace=False))


def load(name):
    return np.load(os.path.join(GOLDEN, name))


def ref_config():
    with open(os.path.join(GOLDEN, "mb_istft_vits2_multi.json")) as f:
        return json.load(f)


def g2p_words():
    words = ["прив+ет", "абстр+акция", "+ёлка", "подъ+езд", "семь+я", "чащ+а", "й+од", "объявл+ение", "в+ьюга", "съ+ёмка",
             "по-р+усски", "+я", "мышь", "компь+ютер", "ш+ёлк", "Гог+оль"]
    letters = "абвгдеёжзийклмнопрстуфхцчшщъыьэюя"
    rng = np.random.RandomState(0)
    for _ in range(300):
        n = rng.randint(1, 9)
        w = "".join(letters[i] for i in rng.randint(0, len(letters), n))
        p = rng.randint(0, n)
        words.append(w[:p] + "+" + w[p:])
    return words


def spline_inputs():
    g = torch.Generator().manual_seed(5)
    n = 4000
    x = torch.randn(n, generator=g) * 3.0
    uw, uh, ud = torch.randn(n, 10, generator=g), torch.randn(n, 10, generator=g), torch.randn(n, 9, generator=g)
    return x, uw, uh, ud


def infer_inputs(T, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, 62, (1, T), generator=g)
    eps_dp = torch.randn(1, 2, T, generator=g)
    eps_z = torch.randn(1, 192, 24 * T, generator=g)
    return tok, eps_dp, eps_z, [0.667, 1.0, 0.8]


def tiny_training_json():
    """The reference configuration at reduced width (64 instead of 192 channels, three encoder layers, two resblock
    kernels): the architecture of tests/golden/tiny_model.onnx (oracle/make_tiny_onnx.py)."""
    j = copy.deepcopy(ref_config())
    j["model"].update(inter_channels=64, hidden_channels=64, filter_channels=128, n_heads=2, n_layers=3, kernel_size=3,
                      resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5]], upsample_rates=[4, 4],
                      upsample_initial_channel=64, upsample_kernel_sizes=[16, 16], gin_channels=32)
    j["data"]["n_speakers"] = 4
    return j


def training_json(flag):
    """tiny_training_json() with the inverse-STFT decoder selected by `flag`"""
    j = tiny_training_json()
    j["model"].update(mb_istft_vits=False, ms_istft_vits=False, istft_vits=False)
    j["model"][flag] = True
    return j


def variant_inputs(cfg):
    g = torch.Generator().manual_seed(3)
    T = 19
    tok = torch.randint(0, N_VOCAB, (1, T), generator=g)
    eps_dp = torch.randn(1, 2, T, generator=g)
    eps_z = torch.randn(1, cfg["inter_channels"], 400 * T, generator=g)     # the random SDP of this seed is slow-spoken
    return tok, eps_dp, eps_z, [0.8, 1.0, 0.8]
