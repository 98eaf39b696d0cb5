"""Inputs of the GPT-SoVITS prompt-token tests: the seeded HuBERT (the ContentVec tests' model, which has
chinese-hubert-base's shape) and s2 tensors, the cases of tests/golden/ref_sovits_semantic.npz, and the HuBERT-like feature
rows of the extract_latent cases."""
import os

import numpy as np
import torch

import contentvec_inputs as CI
from vosk_tts_b200 import config as C, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "ref_sovits_semantic.npz")
SEED = 2525
S2_32K = {"data": {"sampling_rate": 32000}}          # the published v1 s2 config's rate: a 9600-sample pad
S2_24K = {"data": {"sampling_rate": 24000}}          # a 7200-sample pad
# waveform cases: (samples at 16 kHz before the pad, speech seed, s2 config)
WAVE = {
    "w48000": (48000, 61, S2_32K),       # the shortest prompt: 179 HuBERT frames, so ssl_proj drops one
    "w48320": (48320, 62, S2_32K),       # 180 frames
    "w10s": (160000, 63, S2_32K),        # 529 frames
    "w20s": (320000, 64, S2_32K),        # the longest prompt: 1029 frames
    "w24k": (64000, 65, S2_24K),
}
# extract_latent cases: (feature rows, seed); "ties" runs on the codebook of s2_ties
FEAT = {"f_odd": (37, 71), "f_even": (64, 72), "ties": (24, 73)}
TIE_PAIR = (200, 300)                    # codewords b -/+ d around the projection of a zero row: an exact tie
ZERO_ROWS = (10, 11)                     # the zero feature rows of "ties" (pair row 5)


def hubert():
    return CI.model()


def cv():
    return C.contentvec_config()


_S2 = []
_ROWS = []
TIE_ROW0 = 600                           # the first codebook row of the "ties" rows


def codebook_rows():
    """HuBERT's rows of every waveform case (padded), from the float64 restatement of ContentVec (oracle/contentvec_oracle.py,
    checked against transformers' HubertModel by tests/test_contentvec_host.py), [N, 768] float64.  The codebook is drawn from
    the cases themselves: a seeded HuBERT maps a whole recording to rows much closer to each other than to any other
    recording's (its attention and GroupNorm see the whole clip), so a codebook drawn from other recordings gives each case
    one or two codes."""
    if not _ROWS:
        from oracle import contentvec_oracle as CO
        sd = CI.folded()
        _ROWS.append(np.concatenate([CO.contentvec_units(sd, cv(), padded(name), torch.float64).numpy() for name in WAVE]))
    return _ROWS[0]


def s2():
    """The seeded s2 tensors (synthetic.make_random_sovits), the codebook drawn from codebook_rows()."""
    if not _S2:
        _S2.append(synthetic.make_random_sovits(hubert(), codebook_rows(), SEED))
    return {k: v.clone() for k, v in _S2[0].items()}


def cfg(s2_config=S2_32K):
    return C.sovits_config(s2_config, codebook=1024)


def clip(name):
    """The 16 kHz recording of a waveform case, before the pad."""
    n, seed, _ = WAVE[name]
    return CI.speech(n, seed)


def padded(name):
    """The recording with the reference's pad appended (inference_cli.py:176-192): what HuBERT reads."""
    n, seed, s2c = WAVE[name]
    return np.concatenate([clip(name), np.zeros(C.sovits_pad(s2c["data"]["sampling_rate"]), np.float32)])


def feats(name):
    """Rows [T, 768] of an extract_latent case: for "f_odd" / "f_even" HuBERT-like rows, gamma * n + beta of the encoder's last
    LayerNorm with n zero-mean unit-variance over the channels; for "ties" HuBERT's rows of the codebook's recordings from
    TIE_ROW0 (so that they pick codewords drawn from them) with two zero rows (ZERO_ROWS)."""
    T, seed = FEAT[name]
    if name == "ties":
        x = codebook_rows()[TIE_ROW0:TIE_ROW0 + T].astype(np.float32)
        x[list(ZERO_ROWS)] = 0
        return x
    h = hubert()
    gamma = h["encoder.layers.11.final_layer_norm.weight"].double().numpy()
    beta = h["encoder.layers.11.final_layer_norm.bias"].double().numpy()
    z = np.random.default_rng(seed).standard_normal((T, gamma.size))
    z = (z - z.mean(1, keepdims=True)) / z.std(1, keepdims=True)
    return (gamma * z + beta).astype(np.float32)


def s2_ties():
    """s2() with exact ties for the "ties" rows: the codes of its pair rows 0..3 duplicated at other indices (two above and
    two below the original), and TIE_PAIR set to b - d and b + d, b ssl_proj's bias (the projection of a zero pair) and d a
    vector of +-1/8: all on a dyadic grid, so both scores are the same in fp32 and in float64."""
    from oracle import sovits_oracle as O
    sd = s2()
    E = sd["quantizer.vq.layers.0._codebook.embed"]
    codes, _, _ = O.extract_latent(feats("ties"), sd)
    K = E.shape[0]
    for i, c in enumerate(codes[:4]):
        j = (int(c) + (K // 2 if i % 2 == 0 else K // 3)) % K
        E[j] = E[int(c)]
    b = sd["ssl_proj.bias"]
    d = torch.from_numpy(np.where(np.random.default_rng(74).random(b.numel()) < 0.5, -0.125, 0.125).astype(np.float32))
    E[TIE_PAIR[0]] = b - d
    E[TIE_PAIR[1]] = b + d
    return sd
