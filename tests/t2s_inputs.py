"""Seeded GPT-SoVITS text-to-semantic models and inputs shared by the t2s tests."""
import numpy as np

from vosk_tts_b200 import config, synthetic

SMALL = {"hidden_dim": 64, "embedding_dim": 64, "head": 2, "n_layer": 2, "vocab_size": 65, "phoneme_vocab_size": 30, "dropout": 0.0,
         "EOS": 64}
UPSTREAM = {"hidden_dim": 512, "embedding_dim": 512, "head": 16, "n_layer": 24, "vocab_size": 1025, "phoneme_vocab_size": 732,
            "dropout": 0.0, "EOS": 1024}     # the configuration of the published checkpoints
WIDE = {"hidden_dim": 128, "embedding_dim": 128, "head": 4, "n_layer": 3, "vocab_size": 257, "phoneme_vocab_size": 60,
        "dropout": 0.0, "EOS": 256}


def _block(hidden, heads, vocab, layers=2):
    return {"hidden_dim": hidden, "embedding_dim": hidden, "head": heads, "n_layer": layers, "vocab_size": vocab,
            "phoneme_vocab_size": 60, "dropout": 0.0, "EOS": vocab - 1}


# the head widths above 32 (dk = hidden / heads), the vocabularies whose padded sort size is the vocabulary itself or above
# 2048, and the widest shape the engine takes (FFN 4096: t2s_ffn2_kernel's 80 KiB of shared memory)
D64 = _block(128, 2, 1024)
D96 = _block(192, 2, 2049)
D96_1 = _block(96, 1, 65)          # width 96: the tensor-core prefill (precision mode >= 1) refuses it
D128 = _block(256, 2, 4096)
MAX = _block(1024, 8, 4096)


def model(block=SMALL, seed=5, eos_scale=1.0, eos_logit=None):
    """eos_logit: the last layer's norm2 weight scaled by 0.3 and the EOS row of ar_predict_layer set so that the hidden rows'
    common part (norm2's bias) gives EOS that logit: EOS then competes with the top tokens at every step, and the repetition
    penalty, which never touches it, lets it win sooner or later."""
    cfg = config.t2s_config(block)
    sd = synthetic.make_random_t2s(cfg, seed, eos_scale=eos_scale)
    if eos_logit is not None:
        last = "h.layers.%d.norm2." % (cfg["cv_layers"] - 1)
        sd[last + "weight"].mul_(0.3)
        b = sd[last + "bias"]
        sd["ar_predict_layer.weight"][-1] = eos_logit * b / float(b @ b)
    return sd, cfg


def phones(cfg, n, seed):
    return np.random.default_rng(seed).integers(0, cfg["t2s_phone_vocab"], n).astype(np.int64)


def prompt(cfg, n, seed, repeat=False):
    r = np.random.default_rng(seed)
    hi = 6 if repeat else cfg["t2s_vocab"] - 1          # a few distinct tokens repeat often
    return r.integers(0, hi, n).astype(np.int64)


def q_draws(cfg, steps, seed):
    """[steps, V] Exp(1) draws, as a seeded numpy stream standing in for Tensor.exponential_."""
    return np.random.default_rng(seed).exponential(1.0, (steps, cfg["t2s_vocab"])).astype(np.float32)
