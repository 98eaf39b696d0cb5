"""Seeded BERT models and word-piece sentences of the BERT tests: the production shape (rubert-base: 768 wide, 12 heads, FFN
3072, the 10 layers the exported graph runs) with a small vocabulary, and a tiny shape (128 wide, 4 heads of 32, FFN 512, 4
layers of which 2 run)."""
import numpy as np

from vosk_tts_b200 import config as C, synthetic

SEED = 2468
LENGTHS = [2, 7, 64, 300, 512]           # word pieces per sentence, up to the position table


def production():
    return C.bert_config({"vocab_size": 1200})


def tiny():
    return C.bert_config({"hidden_size": 128, "num_attention_heads": 4, "intermediate_size": 512, "num_hidden_layers": 4,
                          "vocab_size": 300})


def model(bt):
    return synthetic.make_random_bert(bt, SEED)


def sentence(bt, L, salt=0):
    """Seeded ids of one sentence: [CLS] = 2, L - 2 pieces, [SEP] = 3 (rubert's vocab.txt order)."""
    rng = np.random.default_rng(SEED * 1000 + L * 7 + salt)
    ids = rng.integers(5, bt["bt_vocab"], L).astype(np.int64)
    ids[0], ids[-1] = 2, 3
    return ids


def ragged(bt, n=64):
    """n sentences of 2 .. 512 pieces."""
    rng = np.random.default_rng(SEED + n)
    return [sentence(bt, int(L), salt=i) for i, L in enumerate(rng.integers(2, bt["bt_max_pos"] + 1, n))]
