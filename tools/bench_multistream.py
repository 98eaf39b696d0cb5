"""Times multistream StableTTS text to waveform from word pieces on the GPU (vtts_stabletts_synthesise_pieces_wav: BERT run and
its rows gathered inside the text phase) against the composition it replaces (vtts_bert_features, the gather on the host,
vtts_stabletts_synthesise_wav), in alternating rounds, and the host front end (WordPiece tokenizer and g2p_multistream_scales)
of Synth.  Shapes: rubert-base (768 wide, the 10 layers the exported graph runs, a 120000-piece vocabulary), StableTTS's
text encoder and decoder at their reference widths, HiFi-GAN v1, seeded synthetic weights; 5 flow-matching steps (Model's
default), precision mode 1.  Workloads: one sentence of 150 tokens and 64 ragged sentences of 20-150 tokens, a word piece
per 4 tokens.  Every figure is the median over rounds of a host clock ending in a synchronise (the waveform is on the
host).  Prints the card, its power limit and SM clocks, read in the same run, and one JSON line.

    python tools/bench_multistream.py [--rounds 20] [--warmup 3]"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bert_inputs as BI  # noqa: E402
import hifigan_inputs as HI  # noqa: E402
from bench_stabletts import card  # noqa: E402
from vosk_tts_b200 import config as C, synthetic  # noqa: E402
from vosk_tts_b200.stabletts import StableTTS  # noqa: E402
from vosk_tts_b200.synth import Synth  # noqa: E402
from vosk_tts_b200.wordpiece import BertWordPieceTokenizer  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def front_end_ms(rounds):
    """Synth's host work for one sentence of the fixture's words: tokenizer, token selection and g2p_multistream_scales."""
    with open(os.path.join(GOLDEN, "multistream_front.json"), encoding="utf-8") as f:
        fix = json.load(f)
    model = types.SimpleNamespace(dic=fix["dictionary"], config={"phoneme_id_map": fix["phoneme_id_map"], "model_type": "multistream_v3"},
                                  tokenizer=BertWordPieceTokenizer(os.path.join(GOLDEN, "multistream_vocab.txt")))
    s = Synth(model)
    text = "Привет, мир! Мой дом, мой мир; моя жизнь: вот так. Он сказал: \"привет\" и ушёл... Раз, два, три, четыре, пять. " \
           "Ах_ вот как_ понятно. Ёлка, ёжик, йод - да, да... нет?"
    t = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        enc, keep = s._word_pieces(text.lower(), nopunc=True)
        ids, rows, extra = s._multistream(text, True, True, len(keep))
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t)), len(ids), len(enc.ids)


def utterances(bt, cfg, lens, rng):
    out = []
    for i, T in enumerate(lens):
        L = max(2, T // 4)
        rows = np.sort(rng.integers(0, L, T)).astype(np.int32)
        out.append((rng.integers(0, cfg["n_vocab"], (cfg["n_streams"], T)).astype(np.int64), BI.sentence(bt, L, salt=i), rows))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multistream.py measures on a GPU; none is visible")
    out = {"card": card()}
    print("card (name, power limit, max SM clock, SM clock):", out["card"])
    fe, n_tok, n_pieces = front_end_ms(a.rounds)
    out["front_end"] = {"ms": round(fe, 3), "tokens": n_tok, "pieces": n_pieces}
    print("host front end:", json.dumps(out["front_end"]))
    bt = C.bert_config({"vocab_size": 120000})
    cfg = C.stabletts_config({"n_vocab": 178})
    tts = StableTTS(None, synthetic.make_random_stabletts(cfg, 5), precision=1, vocoder=HI.checkpoint(), bert=(synthetic.make_random_bert(bt, 77), bt))
    rng = np.random.default_rng(0)
    for name, lens in (("sentence_150", [150]), ("ragged_64", [int(v) for v in rng.integers(20, 151, 64)])):
        us = utterances(bt, tts.cfg, lens, rng)
        xs, sids = [u[0] for u in us], [0] * len(us)

        def fused():
            return tts.synthesise(xs, None, sids, n_timesteps=5, seed=3, pieces=[u[1] for u in us], bert_rows=[u[2] for u in us])

        def composed():
            feats = tts.bert_features([u[1] for u in us])
            return tts.synthesise(xs, [np.ascontiguousarray(f[u[2]].T) for f, u in zip(feats, us)], sids, n_timesteps=5, seed=3,
                                  return_wav=True)

        for _ in range(a.warmup):
            fused()
            composed()
        tf, tc = [], []
        for _ in range(a.rounds):
            for fn, acc in ((fused, tf), (composed, tc)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = fn()
                acc.append((time.perf_counter() - t0) * 1e3)
        same = all(np.array_equal(x, y) for x, y in zip(fused()["wav"], composed()["wav"]))
        res = {"tokens": int(sum(lens)), "pieces": int(sum(len(u[1]) for u in us)), "frames": int(sum(r["mel_lengths"])),
               "fused_ms": round(float(np.median(tf)), 3), "composed_ms": round(float(np.median(tc)), 3), "wav_bit_identical": same}
        out[name] = res
        print(name, json.dumps(res))
    tts.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
