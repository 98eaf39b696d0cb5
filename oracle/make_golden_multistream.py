"""Stores what the reference's multistream front end feeds its graphs, so that tests/test_multistream_host.py runs without the
reference tree.

Run once where the reference tree is present (``python oracle/make_golden_multistream.py``).  It runs the unmodified
vosk_tts/synth.py `Synth` of the reference, with a stub `onnxruntime` module, over a model namespace holding
- a generated dictionary and a phoneme_id_map of every phone (plain and with each _B/_I/_E/_S suffix) and every punctuation
  mark, except the suffixed forms of the "_" phone, which the reference's v2 front end then fails on as it does on a real map;
- the real `tokenizers.BertWordPieceTokenizer` over a generated vocab.txt of whole words, words reachable only as "##" pieces,
  and missing words, which give [UNK];
- a stub bert_onnx whose row i holds i, so the `bert` feed records the row each phone took;
- a stub onnx session that records the feeds.
For every text and every front end (v1, v2, v3 and v2 without BERT) it stores the feeds or the exception, and for every
text the direct results of g2p_multistream / g2p_multistream_scales and get_word_bert's token selection.  Writes
tests/golden/multistream_front.json and tests/golden/multistream_vocab.txt.
"""
import importlib
import json
import os
import re
import sys
import types
import unicodedata
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/vosk_tts"
GOLDEN = os.path.join(ROOT, "tests", "golden")

TEXTS = [
    "Привет, мир!",
    "мой ёжик ещё ест йогурт",
    "з+амок и зам+ок",
    "привет_ как дела",
    "Привет _ мир",
    "Он сказал: \"привет\" и ушёл.",
    "\"Цитата\" - сказал он. \"Ещё одна!\"",
    "Ну... и что?",
    "Мама - папа",
    "мама -папа",
    "Это — всё!",
    "Что?!",
    "Я (кажется) прав.",
    "МОСКВА Столица",
    "из-за угла",
    "кто-то пришёл",
    "абырвалг",
    "раз" * 34,
    "",
    "привет + мир",
    "мой дом, мой мир; моя жизнь: вот так.",
    "да, да... нет?",
    "При+вет, м+ир!",
    "ёлка ёжик йод",
    "  пробелы   вокруг  ",
    "раз, два, три, четыре, пять.",
    "Он ушёл... Она пришла!",
    "(тест)",
    "Ах_ вот как_ понятно.",
    "из-за мой дом",
]
# (model_type, with BERT's tokenizer)
VARIANTS = {"v1": ("multistream_v1", True), "v2": ("multistream_v2", True), "v3": ("multistream_v3", True),
            "v2_nobert": ("multistream_v2", False)}
PUNCT = [" ", "^", "$", "_", ",", ".", "!", "?", ";", ":", "...", "-", "(", ")"]
SPECIAL = ["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"]


def _norm(w):
    return "".join(c for c in unicodedata.normalize("NFD", w.lower()) if unicodedata.category(c) != "Mn")


def _load_reference():
    ort = types.ModuleType("onnxruntime")
    ort.InferenceSession = ort.SessionOptions = None
    sys.modules["onnxruntime"] = ort
    pkg = types.ModuleType("ref_vosk_tts")
    pkg.__path__ = [REF]
    sys.modules["ref_vosk_tts"] = pkg
    return importlib.import_module("ref_vosk_tts.synth"), importlib.import_module("ref_vosk_tts.g2p")


class _Bert:
    def run(self, names, feeds):
        n = len(feeds["input_ids"][0])
        return [np.repeat(np.arange(n, dtype=np.float32)[:, None], 2, 1)]


class _Onnx:
    def __init__(self):
        self.feeds = None

    def run(self, names, feeds):
        self.feeds = feeds
        return [np.full((1, 300), 0.4, np.float32)]


def main():
    synth_mod, g2p = _load_reference()
    from tokenizers import BertWordPieceTokenizer
    words = sorted({w for t in TEXTS for w in t.replace("—", "-").replace("+", "").replace("_", " ").lower().split()})
    words = sorted({p.strip(",.!?;:\"()") for w in words for p in w.split("-")} - {""})
    dic, vocab = {}, list(SPECIAL) + [",", ".", "!", "?", "-", "\"", "(", ")", ":", ";"]
    for w in words:
        h = zlib.crc32(w.encode())
        if h % 3 == 0:
            dic[w] = g2p.convert(w)
        n = _norm(w)
        if w == "абырвалг" or len(n) > 100:
            continue
        if h % 4 == 1 and len(n) > 3:               # only reachable as pieces
            vocab += [n[:2], "##" + n[2:]]
        elif h % 7 != 3:
            vocab.append(n)
    vocab = list(dict.fromkeys(vocab))
    vpath = os.path.join(GOLDEN, "multistream_vocab.txt")
    with open(vpath, "w", encoding="utf-8") as f:
        f.write("\n".join(vocab) + "\n")
    dic["мой"] = "m o0 j"                           # a dictionary pronunciation that convert would not give
    phones = set()
    for t in TEXTS:
        for pattern in ("(\\.\\.\\.|- |[ ,.?!;:\"()])", "(\\.\\.\\.|- |[ ,.?!;:\"()_])"):   # the splits of synth.py:276, :364
            for w in re.split(pattern, t.strip().replace("—", "-").replace(" -", "- ").lower()):
                if w and not re.match(pattern, w) and w not in ("-", "\""):
                    phones.update((dic[w] if w in dic else g2p.convert(w)).split())
    id_map = {}
    for p in PUNCT:
        id_map[p] = len(id_map)
    for p in sorted(phones - set(PUNCT)):
        for s in ("", "_B", "_I", "_E", "_S"):
            id_map[p + s] = len(id_map)
    for p in ("_B", "_I", "_S"):                    # the "_" phone's suffixed forms but __E
        id_map["_" + p] = len(id_map)
    tok = BertWordPieceTokenizer(vpath, unk_token="[UNK]", lowercase=True)

    cases, direct = [], []
    for i, text in enumerate(TEXTS):
        for name, (model_type, with_bert) in VARIANTS.items():
            onnx = _Onnx()
            model = types.SimpleNamespace(dic=dic, tokenizer=tok if with_bert else None, bert_onnx=_Bert(), onnx=onnx,
                                          config={"model_type": model_type, "phoneme_id_map": id_map,
                                                  "inference": {"noise_level": 0.667, "speech_rate": 1.0, "duration_noise_level": 0.8,
                                                                "scale": 1.0}})
            kw = {"speaker_id": i % 3, "speech_rate": 1.25 if i % 4 == 1 else None, "scale": 0.5 if i % 5 == 2 else None}
            case = {"text": text, "variant": name, "args": kw}
            try:
                audio = synth_mod.Synth(model).synth_audio(text, **kw)
                f = onnx.feeds
                case.update({"input": f["input"][0].T.tolist(), "input_lengths": f["input_lengths"].tolist(),
                             "rows": None if not with_bert else f["bert"][0, 0].astype(int).tolist(),
                             "bert_shape": list(f["bert"].shape),
                             "phone_duration_extra": None if f["phone_duration_extra"] is None else f["phone_duration_extra"][0].tolist(),
                             "scales": f["scales"].tolist(), "sid": f["sid"].tolist(), "audio": audio.tolist()[:4],
                             "audio_len": int(audio.size), "error": None})
            except (KeyError, IndexError) as e:
                case["error"] = type(e).__name__
            cases.append(case)
        s = synth_mod.Synth(types.SimpleNamespace(dic=dic, tokenizer=tok, bert_onnx=_Bert(), config={"phoneme_id_map": id_map}))
        d = {"text": text}
        for nopunc in (False, True):
            enc = tok.encode(text.replace("+", "").replace("_", ""))
            d["tokens"], d["ids"] = enc.tokens, enc.ids
            d["selected_nopunc" if nopunc else "selected"] = s.get_word_bert(text, nopunc=nopunc)[:, 0].astype(int).tolist()
        emb = np.arange(200, dtype=np.int64)[:, None]
        for key, fn in (("g2p_multistream", lambda e: s.g2p_multistream(text, e)),
                        ("g2p_multistream_pos", lambda e: s.g2p_multistream(text, e, word_pos=True)),
                        ("g2p_multistream_scales", lambda e: s.g2p_multistream_scales(text, e))):
            try:
                r = fn(emb)
                d[key] = {"ids": [list(map(int, x)) for x in r[0]], "rows": [int(x[0]) for x in r[1]],
                          "extra": list(r[2]) if len(r) > 2 else None}
            except KeyError as e:
                d[key] = {"error": "KeyError"}
        direct.append(d)
    out = {"vocab": os.path.basename(vpath), "dictionary": dic, "phoneme_id_map": id_map, "cases": cases, "direct": direct}
    with open(os.path.join(GOLDEN, "multistream_front.json"), "w", encoding="utf-8") as f:
        json.dump(out, f, ensure_ascii=False, indent=0)
    errs = [(c["variant"], c["text"], c["error"]) for c in cases if c["error"]]
    print("%d cases, errors: %s" % (len(cases), errs))


if __name__ == "__main__":
    main()
