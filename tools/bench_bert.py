"""Times BERT on the GPU (Engine.bert_features: embeddings and the 10 post-LN layers bert-export.py runs, rubert-base's shape,
seeded synthetic weights) in precision modes 0 (fp32 FFMA) and 1 (split-bf16 tensor cores): one 40-piece sentence, and 64
ragged sentences of 8-128 pieces.  Every figure is the median of CUDA events around the call and of a host clock ending in a
synchronise (the rows are on the host); the rate is the FLOPs from the shapes (oracle/bert_oracle.flops) over the host time.
With --cpu it also times transformers' BertModel on the CPU in fp32 for the 40-piece sentence, labelled as such (the
reference runs the graph on ONNX Runtime, which is not installed here).  Prints the card, its power limit and SM clocks, and
one JSON line.

    python tools/bench_bert.py [--rounds 20] [--warmup 3] [--cpu]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bert_inputs as BI  # noqa: E402
import stabletts_cfm_inputs as SI  # noqa: E402
from bench_stabletts import card, timed  # noqa: E402
from oracle import bert_oracle  # noqa: E402
from vosk_tts_b200 import config as C, synthetic  # noqa: E402
from vosk_tts_b200.stabletts import StableTTS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bert.py measures on a GPU; none is visible")
    bt = C.bert_config({"vocab_size": 120000})        # rubert-base's vocabulary size
    sd = synthetic.make_random_bert(bt, 77)
    out = {"card": card(), "mflop_per_piece_gemm": round(bert_oracle.flops(bt, 1) / 1e6, 2)}
    print("card (name, power limit, max SM clock, SM clock):", out["card"])
    rng = np.random.default_rng(0)
    one = [BI.sentence(bt, 40)]
    ragged = [BI.sentence(bt, int(L), salt=i) for i, L in enumerate(rng.integers(8, 129, 64))]
    for precision in (0, 1):
        tts = StableTTS(None, SI.model(), precision=precision, bert=(sd, bt))
        res = {}
        for name, sents in (("sentence_40", one), ("ragged_64", ragged)):
            fn = lambda: tts.engine.bert_features(sents)
            for _ in range(a.warmup):
                fn()
            ms_ev, ms_host = timed(fn, a.rounds)
            fl = sum(bert_oracle.flops(bt, len(s)) for s in sents)
            res[name] = {"pieces": int(sum(len(s) for s in sents)), "ms_events": round(ms_ev, 3), "ms_host": round(ms_host, 3),
                         "tflops_host": round(fl / (ms_host * 1e-3) / 1e12, 2)}
            print("precision %d" % precision, name, json.dumps(res[name]))
        tts.close()
        out["precision%d" % precision] = res
    if a.cpu:
        import transformers
        cfg = transformers.BertConfig(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                                      vocab_size=bt["bt_vocab"])
        m = transformers.BertModel(cfg, add_pooling_layer=False).eval()
        m.load_state_dict(sd)
        x = torch.as_tensor(one[0])[None]
        with torch.no_grad():
            for _ in range(a.warmup):
                m(input_ids=x, output_hidden_states=True)
            t = []
            for _ in range(a.rounds):
                t0 = time.perf_counter()
                m(input_ids=x, output_hidden_states=True)
                t.append((time.perf_counter() - t0) * 1e3)
        out["cpu_torch_bertmodel_sentence_40_ms"] = round(float(np.median(t)), 2)
        out["cpu_threads"] = torch.get_num_threads()
        print("CPU, torch BertModel fp32 (all 12 layers), 40 pieces: %.2f ms on %d threads" % (out["cpu_torch_bertmodel_sentence_40_ms"],
                                                                                                out["cpu_threads"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
