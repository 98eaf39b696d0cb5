"""GPT-SoVITS text-to-semantic decoding on the GPU at the upstream width (24 post-LN layers, 512 wide, 16 heads, 1025 semantic
tokens, 732 phones; seeded weights whose EOS row is zeroed so that early_stop_num pins the step count):
  - B = 1, 100 phones, no prompt, 500 steps;
  - B = 1, 100 phones, a 150-token prompt, 500 steps after it;
  - 64 ragged sentences (40..160 phones, prompts of 0..150 tokens) in one call, 500 steps each.
Times come from a host clock around whole calls (each ends in a device synchronise), the best of --repeats after a warm-up
call of the same shape; ms per step is the whole call (prefill included) over the decode steps.
Weight bytes per step: the fp32 layer weights and ar_predict_layer one step streams, over the step time, against the H100
SXM's 3.35 TB/s.  --profile: one more call under torch.profiler, kernel time by name (a run of its own)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vosk_tts_b200 import config, synthetic               # noqa: E402
from vosk_tts_b200.gpt_sovits import Text2Semantic        # noqa: E402

UPSTREAM = {"hidden_dim": 512, "embedding_dim": 512, "head": 16, "n_layer": 24, "vocab_size": 1025, "phoneme_vocab_size": 732,
            "dropout": 0.0, "EOS": 1024}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception as e:                                   # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--precision", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    cfg = config.t2s_config(UPSTREAM)
    sd = synthetic.make_random_t2s(cfg, 7, eos_scale=0.0)
    H, F, V, L = cfg["cv_hidden"], cfg["cv_ffn"], cfg["t2s_vocab"], cfg["cv_layers"]
    wbytes = 4 * (L * (3 * H * H + H * H + 2 * H * F) + H * V)
    m = Text2Semantic((sd, cfg), precision=a.precision)
    r = np.random.default_rng(0)
    ph = lambda n: r.integers(0, cfg["t2s_phone_vocab"], n)
    pr = lambda n: r.integers(0, V - 1, n)
    cases = {"B1": ([ph(100)], None), "B1_prompt150": ([ph(100)], [pr(150)]),
             "B64_ragged": ([ph(int(n)) for n in r.integers(40, 161, 64)], [pr(int(n)) for n in r.integers(0, 151, 64)])}
    res = {"card": card(), "precision": a.precision, "weight_bytes_per_step": wbytes, "cases": {}}
    for name, (phones, prompts) in cases.items():
        B = len(phones)
        kw = dict(early_stop_num=a.steps - 1, seeds=list(range(B)))
        toks, _ = m.decode(phones, prompts, **kw)                    # warm-up (and graph capture)
        ts = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            toks, _ = m.decode(phones, prompts, **kw)
            ts.append(time.perf_counter() - t0)
        t = min(ts)
        steps = a.steps                                              # the call's time includes its prefill
        gen = sum(len(x) + 1 - (0 if prompts is None else len(prompts[b])) for b, x in enumerate(toks))
        res["cases"][name] = {"B": B, "call_ms": 1e3 * t, "steps": steps, "ms_per_step": 1e3 * t / steps,
                              "tokens_per_s": gen / t, "weight_GBps": wbytes * steps / t / 1e9,
                              "share_of_3.35TBps": wbytes * steps / t / 3.35e12, "all_calls_ms": [1e3 * x for x in ts]}
        print(name, json.dumps(res["cases"][name]), flush=True)
    print(json.dumps(res))
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        phones, prompts = cases["B1"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.decode(phones, prompts, early_stop_num=a.steps - 1, seeds=[0])
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=15))
    m.close()


if __name__ == "__main__":
    main()
