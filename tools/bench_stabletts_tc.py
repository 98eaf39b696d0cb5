"""Times StableTTS's mel phase in precision mode 2 (convs and attention on the split-bf16 tensor cores) against mode 1 (fp32
FFMA), in alternating rounds on the same seeded weights and inputs.  Shapes: the decoder and text encoder at their reference
widths (H 384, F 768, 6 blocks), HiFi-GAN v1, 22050 Hz / hop 256 (86.1 frames per second).  Workloads:
  - one 10 s utterance (861 frames) through the decoder alone, 10 steps, guidance 0.5;
  - 150 tokens text to waveform, 5 steps;
  - 64 ragged utterances of 2-10 s through the decoder alone, 10 steps.
Every figure is the median over rounds of a host clock ending in a synchronise (results are on the host).  TFLOP/s is the
decoder's estimator work (its dense convs and attention, both branches, counted from the shapes) over the call's time.
Prints the card, its power limit and SM clocks, read in the same run, and one JSON line.

    python tools/bench_stabletts_tc.py [--rounds 15] [--warmup 3]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import hifigan_inputs as HI  # noqa: E402
from bench_stabletts import card  # noqa: E402
from vosk_tts_b200 import config as C, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402
from vosk_tts_b200.stabletts import StableTTS  # noqa: E402


def estimator_flops(cfg, frames, steps, guided=True):
    """FLOPs of the estimator's dense convs and attention over `frames` rows, `steps` Euler steps (x2 with guidance), plus
    cond_proj once per branch."""
    NC, MC, H, F, NL, k = (int(cfg[n]) for n in ("noise_channels", "cond_channels", "hidden_channels", "filter_channels", "n_layers", "kernel_size"))
    br = 2 if guided else 1
    per_row = (NC + H) * H + NL * (3 * H * H + H * H + 2 * k * H * F) + (NL // 2) * k * 2 * H * H + H * NC
    f = 0.0
    for T in frames:
        f += 2.0 * br * steps * (T * per_row + NL * 2 * T * T * H)         # convs, then q k^T and p v
        f += 2.0 * br * T * k * (MC * F + F * F + F * H)                     # cond_proj
    return f


def median_ms(fn, rounds):
    t = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    rng = np.random.default_rng(5)
    cfg = C.stabletts_cfm_config()
    sd = synthetic.make_random_stabletts_cfm(cfg, 11)
    engs = {}
    for p in (1, 2):
        blob, man = weights.pack_stabletts_cfm(sd, cfg, precision=p)
        engs[p] = Engine(cfg, blob, man, device=0, precision=p)
    tcfg = C.stabletts_config({"n_vocab": 120})
    tsd = synthetic.make_random_stabletts(tcfg, 12)
    tts = {p: StableTTS({"n_vocab": 120}, tsd, device=0, precision=p, vocoder=HI.folded()) for p in (1, 2)}

    one = [rng.standard_normal((861, cfg["cond_channels"]), dtype=np.float32)]
    lens64 = rng.integers(172, 862, 64)
    many = [rng.standard_normal((int(T), cfg["cond_channels"]), dtype=np.float32) for T in lens64]
    T = 150
    ids = rng.integers(0, 120, (tcfg["n_streams"], T))
    bert = rng.standard_normal((tcfg["bert_dim"], T), dtype=np.float32)
    frames = {}

    def text(p):
        r = tts[p].synthesise(ids, bert, 0, n_timesteps=5, return_wav=True)
        frames["text"] = r["mel_lengths"]
        return r

    work = {
        "cfm_10s": (lambda p: engs[p].cfm_decode(one, 0, n_timesteps=10), estimator_flops(cfg, [861], 10)),
        "text_150_wav": (text, None),
        "cfm_64_ragged": (lambda p: engs[p].cfm_decode(many, 0, n_timesteps=10),
                          estimator_flops(cfg, [int(v) for v in lens64], 10)),
    }
    res = {}
    for name, (fn, flops) in work.items():
        for p in (1, 2):
            for _ in range(a.warmup):
                fn(p)
        # alternating rounds: mode 1, mode 2, mode 1, ...
        ts = {1: [], 2: []}
        for _ in range(a.rounds):
            for p in (1, 2):
                ts[p].append(median_ms(lambda: fn(p), 1))
        if flops is None:
            flops = estimator_flops(cfg, [int(frames["text"])], 5)
        res[name] = {("mode%d" % p): {"ms": round(float(np.median(ts[p])), 3), "tflops": round(float(flops / (np.median(ts[p]) * 1e-3) / 1e12), 2)}
                     for p in (1, 2)}
        res[name]["speedup"] = round(res[name]["mode1"]["ms"] / res[name]["mode2"]["ms"], 3)
        print(name, res[name])
    # the same calls' outputs in the two modes: how far mode 2's mel moves
    m1, _ = engs[1].cfm_decode(one, 0, n_timesteps=10)
    m2, _ = engs[2].cfm_decode(one, 0, n_timesteps=10)
    res["cfm_10s"]["max_abs_diff_mode2_vs_mode1"] = float(np.abs(m1 - m2).max())
    print("card:", card())
    print(json.dumps({"card": card(), "results": res}))
    for p in (1, 2):
        engs[p].close()
        tts[p].close()


if __name__ == "__main__":
    main()
