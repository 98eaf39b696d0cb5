"""Times StableTTS text-to-mel against its decoder alone on seeded synthetic weights: a 150-token utterance (about 860 frames)
and a ragged batch of 64.  For each, alternating in one process: Engine.cfm_decode on mu rows of the same frame counts, the full
Engine.stabletts_synthesise, and the text phase alone (a call given no room for the mel, which returns after the frame
counts).  Every figure is taken twice: with CUDA events around the calls and with a host clock ending in a synchronise.  Prints
the card, its power limit and SM clock, and one JSON line.

    python tools/bench_stabletts.py [--rounds 10] [--warmup 3] [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vosk_tts_b200 import config as C, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine, VttsError  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    return q


def workload(cfg, rng, lens):
    T = max(lens)
    ids = rng.integers(0, cfg["n_vocab"], (len(lens), cfg["n_streams"], T))
    bert = rng.standard_normal((len(lens), T, cfg["bert_dim"]), dtype=np.float32)
    return ids, bert, np.array(lens, np.int64)


def timed(fn, rounds):
    """(device-event ms, host-clock ms) medians of `rounds` calls; every call ends synchronised (results are on the host)."""
    ev, host = [], []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        host.append((time.perf_counter() - t0) * 1e3)
        ev.append(a.elapsed_time(b))
    return float(np.median(ev)), float(np.median(host))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--length-scale", type=float, default=1.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stabletts.py measures on a GPU; none is visible")
    cfg = C.stabletts_config({"n_vocab": 120})
    sd = synthetic.make_random_stabletts(cfg, 9753)
    eng = Engine(cfg, *weights.pack_stabletts(sd, cfg), device=0, precision=1)
    rng = np.random.default_rng(0)
    out = {"card": card(), "steps": a.steps}
    print("card (name, power limit, max SM clock, SM clock):", out["card"])
    for name, lens in (("single_150_tokens", [150]), ("ragged_64", [int(v) for v in rng.integers(20, 151, 64)])):
        ids, bert, ln = workload(cfg, rng, lens)
        kw = dict(lengths=ln, n_timesteps=a.steps, length_scale=a.length_scale, seed=1)
        full = lambda: eng.stabletts_synthesise(ids, bert, 1, **kw)
        r = full()
        frames = [int(v) for v in r["mel_lengths"]]
        mu = [rng.standard_normal((f, cfg["cond_channels"]), dtype=np.float32) for f in frames]      # the decoder's cost depends on the shape only
        dec = lambda: eng.cfm_decode(mu, 1, n_timesteps=a.steps, seed=1)

        def text_only():
            try:
                eng.stabletts_synthesise(ids, bert, 1, mel_frames=1, **kw)
            except VttsError as ex:
                assert ex.code == -4
        res = {"tokens": int(ln.sum()), "frames": int(sum(frames)), "longest": max(frames)}
        for _ in range(a.warmup):
            dec(), full(), text_only()
        acc = {"decoder": [], "text_to_mel": [], "text_phase": []}
        for _ in range(a.rounds):          # alternating, so that a drifting clock touches all three alike
            for k, fn in (("decoder", dec), ("text_to_mel", full), ("text_phase", text_only)):
                acc[k].append(timed(fn, 1))
        for k, v in acc.items():
            res[k + "_ms_events"] = round(float(np.median([x[0] for x in v])), 3)
            res[k + "_ms_host"] = round(float(np.median([x[1] for x in v])), 3)
        res["text_to_mel_over_decoder"] = round(res["text_to_mel_ms_host"] / res["decoder_ms_host"], 4)
        out[name] = res
        print(name, json.dumps(res))
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
