"""Times the StableTTS vocoder on seeded synthetic weights, in precision modes 0 (fp32 FFMA) and 1 (split-bf16 tensor cores
for every upsampling conv and the MRFs of stages 1-3): the vocoder alone (Engine.hifigan_vocode) on a 10 s mel (860 frames)
and on 64 ragged 2-10 s mels, and text-to-waveform (Engine.stabletts_synthesise with want_wav) against text-to-mel on a
150-token utterance and 64 ragged ones.  Every figure is taken with CUDA events around the call and with a host clock ending
in a synchronise; the vocoder's rate is its FLOPs (from the shapes) over the host time.  Also reports the library's device
bytes after the largest call (its workspace only grows, so this is the peak).  Prints the card, its power limit and SM clock,
and one JSON line.

    python tools/bench_hifigan.py [--rounds 10] [--warmup 3]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

from bench_stabletts import card, timed, workload  # noqa: E402
from vosk_tts_b200 import config as C, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine, live_bytes  # noqa: E402


def flops_per_frame(h, n_mels=80):
    """Multiply-adds x 2 of the Generator per mel frame: conv_pre, each ConvTranspose1d (K taps per input row over its phases),
    each MRF (2 convs per dilation of ResBlock1 at the stage's rate), conv_post."""
    c = int(h["upsample_initial_channel"])
    f = 2.0 * n_mels * c * 7
    rm = 1
    for u, k in zip(h["upsample_rates"], h["upsample_kernel_sizes"]):
        f += 2.0 * c * (c // 2) * k * rm
        rm *= u
        c //= 2
        for ks, dils in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
            f += len(dils) * 2 * 2.0 * c * c * ks * rm
    return f + 2.0 * c * 7 * rm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hifigan.py measures on a GPU; none is visible")
    cfg = C.stabletts_config({"n_vocab": 120})
    h = C.hifigan_config()
    sd = synthetic.make_random_stabletts(cfg, 9753)
    voc = (weights.fold_weight_norm(synthetic.make_random_hifigan(4242, h)), h)
    fpf = flops_per_frame(h)
    out = {"card": card(), "gflop_per_frame": round(fpf / 1e9, 4)}
    print("card (name, power limit, max SM clock, SM clock):", out["card"])
    rng = np.random.default_rng(0)
    single = [860]
    ragged = [int(v) for v in rng.integers(172, 861, 64)]            # 2-10 s at 22 050 Hz / 256
    tok_ragged = [int(v) for v in rng.integers(30, 151, 64)]
    for precision in (0, 1):
        base = live_bytes()[0]
        ecfg = dict(cfg, vocoder=h)
        eng = Engine(ecfg, *weights.pack_stabletts(sd, cfg, vocoder=voc), device=0, precision=precision)
        res = {}
        for name, lens in (("vocode_860", single), ("vocode_ragged_64", ragged)):
            mels = [(-5.5 + 2.1 * rng.standard_normal((T, 80))).astype(np.float32) for T in lens]
            fn = lambda: eng.hifigan_vocode(mels)
            for _ in range(a.warmup):
                fn()
            v = [timed(fn, 1) for _ in range(a.rounds)]
            r = {"frames": int(sum(lens)), "ms_events": round(float(np.median([x[0] for x in v])), 3),
                 "ms_host": round(float(np.median([x[1] for x in v])), 3)}
            r["tflops_host"] = round(fpf * sum(lens) / (r["ms_host"] * 1e-3) / 1e12, 2)
            res[name] = r
            print("precision %d" % precision, name, json.dumps(r))
        for name, lens in (("text_150_tokens", [150]), ("text_ragged_64", tok_ragged)):
            ids, bert, ln = workload(cfg, rng, lens)
            kw = dict(lengths=ln, n_timesteps=10, seed=1)
            mel = lambda: eng.stabletts_synthesise(ids, bert, 1, **kw)
            wav = lambda: eng.stabletts_synthesise(ids, bert, 1, want_wav=True, **kw)
            frames = int(mel()["mel_lengths"].sum())
            for _ in range(a.warmup):
                mel(), wav()
            acc = {"text_to_mel": [], "text_to_wav": []}
            for _ in range(a.rounds):
                for k, fn in (("text_to_mel", mel), ("text_to_wav", wav)):
                    acc[k].append(timed(fn, 1))
            r = {"frames": frames}
            for k, v in acc.items():
                r[k + "_ms_events"] = round(float(np.median([x[0] for x in v])), 3)
                r[k + "_ms_host"] = round(float(np.median([x[1] for x in v])), 3)
            res[name] = r
            print("precision %d" % precision, name, json.dumps(r))
        res["device_bytes_after"] = live_bytes()[0] - base
        eng.close()
        out["precision%d" % precision] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
