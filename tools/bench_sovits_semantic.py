"""Times GPT-SoVITS prompt tokens (gpt_sovits.SemanticEncoder.prompts: HuBERT, ssl_proj, the codebook argmax) on the GPU through
the host API, with the card name, power limit and SM clock read before and after in the same run: a 10 s prompt at batch 1 and
64 ragged 3-20 s prompts in one call, in precision modes 1 and 0.  FLOP from the shapes: HuBERT's per frame
(oracle.contentvec_oracle.flops_per_frame) plus the tail's 2 (2 H) H + 2 H K per code.  The share of the call outside HuBERT is
the tail alone (SemanticEncoder.extract_latent on rows of the same counts) over the whole call.  Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import contentvec_inputs as CI  # noqa: E402
import sovits_inputs as SI  # noqa: E402
from oracle import contentvec_oracle as O  # noqa: E402
from vosk_tts_b200 import config as C, synthetic  # noqa: E402
from vosk_tts_b200.gpt_sovits import SemanticEncoder  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def timed(fn, n):
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    cv = SI.cv()
    hub = SI.hubert()
    s2 = synthetic.make_random_sovits(hub)
    cfg = SI.cfg()
    H, K, pad = cv["cv_hidden"], cfg["sv_codebook"], cfg["sovits_pad"]
    x10 = CI.speech(160000, 0)
    rng = np.random.default_rng(0)
    lens = rng.integers(48000, 320001, 64)
    clips = [CI.speech(int(n), i) for i, n in enumerate(lens)]
    frames = lambda n: C.contentvec_frames(int(n) + pad)
    flops = lambda T: O.flops_per_frame(cv, T) * T + (T // 2) * (2 * 2 * H * H + 2 * H * K)
    f10, f64 = flops(frames(160000)), float(sum(flops(frames(n)) for n in lens))
    rows10 = [np.zeros((frames(160000), H), np.float32)]
    rows64 = [np.zeros((frames(n), H), np.float32) for n in lens]
    out = {"gpu_before": gpu_info(), "gflop_10s": round(f10 / 1e9, 2), "ragged64_audio_s": round(float(lens.sum()) / 16000, 1)}
    for precision in (1, 0):
        enc = SemanticEncoder((s2, cfg), (hub, cv), device=0, precision=precision)
        lat = lambda rows: enc.engine.sovits_latent(rows)
        for _ in range(3):
            enc.prompts([x10])
            enc.prompts(clips)
            lat(rows10)
            lat(rows64)
        t1 = timed(lambda: enc.prompts([x10]), 20)
        t64 = timed(lambda: enc.prompts(clips), 5)
        l1 = timed(lambda: lat(rows10), 20)
        l64 = timed(lambda: lat(rows64), 5)
        out["mode%d" % precision] = {"prompt10s_ms": round(t1, 3), "prompt10s_tflops": round(f10 / t1 / 1e9, 2),
                                     "prompt10s_outside_hubert": round(l1 / t1, 3),
                                     "ragged64_ms": round(t64, 2), "ragged64_tflops": round(f64 / t64 / 1e9, 2),
                                     "ragged64_outside_hubert": round(l64 / t64, 3)}
        enc.close()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
