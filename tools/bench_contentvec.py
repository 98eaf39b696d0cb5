"""Times ContentVec (vtts_content_units) and conversion from source waveforms (vtts_quickvc_convert_wav, g precomputed) on the
GPU through the host API, with the card name, power limit and SM clock read before and after in the same run: a 10 s source
(499 frames) at batch 1 and 64 ragged sources (2-10 s) in one call, in precision modes 1 and 0; ContentVec's FLOP per frame
from the shapes (oracle.contentvec_oracle.flops_per_frame) and TFLOP/s end to end; the fp32 CPU restatement of ContentVec
(oracle/contentvec_oracle.py, which matches the reference module within 1e-5) on the same 10 s source.  Prints one JSON line."""
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
import quickvc_convert_inputs as QC  # noqa: E402
import quickvc_inputs as QI  # noqa: E402
from oracle import contentvec_oracle as O  # noqa: E402
from vosk_tts_b200 import config as C, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402


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
    import torch
    cv = CI.cv()
    cfg = dict(QI.config(), contentvec=cv)
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    g = np.random.RandomState(0).rand(256).astype(np.float32)
    g /= np.linalg.norm(g)
    x10 = CI.speech(160000, 0)
    rng = np.random.default_rng(0)
    lens = rng.integers(32000, 160001, 64)
    clips = [CI.speech(int(n), i) for i, n in enumerate(lens)]
    frames = np.array([C.contentvec_frames(int(n)) for n in lens])
    flops = lambda T: O.flops_per_frame(cv, T) * T
    f10, f64 = flops(499), float(sum(flops(int(T)) for T in frames))
    out = {"gpu_before": gpu_info(), "mflop_per_frame_10s": round(f10 / 499 / 1e6, 1)}
    for precision in (1, 0):
        eng = Engine(cfg, blob, man, device=0, precision=precision)
        eng.reserve_contentvec(160000, 64)
        for _ in range(3):
            eng.content_units(x10)
            eng.quickvc_convert_wav(x10, g)
            eng.content_units(clips)
        t_u = timed(lambda: eng.content_units(x10), 20)
        t_w = timed(lambda: eng.quickvc_convert_wav(x10, g), 20)
        t_64 = timed(lambda: eng.content_units(clips), 5)
        out["mode%d" % precision] = {"units10s_ms": round(t_u, 3), "units10s_tflops": round(f10 / t_u / 1e9, 2),
                                     "wav2wav10s_ms": round(t_w, 3),
                                     "units_ragged64_ms": round(t_64, 2), "units_ragged64_tflops": round(f64 / t_64 / 1e9, 2),
                                     "ragged64_audio_s": round(float(lens.sum()) / 16000, 1)}
        eng.close()
    out["gpu_after"] = gpu_info()
    t0 = time.perf_counter()
    with torch.no_grad():
        O.contentvec_units(CI.folded(), cv, x10, torch.float32)
    out["cpu_fp32_units10s_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
