"""Times the QuickVC speaker encoder (vtts_speaker_embedding) on the GPU, with the card name, power limit and SM clock read in
the same run: the enrolment of a 10 s target, 64 ragged targets in one call, the LSTM recurrence kernel's device time, and
the float64 CPU oracle on the same 10 s clip.  Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import quickvc_inputs as QI  # noqa: E402
from oracle import quickvc_oracle as O, vc_oracle  # noqa: E402
from vosk_tts_b200 import weights  # noqa: E402
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
    cfg = QI.config()
    sd = QI.speaker_encoder()
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(sd), cfg)
    eng = Engine(cfg, blob, man, device=0, precision=1)
    rng = np.random.default_rng(0)
    wav10 = (0.1 * rng.standard_normal(10 * 16000)).astype(np.float32)
    lens = rng.integers(2 * 16000, 10 * 16000, 64)
    batch = (0.1 * rng.standard_normal((64, int(lens.max())))).astype(np.float32)
    for _ in range(5):
        eng.speaker_embedding(wav10)
        eng.speaker_embedding(batch, lens)
    info0 = gpu_info()
    t1 = timed(lambda: eng.speaker_embedding(wav10), 50)
    t64 = timed(lambda: eng.speaker_embedding(batch, lens), 20)
    info1 = gpu_info()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            eng.speaker_embedding(wav10)
        torch.cuda.synchronize()
    rec = [e for e in prof.key_averages() if "lstm_rec_kernel" in e.key]
    rec_us = sum(e.device_time_total for e in rec) / 20.0 if rec else None
    y = torch.from_numpy(wav10)[None].double()
    t0 = time.perf_counter()
    mel = vc_oracle.mel_spectrogram(y, cfg["filter_length"], cfg["n_mel_channels"], cfg["sampling_rate"], cfg["hop_length"],
                                    cfg["win_length"], cfg["mel_fmin"], cfg["mel_fmax"])[0].numpy()
    O.embed(mel, sd)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"gpu_before": info0, "gpu_after": info1, "enrol_10s_ms": round(t1, 3), "ragged64_ms": round(t64, 3),
                      "ragged64_audio_s": round(float(lens.sum()) / 16000, 1),
                      "recurrence_device_us_per_call": None if rec_us is None else round(rec_us, 1),
                      "cpu_oracle_10s_ms": round(cpu_ms, 1), "cpu_threads": torch.get_num_threads()}))
    eng.close()


if __name__ == "__main__":
    main()
