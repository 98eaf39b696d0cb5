"""Times the StableTTS flow-matching decoder (vtts_cfm_decode) on the GPU, with the card name, power limit and SM clock read
before and after in the same run: a 10 s utterance (860 frames at hop 256 / 22.05 kHz) and 64 ragged utterances (2-10 s) in one
call, 10 Euler steps with guidance 0.5, precision modes 1 and 0; the host API's wall clock (staging, copies and kernels, ending
in the call's synchronise) and CUDA events on the engine's stream around the call; TFLOP/s end to end from the FLOP model of
the shapes (flops_per_frame below); the fp32 CPU restatement (oracle/stabletts_cfm_oracle.py, which matches the reference
within 2e-5) on the 10 s utterance.  Both modes run the same fp32 FFMA kernels today, so their numbers measure the spread.
Prints one JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import stabletts_cfm_inputs as SI  # noqa: E402
from oracle import stabletts_cfm_oracle as O  # noqa: E402
from vosk_tts_b200 import weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def flops_per_frame(cfg, T, guided=True):
    """FLOP of one Euler step per mel frame of a T-frame utterance: the estimator's convs (2 Cin Cout k each) and the
    attention's QK^T and PV (4 T hidden per block), for both branches when guided.  cond_proj runs once per call and is
    counted by flops_per_call."""
    NC, H, F, NL, k = (cfg[n] for n in ("noise_channels", "hidden_channels", "filter_channels", "n_layers", "kernel_size"))
    blk = 2 * (H * 3 * H + H * H + H * F * k + F * H * k) + 4 * T * H
    est = 2 * (NC + H) * H + NL * blk + (NL // 2) * 2 * (2 * H * H * k) + 2 * H * NC
    return est * (2 if guided else 1)


def flops_per_call(cfg, T, n, guided=True):
    MC, H, F, k = (cfg[m] for m in ("cond_channels", "hidden_channels", "filter_channels", "kernel_size"))
    prenet = 2 * k * (MC * F + F * F + F * H) * (2 if guided else 1)
    return T * (n * flops_per_frame(cfg, T, guided) + prenet)


def timed(fn, n, stream):
    import torch
    host, dev = [], []
    s = torch.cuda.ExternalStream(stream)
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        t0 = time.perf_counter()
        fn()
        host.append(time.perf_counter() - t0)
        b.record(s)
        b.synchronize()
        dev.append(a.elapsed_time(b))
    return float(np.median(host)) * 1e3, float(np.median(dev))


def main():
    import torch
    cfg = SI.config()
    sd = SI.model(cfg)
    blob, man = weights.pack_stabletts_cfm(sd, cfg)
    n, T10 = 10, 860
    mu10, nz10 = SI.inputs("bench", T10)
    lens = np.random.default_rng(0).integers(172, 861, 64)
    batch = [SI.inputs("bench%d" % i, int(T))[0].T for i, T in enumerate(lens)]
    f10, f64 = flops_per_call(cfg, T10, n), float(sum(flops_per_call(cfg, int(T), n) for T in lens))
    out = {"gpu_before": gpu_info(), "steps": n, "guidance": 0.5, "mflop_per_frame_step": round(flops_per_frame(cfg, T10) / 1e6, 1)}
    for precision in (1, 0):
        eng = Engine(cfg, blob, man, device=0, precision=precision)
        for _ in range(3):
            eng.cfm_decode(mu10.T, 0, n_timesteps=n, noise=nz10.T)
            eng.cfm_decode(batch, 0, n_timesteps=n)
        h1, d1 = timed(lambda: eng.cfm_decode(mu10.T, 0, n_timesteps=n, noise=nz10.T), 20, eng.stream())
        h64, d64 = timed(lambda: eng.cfm_decode(batch, 0, n_timesteps=n), 5, eng.stream())
        out["mode%d" % precision] = {"utt10s_host_ms": round(h1, 3), "utt10s_event_ms": round(d1, 3), "utt10s_tflops": round(f10 / d1 / 1e9, 2),
                                     "ragged64_host_ms": round(h64, 2), "ragged64_event_ms": round(d64, 2),
                                     "ragged64_tflops": round(f64 / d64 / 1e9, 2), "ragged64_frames": int(lens.sum())}
        eng.close()
    out["gpu_after"] = gpu_info()
    t0 = time.perf_counter()
    O.decode(sd, cfg, mu10, 0, nz10, n, 1.0, 0.5, torch.float32)
    out["cpu_fp32_utt10s_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
