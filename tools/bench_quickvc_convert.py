"""Times QuickVC conversion (vtts_quickvc_convert) on the GPU through the host API, g precomputed, with the card name, power
limit and SM clock read in the same run: a 10 s source (500 content frames) at batch 1 and 64 ragged clips (2-10 s) in one
call, in precision modes 1 and 0; the model FLOP of each from the shapes; the float64 CPU oracle on the same 10 s source.
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
import quickvc_convert_inputs as QC  # noqa: E402
import quickvc_inputs as QI  # noqa: E402
from oracle import quickvc_convert_oracle as O  # noqa: E402
from vosk_tts_b200 import weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def flop_per_frame(cfg):
    """Multiply-adds x 2 of one content frame: enc_p, the flow, the decoder (conv_pre, upsamplers, MRF stages, conv_post)."""
    H, I, C0 = cfg["hidden_channels"], cfg["inter_channels"], cfg["upsample_initial_channel"]
    f = 768 * H + 16 * (5 * H * 2 * H + H * 2 * H) + H * 2 * I                       # enc_p (last rss is H wide: close enough)
    f += cfg["flow_n_flows"] * (I // 2 * H + cfg["flow_wn_layers"] * (5 * H * 2 * H + H * 2 * H) + H * I // 2)
    f += 7 * I * C0
    ch, rate = C0, 1
    for u, K in zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"]):
        f += rate * ch * (ch // 2) * K                                                # transposed conv: K taps per input frame
        ch //= 2
        rate *= u
        for k, ds in zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]):
            f += rate * len(ds) * 2 * k * ch * ch
    f += rate * 7 * ch * cfg["subbands"] * (cfg["gen_istft_n_fft"] + 2)
    return 2.0 * f


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
    sd = weights.fold_weight_norm(QC.model())
    blob, man = weights.pack_quickvc(sd, cfg)
    g = np.random.RandomState(0).rand(256).astype(np.float32)
    g /= np.linalg.norm(g)
    u10 = QC.units(500, 0)
    rng = np.random.default_rng(0)
    lens = rng.integers(100, 500, 64)
    clips = [QC.units(int(n), 1)[:int(n)] for n in lens]
    fpf = flop_per_frame(cfg)
    out = {"gpu_before": gpu_info(), "flop_per_frame": fpf}
    for precision in (1, 0):
        eng = Engine(cfg, blob, man, device=0, precision=precision)
        for _ in range(3):
            eng.quickvc_convert(u10, g)
            eng.quickvc_convert(clips, g)
        t1 = timed(lambda: eng.quickvc_convert(u10, g), 30)
        t64 = timed(lambda: eng.quickvc_convert(clips, g), 10)
        out["mode%d" % precision] = {"src10s_ms": round(t1, 3), "src10s_tflops": round(fpf * 500 / t1 / 1e9, 2),
                                     "ragged64_ms": round(t64, 3), "ragged64_tflops": round(fpf * float(lens.sum()) / t64 / 1e9, 2),
                                     "ragged64_audio_s": round(float(lens.sum()) * 0.02, 1)}
        eng.close()
    out["gpu_after"] = gpu_info()
    t0 = time.perf_counter()
    O.infer(u10, g, sd, cfg, QC.eps(500, 0))
    out["cpu_oracle_src10s_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    out["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
