"""Times resampling of recordings on the GPU (vtts_resample) through the host API, with the card name, power limit and SM clock
read in the same run: 64 ragged clips of 2-10 s at 44.1 and at 48 kHz resampled to 16 kHz in one call, with and without
the trim.  Reports the call time twice: from CUDA events recorded on the engine's stream around the call (its uploads,
kernels and readback) and from the host clock around the call (which ends in a stream synchronise).  Then the output samples
per second and the kernels' own time (torch.profiler, in a separate pass).  The bytes the kernels move over that time are
given against the H100 SXM's 3.35 TB/s twice: the algorithmic minimum (input read once, output written once, read once
more by the trim's energies), and that plus the taps every CTA re-reads from L2 into shared memory; the single-thread
scipy.signal.resample_poly time of the same clips on this host; and QuickVC waveform to waveform for a 10 s source at
44.1 kHz (resampled in the same call chain) next to the same source at 16 kHz.  Prints one JSON line."""
import json
import math
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
from vosk_tts_b200 import quickvc, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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


def event_ms(eng, fn, n):
    """Median time between CUDA events recorded on the engine's stream right before and after the call."""
    import torch
    st = torch.cuda.ExternalStream(eng.stream())
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernel_ms(fn, n):
    """Mean GPU time per call of each of the engine's resampling kernels, from torch.profiler over n calls."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
    out = {}
    for ev in prof.key_averages():
        for k in ("resample_kernel", "frame_energy_kernel"):
            if k in ev.key:
                out[k] = out.get(k, 0.0) + ev.device_time_total / 1e3 / n
    return out


def rs_window(tile, up, down, K):
    return ((tile - 1) * down + up - 1) // up + K + 1      # resample.cuh's rs_window


def tap_rereads(lens, fr, to):
    """Bytes of taps the CTAs of one resample_kernel launch load (resample.cuh's tile and shared-memory rules)."""
    g = math.gcd(fr, to)
    up, down = to // g, fr // g
    K = -(-(20 * max(up, down) + 1) // up)
    if up * (K | 1) > 16384:
        return 0                                            # taps read through L2 per output, not staged
    tile = 1024
    while tile > 32 and rs_window(tile, up, down, K) > 16384:
        tile //= 2
    ctas = sum(-(-(-(-int(n) * up // down)) // tile) for n in lens)
    return ctas * up * K * 4


def main():
    import scipy.signal
    import torch
    torch.cuda.init()
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    eng = Engine(dict(QI.config(), contentvec=CI.cv()), blob, man, device=0, precision=1)
    out = {"gpu_before": gpu_info()}
    rng = np.random.default_rng(0)
    for fr in (44100, 48000):
        lens = rng.integers(2 * fr, 10 * fr, 64)
        clips = [(rng.standard_normal(int(n)) * 0.1).astype(np.float32) for n in lens]
        for c in clips:
            c[: fr // 2] = 0.0                                   # half a second of leading silence for the trim to cut
        n_in = int(lens.sum())
        n_out = int(sum(-(-int(n) * 160 // (fr // 100)) for n in lens))
        res = {"audio_s": round(n_in / fr, 1), "samples_in": n_in, "samples_out": n_out}
        for trim in (None, 20.0):
            key = "trim" if trim else "plain"
            for _ in range(3):
                eng.resample(clips, fr, 16000, trim_top_db=trim)
            ms = timed(lambda: eng.resample(clips, fr, 16000, trim_top_db=trim), 20)
            ev_ms = event_ms(eng, lambda: eng.resample(clips, fr, 16000, trim_top_db=trim), 20)
            km = kernel_ms(lambda: eng.resample(clips, fr, 16000, trim_top_db=trim), 10)
            kt = sum(km.values())
            moved = 4 * (n_in + n_out) + (4 * n_out if trim else 0)
            taps = tap_rereads(lens, fr, 16000)
            res[key] = {"call_ms_host": round(ms, 3), "call_ms_device_events": round(ev_ms, 3),
                        "out_samples_per_s": round(n_out / ms * 1e3, 0),
                        "kernel_ms": {k: round(v, 4) for k, v in km.items()}, "kernel_bytes_min": moved,
                        "kernel_bytes_with_tap_rereads": moved + taps,
                        "kernel_TBps_min": round(moved / kt / 1e9, 3) if kt else None,
                        "share_of_3.35TBps_min": round(moved / kt / 1e9 / (HBM_BYTES_PER_S / 1e12), 3) if kt else None,
                        "kernel_TBps_with_tap_rereads": round((moved + taps) / kt / 1e9, 3) if kt else None}
        t0 = time.perf_counter()
        for c in clips:
            scipy.signal.resample_poly(c, 160, fr // 100)
        res["cpu_resample_poly_1thread_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        out["from_%d" % fr] = res
    eng.close()
    # QuickVC waveform to waveform: a 10 s source at 16 kHz, and the same length at 44.1 kHz resampled first
    vc = quickvc.QuickVC.__new__(quickvc.QuickVC)
    vc.engine = Engine(dict(QI.config(), contentvec=CI.cv()), blob, man, device=0, precision=1)
    vc.sampling_rate = 16000
    g = np.random.RandomState(0).rand(256).astype(np.float32)
    g /= np.linalg.norm(g)
    s16, s44 = CI.speech(160000, 1), CI.speech(441000, 2)
    for _ in range(3):
        vc.convert(s16, g=g)
        vc.convert(s44, g=g, sampling_rate=44100)
    out["quickvc_wav2wav_10s_16k_ms"] = round(timed(lambda: vc.convert(s16, g=g), 20), 3)
    out["quickvc_wav2wav_10s_44k_ms"] = round(timed(lambda: vc.convert(s44, g=g, sampling_rate=44100), 20), 3)
    vc.close()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
