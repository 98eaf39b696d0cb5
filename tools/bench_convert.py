"""Voice conversion (vtts_convert) on the reference architecture with synthetic weights: a B=1 call on a ~10 s clip (the speech
fixture tiled) and a B=64 ragged call, precision mode 1.  For each: the engine stream's time of a whole call (CUDA events on
the engine's stream around the host-API call: input copy, every kernel, output copy) and the host wall time of the call,
samples/s and RTF; then the repo's CPU oracle (oracle/vc_oracle.voice_conversion, all host cores) on the B=1 clip as the
CPU comparison.  Prints one JSON line."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import vc_inputs as VI  # noqa: E402
from oracle import vc_oracle as vo  # noqa: E402
from vosk_tts_b200 import config as CF, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402


def timed(e, fn, reps):
    st = torch.cuda.ExternalStream(e.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev, host = [], []
    for _ in range(reps):
        e0.record(st)
        t0 = time.perf_counter()
        fn()
        host.append(time.perf_counter() - t0)
        e1.record(st)
        e1.synchronize()
        dev.append(e0.elapsed_time(e1) / 1e3)
    return float(np.median(dev)), float(np.median(host))


def main():
    precision = int(os.environ.get("VTTS_PRECISION", "1"))
    cfg = CF.DEFAULT_CONFIG
    sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234, posterior=True))
    blob, man = weights.pack(sd, cfg, posterior=True)
    e = Engine(cfg, blob, man, precision=precision)
    sr = cfg["sampling_rate"]
    sp = VI.speech()
    clip = VI.wav_float(np.tile(np.concatenate([sp["a"], sp["b"]]), 4)[: 10 * sr + 77])
    rng = np.random.RandomState(0)
    lens = rng.randint(sr, 8 * sr, size=64)
    batch = np.zeros((64, int(lens.max())), np.float32)
    src = np.tile(np.concatenate([sp["a"], sp["b"]]), 8)
    for b in range(64):
        o = rng.randint(0, src.size - lens[b])
        batch[b, : lens[b]] = VI.wav_float(src[o:o + lens[b]])
    out = {"gpu": torch.cuda.get_device_name(0), "precision": precision}
    for name, fn, n_samples in (("b1_10s", lambda: e.convert(clip, 3, 7, seed=1), clip.size),
                                ("b64_ragged", lambda: e.convert(batch, np.arange(64) % 200, (np.arange(64) * 7) % 200,
                                                                 lengths=lens, seed=1), int(lens.sum()))):
        for _ in range(3):
            fn()                                   # eager, capture, first replay
        dev, host = timed(e, fn, 10)
        out[name] = {"samples": n_samples, "audio_s": n_samples / sr, "device_ms": dev * 1e3, "host_api_ms": host * 1e3,
                     "samples_per_s": n_samples / host, "rtf": host / (n_samples / sr)}
    e.close()
    torch.set_num_threads(os.cpu_count())
    d = VI.training_json("mel")["data"]
    y = torch.from_numpy(clip)[None]
    t0 = time.perf_counter()
    with torch.no_grad():
        spec = vo.mel_spectrogram(y, d["filter_length"], d["n_mel_channels"], sr, d["hop_length"], d["win_length"], d["mel_fmin"],
                                  d["mel_fmax"])
        T = spec.shape[2]
        vo.voice_conversion(sd, cfg, spec, torch.tensor([T]), torch.tensor([3]), torch.tensor([7]),
                            torch.randn(1, cfg["inter_channels"], T))
    cpu = time.perf_counter() - t0
    out["cpu_oracle_b1_10s"] = {"threads": os.cpu_count(), "s": cpu, "rtf": cpu / (clip.size / sr)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
