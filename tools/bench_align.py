"""Forced alignment (vtts_align) on the reference architecture with synthetic weights, precision mode 1: a B=1 call on a ~10 s
clip (the speech fixture tiled) with ~300 tokens, and a B=64 ragged call (1-8 s clips, ~3 frames per token).  For each: the
engine stream's time of a whole call (CUDA events on the engine's stream around the host-API call: input copy, every kernel,
output copy) and the host wall time of the call, as aligned audio-seconds per second; then the repo's CPU oracle
(oracle/align_oracle.align, all host cores) on the B=1 clip as the CPU comparison.  Prints the card's name, power limit and
SM clock of the same run and one JSON line."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import vc_inputs as VI  # noqa: E402
from oracle import align_oracle as ao, vc_oracle as vo  # noqa: E402
from vosk_tts_b200 import config as CF, synthetic, weights  # noqa: E402
from vosk_tts_b200.engine import Engine  # noqa: E402
from bench_convert import timed  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                      # noqa: BLE001
        q = "nvidia-smi unavailable: %s" % ex
    return q


def tokens(rng, n, nv):
    ids = rng.randint(1, nv, size=n).astype(np.int64)
    ids[1::2] = 0
    return ids


def main():
    precision = int(os.environ.get("VTTS_PRECISION", "1"))
    cfg = CF.DEFAULT_CONFIG
    sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234, posterior=True))
    blob, man = weights.pack(sd, cfg, posterior=True)
    e = Engine(cfg, blob, man, precision=precision)
    sr, hop, nv = cfg["sampling_rate"], 256, cfg["n_vocab"]
    sp = VI.speech()
    src = np.tile(np.concatenate([sp["a"], sp["b"]]), 8)
    clip = VI.wav_float(src[: 10 * sr + 77])
    rng = np.random.RandomState(0)
    ids1 = tokens(rng, 301, nv)
    lens = rng.randint(sr, 8 * sr, size=64)
    batch = np.zeros((64, int(lens.max())), np.float32)
    for b in range(64):
        o = rng.randint(0, src.size - lens[b])
        batch[b, : lens[b]] = VI.wav_float(src[o:o + lens[b]])
    tx = np.maximum(1, (lens // hop) // 3)
    idsb = np.zeros((64, tx.max()), np.int64)
    for b in range(64):
        idsb[b, : tx[b]] = tokens(rng, tx[b], nv)
    out = {"gpu": card(), "precision": precision}
    for name, fn, n_samples, n_tok in (("b1_10s_301tok", lambda: e.align(ids1, 301, 3, clip, seed=1), clip.size, 301),
                                       ("b64_ragged", lambda: e.align(idsb, tx, np.arange(64) % 200, batch, lens, seed=1),
                                        int(lens.sum()), int(tx.sum()))):
        for _ in range(3):
            fn()                                   # eager, capture, first replay
        dev, host = timed(e, fn, 20)
        out[name] = {"audio_s": n_samples / sr, "tokens": n_tok, "device_ms": dev * 1e3, "host_api_ms": host * 1e3,
                     "audio_s_per_s": n_samples / sr / host}
    e.close()
    torch.set_num_threads(os.cpu_count())
    d = VI.training_json("mel")["data"]
    t0 = time.perf_counter()
    with torch.no_grad():
        spec = vo.mel_spectrogram(torch.from_numpy(clip)[None], d["filter_length"], d["n_mel_channels"], sr, d["hop_length"],
                                  d["win_length"], d["mel_fmin"], d["mel_fmax"])[0].numpy()
        ao.align(sd, cfg, ids1, spec, 3, torch.randn(1, cfg["inter_channels"], spec.shape[1]))
    cpu = time.perf_counter() - t0
    out["cpu_oracle_b1_10s"] = {"threads": os.cpu_count(), "s": cpu, "audio_s_per_s": clip.size / sr / cpu}
    out["gpu_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
