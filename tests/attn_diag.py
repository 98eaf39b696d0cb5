"""TEST INFRASTRUCTURE (not collected): error / bound and device time of each attention kernel on a few shapes."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import attn_ref as ar
from test_gpu_attention import make_qkv
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine
cfg = C.DEFAULT_CONFIG
blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234)), cfg)
eng = Engine(cfg, blob, man, device=0, precision=2)
layer, H, heads, W = "flow.0.tr", cfg["hidden_channels"], 2, cfg["window_size"]
tabs = ar.layer_tables(blob, man, layer, H // heads)
for lens in ([129], [162], [256], [700], [4765], [5, 1, 7], [1, 129, 64, 300]):
    qkv = make_qkv(lens, H, heads, 100 + lens[0], "plain", 70)
    for kernel in ("tc", "split", "r1", "r4"):
        try:
            out, _, rep, ms = eng.debug_attention(layer, qkv, lens, kernel, iters=20)
        except Exception as ex:
            print(lens[:4], kernel, "refused:", ex)
            continue
        res = ar.reference(qkv, lens, heads, W, tabs, "tc" if kernel == "tc" else "ffma")
        print("%-18s %-5s error/bound %.4f  %.4f ms  %s" % (lens[:4], kernel, ar.worst(out, res), ms, rep))
