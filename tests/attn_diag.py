"""TEST INFRASTRUCTURE (not collected): per-row error map of the tensor-core attention against the torch reference."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_gpu_attention import ref_attention, _inputs
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine
cfg = C.DEFAULT_CONFIG
w = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234))
blob, man = weights.pack(w, cfg)
eng = Engine(cfg, blob, man, device=0, precision=1)
a = "flow.flows.0.pre_transformer.attn_layers.0"
relk, relv = w[a + ".emb_rel_k"][0].double(), w[a + ".emb_rel_v"][0].double()
H = 192
for T, kind in [(129, "plain"), (129, "peaky"), (192, "plain"), (256, "plain"), (320, "plain"), (700, "plain")]:
    qkv = _inputs(T, H, 100 + T, kind)
    ref = ref_attention(qkv, relk, relv, 2, 4).numpy()
    for rep in range(2):
        out, ms = eng.debug_attention("flow.0.tr", qkv.float().numpy(), 1, iters=20)
        e = np.abs(out - ref)
        rows = e.max(1)
        bad = np.nonzero(rows > 2e-4)[0]
        print("T=%d %s rep%d: max %.3e  ms %.4f  bad rows %d %s  head0 %.2e head1 %.2e" % (T, kind, rep, e.max(), ms, len(bad), bad[:8], e[:, :96].max(), e[:, 96:].max()))
out, ms = eng.debug_attention("flow.0.tr", _inputs(4765, H, 1, "plain").float().numpy(), 1, iters=10)
print("T=4765 tc ms", ms)
out, ms = eng.debug_attention("flow.0.tr", _inputs(4765, H, 1, "plain").float().numpy(), 0, iters=3)
print("T=4765 ffma ms", ms)
out, ms = eng.debug_attention("flow.0.tr", _inputs(162, H, 1, "plain").float().numpy(), 1, iters=50)
print("T=162 tc ms", ms)
out, ms = eng.debug_attention("flow.0.tr", _inputs(162, H, 1, "plain").float().numpy(), 0, iters=50)
print("T=162 ffma ms", ms)
