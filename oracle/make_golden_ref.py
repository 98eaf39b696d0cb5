"""Stores what the reference-pinning CPU tests compare against, so that they run without the reference tree.

Run once where the reference tree is present (``python oracle/make_golden_ref.py``); writes under tests/golden/:
  mb_istft_vits2_multi.json   the reference's training configuration of the default architecture
  g2p_reference.json          word -> phonemes of the reference converter (vosk_tts/g2p.py)
  ref_pins.npz                reference outputs of tests/test_oracle_vs_reference.py (seeded inputs, sampled where large)
  ref_decoder_variants.npz    reference outputs of tests/test_decoder_variants.py
"""
import importlib.util
import json
import os
import shutil
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_harness as rh  # noqa: E402
from vosk_tts_b200 import config as C, synthetic  # noqa: E402
import golden_ref as GR  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    assert rh.available(), "needs the reference tree"
    torch.set_num_threads(2)
    shutil.copyfile(rh.REF_CONFIG, os.path.join(GOLDEN, "mb_istft_vits2_multi.json"))

    spec = importlib.util.spec_from_file_location("ref_g2p", os.path.join(rh.REF_ROOT, "vosk_tts", "g2p.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    with open(os.path.join(GOLDEN, "g2p_reference.json"), "w", encoding="utf-8") as f:
        json.dump({w: ref.convert(w) for w in GR.g2p_words()}, f, ensure_ascii=False, indent=0)

    cfg = C.DEFAULT_CONFIG
    net = rh.build_reference_model(synthetic.make_random_checkpoint(cfg, 1234))
    sd = net.state_dict()
    out = {}
    for k, v in sd.items():
        flat = v.detach().reshape(-1).numpy().astype(np.float32)
        out["sd/" + k] = flat[GR.sample_index(flat.size, k, GR.SD_SAMPLE)]
    out["basis"] = sd["dec.stft.inverse_basis"][:, 0].numpy()
    out["pqmf"] = sys.modules["pqmf"].PQMF("cpu").synthesis_filter[0].numpy()
    x, uw, uh, ud = GR.spline_inputs()
    tr = sys.modules["transforms"]
    r, _ = tr.piecewise_rational_quadratic_transform(x.clone(), uw.clone(), uh.clone(), ud.clone(), inverse=True, tails="linear", tail_bound=5.0)
    out["spline"] = r.numpy()
    for T, seed in GR.INFER_CASES:
        tok, eps_dp, eps_z, scales = GR.infer_inputs(T, seed)
        r = rh.reference_infer(net, tok, torch.tensor([T]), torch.tensor([3]), scales, eps_dp, lambda s: eps_z[:, :, : s[2]])
        out["infer%d/o" % T] = r["o"].numpy().astype(np.float32)
        out["infer%d/attn" % T] = r["attn"].numpy().astype(np.uint8)
        z = r["z"].reshape(-1).numpy().astype(np.float32)
        out["infer%d/z_shape" % T] = np.array(r["z"].shape)
        out["infer%d/z" % T] = z[GR.sample_index(z.size, "z%d" % T)]
    np.savez_compressed(os.path.join(GOLDEN, "ref_pins.npz"), **out)

    out = {}
    for flag, kind in GR.DECODER_VARIANTS:
        tj = GR.training_json(flag)
        cfg = C.from_training_json(tj, n_vocab=GR.N_VOCAB)
        net = rh.build_reference_model(synthetic.make_random_checkpoint(cfg, 11), cfg=tj, n_vocab=GR.N_VOCAB)
        tok, eps_dp, eps_z, scales = GR.variant_inputs(cfg)
        torch.set_num_threads(1)
        r = rh.reference_infer(net, tok, torch.tensor([tok.shape[1]]), torch.tensor([2]), scales, eps_dp, lambda s: eps_z[:, :, :s[2]])
        attn = r["attn"][0, 0]
        o = r["o"].reshape(-1).numpy().astype(np.float32)
        out[flag + "/w"] = attn.sum(0).numpy().astype(np.int32)
        out[flag + "/idx"] = attn.argmax(1).numpy()
        out[flag + "/o_shape"] = np.array(r["o"].shape)
        out[flag + "/o"] = o[GR.sample_index(o.size, flag)]
    np.savez_compressed(os.path.join(GOLDEN, "ref_decoder_variants.npz"), **out)


if __name__ == "__main__":
    main()
