"""Stores the reference's forced alignment -- the head of the UNMODIFIED SynthesizerTrn.forward (training/vits2/models.py:
1632-1660) -- for the CPU and GPU tests, so that they run without the reference tree.

Run where the reference tree is present (``python oracle/build_ref_mas.py && python oracle/make_golden_align.py``); writes
ONLY tests/golden/ref_alignment.npz.  Substitutions, all from outside the model:
  * ``monotonic_align`` is the reference's own compiled Cython MAS (oracle/_ref, built by oracle/build_ref_mas.py) behind a
    wrapper that also keeps the neg_cent it is given;
  * the first ``torch.randn_like`` (enc_q's posterior sample, models.py:841) returns the case's seeded eps; later draws
    (duration predictor, training only) are the library's;
  * ``use_noise_scaled_mas`` is off.
Per case of tests/align_inputs.CASES: ids, sid, the path as the token of every frame, w (frames per token), z_p, m_p and
logs_p in full, neg_cent sampled (golden_ref.sample_index), and the float64 2-best margin of the reference's neg_cent.  The
input spectrograms are the reference front end's, already stored in ref_voice_conversion.npz (align_inputs.ref_spec).
"""
import glob
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import align_oracle as ao, ref_harness as rh  # noqa: E402
from oracle.make_golden_vc import build_reference_model  # noqa: E402
from vosk_tts_b200 import config as C, synthetic  # noqa: E402
import align_inputs as AI  # noqa: E402
import golden_ref as GR  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def reference_mas():
    so = glob.glob(os.path.join(ROOT, "oracle", "_ref", "ref_mas_core*.so"))
    if not so:
        raise SystemExit("run oracle/build_ref_mas.py first")
    spec = importlib.util.spec_from_file_location("ref_mas_core", so[0])
    core = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(core)
    seen = []

    def maximum_path(neg_cent, mask):       # the interface SynthesizerTrn.forward calls (models.py:1658)
        seen.append(neg_cent.detach().clone())
        v = neg_cent.detach().cpu().numpy().astype(np.float32)
        path = np.zeros(v.shape, np.int32)
        t_ys = mask.sum(1)[:, 0].detach().cpu().numpy().astype(np.int32)
        t_xs = mask.sum(2)[:, 0].detach().cpu().numpy().astype(np.int32)
        core.maximum_path_c(path, v, t_ys, t_xs)
        return torch.from_numpy(path).to(neg_cent.dtype)

    ma = types.ModuleType("monotonic_align")
    ma.maximum_path = maximum_path
    return ma, seen


def main():
    assert rh.available(), "needs the reference tree"
    torch.set_num_threads(4)
    ma, seen = reference_mas()
    models = rh.import_reference()
    models.monotonic_align = ma
    out, nets = {}, {}
    for case, clip, model, sid, _ in AI.CASES:
        tj = AI.training_json(model)
        cfg = C.from_training_json(tj, n_vocab=AI.n_vocab(model))
        if model not in nets:
            sd = synthetic.make_random_checkpoint(cfg, AI.SEEDS[model], posterior=True)
            net = build_reference_model(sd, tj, AI.n_vocab(model), cfg["spec_channels"])
            net.enc_q.enc.remove_weight_norm()
            net.use_noise_scaled_mas = False
            nets[model] = net
        net = nets[model]
        spec = torch.from_numpy(AI.ref_spec(case))[None]
        T = spec.shape[2]
        assert T == AI.frames(clip)
        ids = torch.from_numpy(AI.ids(case))[None]
        eps = AI.eps_q(case, cfg["inter_channels"], T)
        calls = {"n": 0}
        orig = torch.randn_like

        def randn_like(x, **kw):
            calls["n"] += 1
            if calls["n"] == 1:
                assert tuple(x.shape) == tuple(eps.shape)
                return eps.clone()
            return orig(x, **kw)

        kept = {}
        hook = net.enc_p.register_forward_hook(lambda m, i, o: kept.update(m_p=o[1], logs_p=o[2]))
        torch.randn_like = randn_like
        del seen[:]
        try:
            with torch.no_grad():
                r = net(ids, torch.tensor([ids.shape[1]]), spec, torch.tensor([T]),
                        sid=torch.tensor([sid]) if cfg["n_speakers"] > 0 else None)
        finally:
            torch.randn_like = orig
            hook.remove()
        attn, z_p = r[3], r[7][1]
        path = attn[0, 0].numpy().astype(np.int32)                  # [t_y, t_x]
        assert (path.sum(1) == 1).all()
        tof, w = ao.path_of(path)
        assert np.array_equal(w, attn.sum(2)[0, 0].numpy().astype(np.int32))
        nc = seen[0][0].numpy().astype(np.float32)
        best, second = ao.two_best(nc.astype(np.float64), T, ids.shape[1])
        p = case + "/"
        out[p + "ids"], out[p + "sid"] = ids[0].numpy(), np.int64(sid)
        out[p + "token_of_frame"], out[p + "w"] = tof, w
        out[p + "z_p"] = z_p[0].numpy().astype(np.float32)
        out[p + "m_p"] = kept["m_p"][0].numpy().astype(np.float32)
        out[p + "logs_p"] = kept["logs_p"][0].numpy().astype(np.float32)
        idx = GR.sample_index(nc.size, p + "neg_cent").astype(np.int32)
        out[p + "neg_cent_shape"], out[p + "neg_cent_idx"], out[p + "neg_cent"] = np.array(nc.shape), idx, nc.reshape(-1)[idx]
        out[p + "margin"] = np.float64(best - second)
        print(case, "t_y", T, "t_x", ids.shape[1], "margin", best - second)
    np.savez_compressed(os.path.join(GOLDEN, "ref_alignment.npz"), **out)


if __name__ == "__main__":
    main()
