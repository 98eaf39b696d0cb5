"""Writes tests/golden/ref_stabletts.npz: the seed, the inputs (tests/stabletts_inputs.py) and what the *unmodified* reference
MatchaTTS.synthesise (training/stabletts/matcha/models/matcha_tts.py:93-211) produces for seeded synthetic weights, inputs and
noise: w_round, mel_lengths, decoder_outputs, mel and encoder_outputs.  Needs the reference tree (ref_harness.REF_ROOT); the
tests read only the fixture.

To keep the fixture under a megabyte it stores nothing that follows exactly from what it holds, and this script checks each
such identity bit for bit before it writes: the BERT features and the noise are seeded (their SHA-1 is stored), mel is
decoder_outputs * mel_std + mel_mean in fp32, and encoder_outputs is one column per token repeated w_round times.
stabletts_inputs.load_golden gives the tests the full set back.

The reference modules are imported as they are, on the import shims of make_golden_stabletts_cfm.py.  What matcha_tts.py and
baselightningmodule.py import on top of those and inference never calls is stubbed here: `lightning` (LightningModule becomes an
nn.Module with a no-op save_hyperparameters), matcha.utils.utils.plot_tensor and matcha.utils.monotonic_align.  The noise is
injected by replacing torch.randn for the call: synthesise draws it over the frame axis padded to a multiple of 4, so the
fixture stores those T_pad columns.  Each utterance goes through alone (batch 1), which is how the engine defines a ragged
batch."""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import stabletts_inputs as SI  # noqa: E402
from oracle import make_golden_stabletts_cfm as cfm_maker  # noqa: E402


def import_reference_matcha():
    cfm_maker.import_reference_cfm()
    sys.modules["matcha.utils"].get_pylogger = sys.modules["matcha.utils.pylogger"].get_pylogger
    if "lightning" not in sys.modules:
        class LightningModule(torch.nn.Module):
            def save_hyperparameters(self, *a, **k):
                pass
        lt, lp, lu = (types.ModuleType(n) for n in ("lightning", "lightning.pytorch", "lightning.pytorch.utilities"))
        lt.LightningModule, lu.grad_norm = LightningModule, None
        lt.pytorch, lp.utilities = lp, lu
        sys.modules.update({"lightning": lt, "lightning.pytorch": lp, "lightning.pytorch.utilities": lu})
    for name, attrs in (("matcha.utils.utils", {"plot_tensor": None}), ("matcha.utils.monotonic_align", {})):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            sys.modules[name] = m
            setattr(sys.modules["matcha.utils"], name.rsplit(".", 1)[1], m)
    from matcha.models import matcha_tts
    return matcha_tts


def build_reference(mt, cfg, sd):
    ns = types.SimpleNamespace
    enc = ns(encoder_type="dit", encoder_params=ns(n_feats=int(cfg["noise_channels"]), n_channels=int(cfg["cond_channels"])))
    model = mt.MatchaTTS(n_vocab=int(cfg["n_vocab"]), n_spks=int(cfg["n_spks"]), spk_emb_dim=int(cfg["spk_emb_dim"]),
                         n_feats=int(cfg["noise_channels"]), encoder=enc, duration_predictor=ns(name="deterministic"), decoder={},
                         cfm=ns(solver="euler", sigma_min=1e-4), data_statistics={"mel_mean": float(sd["mel_mean"]), "mel_std": float(sd["mel_std"])},
                         out_size=None)
    model.load_state_dict(sd, strict=True)
    return model.eval()


def reference_synthesise(model, ids, bert, pause, noise, sid, n, temperature, length_scale):
    drawn = {}
    orig = torch.randn

    def randn(*shape, **k):
        drawn["cols"] = int(shape[-1])
        return torch.from_numpy(noise[None, :, :shape[-1]].copy())
    torch.randn = randn
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            out = model.synthesise(torch.from_numpy(ids)[None], torch.tensor([ids.shape[1]]), n, temperature=temperature,
                                   spks=torch.tensor([sid]), bert=torch.from_numpy(bert)[None], length_scale=length_scale,
                                   phone_duration_extra=None if pause is None else torch.from_numpy(pause)[None])
    finally:
        torch.randn = orig
    w = out["attn"][0, 0].sum(1).long().numpy()
    return {"w_round": w, "mel_lengths": out["mel_lengths"].numpy(), "decoder_outputs": out["decoder_outputs"][0].numpy(),
            "mel": out["mel"][0].numpy(), "encoder_outputs": out["encoder_outputs"][0].numpy(), "noise": noise[:, :drawn["cols"]]}


def main():
    mt = import_reference_matcha()
    cfg = SI.config()
    sd = SI.model(cfg)
    model = build_reference(mt, cfg, sd)
    out = {"seed": np.int64(SI.SEED), "cases": np.array([c[0] for c in SI.CASES]),
           "mel_mean": np.float32(sd["mel_mean"]), "mel_std": np.float32(sd["mel_std"])}
    for case in SI.CASES:
        name, lens, sids, n, temp, ls, pauses = case
        for b, (ids, bert, pause, noise) in enumerate(SI.case_inputs(case)):
            r = reference_synthesise(model, ids, bert, pause if pauses.get(b) else None, noise, sids[b], n, temp, ls)
            T = int(r["mel_lengths"][0])
            assert r["noise"].shape[1] == (T + 3) // 4 * 4 and int(r["w_round"].sum()) == T
            w = r["w_round"]
            first = np.cumsum(w) - w
            assert np.array_equal(r["noise"], noise[:, :(T + 3) // 4 * 4])
            assert np.array_equal(r["mel"], SI.denormalise(r["decoder_outputs"], out["mel_mean"], out["mel_std"]))
            assert np.array_equal(r["encoder_outputs"], np.repeat(r["encoder_outputs"][:, first], w, 1))
            k = name + ".%s" + str(b)
            out[k % "ids"], out[k % "pause"] = ids.astype(np.int16), pause
            out[k % "bert_sha1"], out[k % "noise_sha1"] = np.array(SI.sha1(bert)), np.array(SI.sha1(noise))
            out[k % "w_round"], out[k % "mel_lengths"] = w, r["mel_lengths"]
            out[k % "decoder_outputs"], out[k % "encoder_tokens"] = r["decoder_outputs"], r["encoder_outputs"][:, first]
            print(name, b, "tokens", ids.shape[1], "frames", T, "mod 4 =", T % 4)
    path = os.path.join(ROOT, "tests", "golden", "ref_stabletts.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
