"""Writes tests/golden/ref_hifigan.npz: what the *unmodified* reference vocoder (the Generator of
training/stabletts/matcha/hifigan/models.py:148-206, built from config v1 as cli.py:65-71 builds it, after remove_weight_norm)
gives for the seeded weights and mels of tests/hifigan_inputs.py, each utterance alone, followed by clamp(-1, 1) as cli.py:126
does; and for two reference mels of tests/golden/ref_stabletts.npz (MatchaTTS.synthesise's `mel`), the text-to-waveform chain.
Needs the reference tree (ref_harness.REF_ROOT); the tests read only the fixture.

The 56 MB of weights are not stored: they are seeded, and the fixture keeps the SHA-1 of the checkpoint the script builds the
reference model from and of the state dict remove_weight_norm leaves, plus two of the folded tensors in full.  The mels of
the seeded cases are stored.  matcha/hifigan/xutils.py imports matplotlib at module load for its plotting helper, which
inference never calls: it is stubbed, and the package __init__ files are replaced by bare packages."""
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

import hifigan_inputs as HI  # noqa: E402
from oracle import ref_harness  # noqa: E402


def import_reference_hifigan():
    root = os.path.join(ref_harness.REF_ROOT, "training", "stabletts")
    if not os.path.isfile(os.path.join(root, "matcha", "hifigan", "models.py")):
        raise RuntimeError("reference tree not present at %s" % ref_harness.REF_ROOT)
    if "matplotlib" not in sys.modules:
        mpl, pylab = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.pylab")
        mpl.use = lambda *a, **k: None
        mpl.pylab = pylab
        sys.modules.update({"matplotlib": mpl, "matplotlib.pylab": pylab})
    for pkg in ("matcha", "matcha.hifigan"):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = [os.path.join(root, *pkg.split("."))]
            sys.modules[pkg] = m
    import importlib
    return (importlib.import_module("matcha.hifigan.models"), importlib.import_module("matcha.hifigan.config"),
            importlib.import_module("matcha.hifigan.env"))


def main():
    models, config, env = import_reference_hifigan()
    torch.manual_seed(0)
    gen = models.Generator(env.AttrDict(config.v1))
    ck = HI.checkpoint()
    gen.load_state_dict(ck)
    with contextlib.redirect_stdout(io.StringIO()):
        gen.remove_weight_norm()
    gen.eval()
    sd = gen.state_dict()
    out = {"seed": np.int64(HI.SEED), "sha1_checkpoint": np.array(HI.sha1_state(ck)), "sha1_folded": np.array(HI.sha1_state(sd)),
           "folded.conv_post.weight": sd["conv_post.weight"].numpy(), "folded.ups.3.weight": sd["ups.3.weight"].numpy()}

    def run(mel):
        with torch.no_grad():
            return gen(torch.from_numpy(np.ascontiguousarray(mel, np.float32))[None]).clamp(-1, 1)[0, 0].numpy()
    for case in HI.CASES:
        for b, m in enumerate(HI.case_mels(case)):
            out["%s.mel%d" % (case[0], b)] = m
            out["%s.wav%d" % (case[0], b)] = run(m)
    st = dict(np.load(os.path.join(ROOT, "tests", "golden", "ref_stabletts.npz")))
    for key in HI.TEXT_CASES:
        dec = st[key.replace(".mel", ".decoder_outputs")]
        mel = dec * np.float32(st["mel_std"]) + np.float32(st["mel_mean"])       # the reference's denormalize, fp32
        out["text." + key + ".wav"] = run(mel)
    np.savez_compressed(HI.GOLDEN, **out)
    print("wrote", HI.GOLDEN, os.path.getsize(HI.GOLDEN), "bytes")


if __name__ == "__main__":
    main()
