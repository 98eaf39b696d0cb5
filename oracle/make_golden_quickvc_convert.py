"""Stores the reference QuickVC conversion (SynthesizerTrn.infer, vc/models.py:862-872, as vc/convert.py:62-87 calls it) for
the GPU and CPU tests, so that they run without the reference tree.

Run where the reference tree is present (``python oracle/make_golden_quickvc_convert.py``); writes ONLY
tests/golden/ref_quickvc_convert.npz:
  <case>/m_p, /logs_p, /z_p, /z   float32 [inter_channels][frames] (enc_p's stats and sample, the reverse flow's output) at
                                  quickvc_convert_inputs.kept_frames(T): every frame, but 72 of the 250 of the longest case
  <case>/o                        float32 [320 T], the waveform
  <case>/g                        float32 [256], the g infer computed from the target's log-mel
  names, shapes                   the sorted names and shapes of the reference model's whole state dict
for every case (T, target) of tests/quickvc_convert_inputs.CASES, each run alone (B = 1), as convert.py runs.  The model is
the unmodified vc/models.py with the shims of make_golden_quickvc.py, loaded strictly with the seeded checkpoint
quickvc_convert_inputs.model() and run in float64 (net.double()); the units and the noise are quickvc_convert_inputs.units /
eps, the noise
standing in for torch.randn_like in PosteriorEncoder.forward (models.py:270).  The target's log-mel is the one stored in
ref_quickvc.npz.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import make_golden_quickvc as MG  # noqa: E402
import quickvc_inputs as QI  # noqa: E402
import quickvc_convert_inputs as QC  # noqa: E402


def main():
    torch.set_num_threads(4)
    models, _ = MG.import_reference_vc()
    hps = QI.QUICKVC_JSON
    d = hps["data"]
    with contextlib.redirect_stdout(io.StringIO()):
        net = models.SynthesizerTrn(d["filter_length"] // 2 + 1, 10240 // d["hop_length"], **hps["model"]).eval()
    sd = net.state_dict()
    names = sorted(sd)
    out = {"names": np.array(names), "shapes": np.array([",".join(map(str, sd[k].shape)) for k in names])}
    net.load_state_dict(QC.model(), strict=True)
    net = net.double()
    ref = np.load(os.path.join(QI.GOLDEN, "ref_quickvc.npz"))
    seen = {}
    net.enc_p.register_forward_hook(lambda m, a, r: seen.update(z_p=r[0], m_p=r[1], logs_p=r[2]))
    net.flow.register_forward_hook(lambda m, a, r: seen.update(z=r))
    for i, (T, key) in enumerate(QC.CASES):
        c = torch.from_numpy(QC.units(T, i).T.copy()).double()[None]           # [1, 768, T], as convert.py's c
        eps = torch.from_numpy(QC.eps(T, i)).double()[None]
        mel = torch.from_numpy(ref[key + "/mel"]).double()[None]
        orig = torch.randn_like
        torch.randn_like = lambda m: eps.to(m.dtype)
        try:
            with torch.no_grad():
                o = net.infer(c, mel=mel)
                g = net.enc_spk.embed_utterance(mel.transpose(1, 2))
        finally:
            torch.randn_like = orig
        case = "T%d" % T
        keep = QC.kept_frames(T)
        for k in ("m_p", "logs_p", "z_p", "z"):
            out["%s/%s" % (case, k)] = seen[k][0].numpy()[:, keep].astype(np.float32)
        out[case + "/o"] = o[0, 0].numpy().astype(np.float32)
        out[case + "/g"] = g[0].numpy().astype(np.float32)
        print(case, key, o.shape, float(o.abs().max()))
    np.savez_compressed(os.path.join(QI.GOLDEN, "ref_quickvc_convert.npz"), **out)


if __name__ == "__main__":
    main()
