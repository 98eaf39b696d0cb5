"""Writes tests/golden/ref_contentvec.npz from the unmodified reference ContentVec (vc/contentvec.py's HubertModelWithFinalProj
on transformers, eager attention, fp32 as vc/encode.py runs it) with the seeded weights of tests/contentvec_inputs.py.

Per clip (400, 719, 720 and 16000 samples, and 10 s, of contentvec_inputs.speech(n, n)): the units, every frame except the
10 s clip's, of which the frames at both ends and in the middle (contentvec_inputs.kept_frames) are kept.  For the 16000-sample
clip also the feature encoder's output and the transformer's input.  Two end-to-end cases (contentvec_inputs.E2E): the reference
ContentVec's units of a source, then the reference QuickVC SynthesizerTrn.infer (vc/models.py, float64, the seeded checkpoint
of quickvc_convert_inputs, as make_golden_quickvc_convert.py runs it) with quickvc_convert_inputs.eps standing in for
torch.randn_like and a stored target's log-mel: e2e<i>/o the waveform, e2e<i>/g the target's g.

    python oracle/make_golden_contentvec.py        (needs the reference tree and transformers)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
sys.path.insert(0, os.path.join(HERE, ".."))

import contentvec_inputs as CI  # noqa: E402
import quickvc_convert_inputs as QC  # noqa: E402
import quickvc_inputs as QI  # noqa: E402
from oracle import make_golden_quickvc as MG  # noqa: E402


def end_to_end(net, out):
    import contextlib
    import io
    models, _ = MG.import_reference_vc()
    hps = QI.QUICKVC_JSON
    d = hps["data"]
    with contextlib.redirect_stdout(io.StringIO()):
        vc = models.SynthesizerTrn(d["filter_length"] // 2 + 1, 10240 // d["hop_length"], **hps["model"]).eval()
    vc.load_state_dict(QC.model(), strict=True)
    vc = vc.double()
    ref = np.load(os.path.join(QI.GOLDEN, "ref_quickvc.npz"))
    for i, (n, key) in enumerate(CI.E2E):
        with torch.no_grad():
            c = net.extract(torch.from_numpy(CI.speech(n, 500 + i))[None]).transpose(2, 1).double()     # as convert.py:82
        T = c.shape[2]
        eps = torch.from_numpy(QC.eps(T, 500 + i)).double()[None]
        mel = torch.from_numpy(ref[key + "/mel"]).double()[None]
        orig = torch.randn_like
        torch.randn_like = lambda m: eps.to(m.dtype)
        try:
            with torch.no_grad():
                o = vc.infer(c, mel=mel)
                g = vc.enc_spk.embed_utterance(mel.transpose(1, 2))
        finally:
            torch.randn_like = orig
        out["e2e%d/o" % i] = o[0, 0].numpy()
        out["e2e%d/g" % i] = g[0].numpy()
        print("e2e", i, n, T, o.shape)


def main():
    net = CI.build_reference(CI.model())
    out = {}
    for n in CI.LENGTHS + (CI.LONG,):
        x = torch.from_numpy(CI.speech(n, n))[None]
        with torch.no_grad():
            if n == 16000:
                feat = net.feature_extractor(x).transpose(1, 2)
                h = net.feature_projection(feat)
                h = h[0] if isinstance(h, tuple) else h
                h = net.encoder.layer_norm(h + net.encoder.pos_conv_embed(h))
                out["s%d/feat" % n] = feat[0].numpy()
                out["s%d/enc_in" % n] = h[0].numpy()
            u = net.extract(x)[0].numpy()
        out["s%d/units" % n] = u[CI.kept_frames(u.shape[0])] if n == CI.LONG else u
        out["s%d/frames" % n] = np.int64(u.shape[0])
        print(n, u.shape)
    end_to_end(net, out)
    path = os.path.join(CI.GOLDEN, "ref_contentvec.npz")
    np.savez_compressed(path, **{k: np.asarray(v, np.float32) if np.asarray(v).dtype.kind == "f" else v for k, v in out.items()})
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
