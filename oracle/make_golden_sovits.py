"""Writes tests/golden/ref_sovits_semantic.npz: GPT-SoVITS prompt codes from the unmodified reference, run in float64 on the
CPU on seeded weights (tests/sovits_inputs.py).

HuBERT is transformers' HubertModel with synthetic.make_random_contentvec's weights (without final_proj), called as
inference_cli.py:193 calls ssl_model.model(wav); the tail is the reference's own SynthesizerTrn (module/models.py, built with
the published v1 s2 model shape, semantic_frame_rate "25hz") with the seeded ssl_proj and codebook loaded and inited = 1, and
its extract_latent.  Per case the codes, the margin of every code (best minus second-best score, from the float64 restatement
oracle/sovits_oracle.py, which tests/test_sovits_host.py checks against extract_latent), the best score and the runner-up's
index, and how many distinct codes the case uses.  No weights are stored: the tests regenerate them from their seeds.

    python oracle/make_golden_sovits.py /path/to/training/gpt-sovits
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import sovits_inputs as SI                  # noqa: E402
from oracle import sovits_oracle as O       # noqa: E402

# the published v1 s2 config's model block (GPT-SoVITS configs/s2.json): the tail does not depend on it, but the module is built whole
S2_MODEL = {"inter_channels": 192, "hidden_channels": 192, "filter_channels": 768, "n_heads": 2, "n_layers": 6, "kernel_size": 3,
            "p_dropout": 0.1, "resblock": "1", "resblock_kernel_sizes": [3, 7, 11],
            "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]], "upsample_rates": [10, 8, 2, 2, 2],
            "upsample_initial_channel": 512, "upsample_kernel_sizes": [16, 16, 8, 2, 2], "n_layers_q": 3, "use_spectral_norm": False,
            "gin_channels": 512, "semantic_frame_rate": "25hz", "freeze_quantizer": True}


def reference_hubert(sd):
    """transformers' HubertModel (chinese-hubert-base's class, cnhubert.py) with sd loaded, eager attention, float64."""
    from transformers import HubertConfig, HubertModel
    cfg = HubertConfig(conv_bias=False)
    cfg._attn_implementation = "eager"
    net = HubertModel(cfg).eval()
    sd = {k: v for k, v in sd.items() if not k.startswith("final_proj.")}
    missing, unexpected = net.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert set(missing) <= {"encoder.pos_conv_embed.conv.parametrizations.weight.original0",
                            "encoder.pos_conv_embed.conv.parametrizations.weight.original1"}, missing
    return net.double()


def reference_synthesizer(gpt_sovits, s2):
    """The reference's SynthesizerTrn with the s2 tensors loaded (the rest keeps its init: extract_latent does not read it)."""
    sys.path.insert(0, gpt_sovits)
    from module.models import SynthesizerTrn
    torch.manual_seed(0)
    net = SynthesizerTrn(1025, 32, n_speakers=300, **S2_MODEL).eval()
    missing, unexpected = net.load_state_dict(s2, strict=False)
    assert not unexpected and not any(k in missing for k in s2), (unexpected, missing)
    assert int(net.quantizer.vq.layers[0]._codebook.inited.item()) == 1
    return net.double()


def main(gpt_sovits):
    out = {}
    hub = reference_hubert(SI.hubert())
    with torch.no_grad():
        for sd_name, names in (("s2", list(SI.WAVE) + ["f_odd", "f_even"]), ("s2_ties", ["ties"])):
            s2 = getattr(SI, sd_name)()
            net = reference_synthesizer(gpt_sovits, s2)
            for name in names:
                if name in SI.WAVE:
                    wav = torch.from_numpy(SI.padded(name)).double()
                    ssl = hub(wav.unsqueeze(0))["last_hidden_state"].transpose(1, 2)     # inference_cli.py:193-197
                    out[name + "/samples"] = np.int64(wav.numel())
                else:
                    ssl = torch.from_numpy(SI.feats(name)).double().T[None]
                codes = net.extract_latent(ssl)                                           # [1, 1, T // 2]
                codes = codes[0, 0].numpy().astype(np.int64)
                feats = ssl[0].T.numpy()
                oc, margin, best = O.extract_latent(feats, s2)
                g = lambda k: s2[k].double().numpy()
                sc = O.scores(O.project(feats, g("ssl_proj.weight"), g("ssl_proj.bias")), g("quantizer.vq.layers.0._codebook.embed"))
                sc[np.arange(oc.size), oc] = -np.inf
                out[name + "/second"] = sc.argmax(1).astype(np.int64)
                mismatch = np.nonzero(oc != codes)[0]
                assert all(margin[t] == 0 for t in mismatch), (name, mismatch, margin[mismatch])
                out[name + "/frames"] = np.int64(feats.shape[0])
                out[name + "/codes"] = codes
                out[name + "/margin"] = margin
                out[name + "/best"] = best
                out[name + "/distinct"] = np.int64(len(np.unique(codes)))
                print("%-7s %5d HuBERT frames, %4d codes, %4d distinct, least margin %.3g" %
                      (name, feats.shape[0], codes.size, len(np.unique(codes)), float(margin.min())))
    np.savez_compressed(SI.FIXTURE, **out)
    print("wrote", SI.FIXTURE, os.path.getsize(SI.FIXTURE), "bytes")


if __name__ == "__main__":
    main(os.path.abspath(sys.argv[1]))
