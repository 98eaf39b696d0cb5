"""Writes tests/golden/ref_stabletts_cfm.npz: the seed, the inputs (tests/stabletts_cfm_inputs.py) and the mel the *unmodified* reference CFM / Decoder
(training/stabletts/matcha/models/components/flow_matching.py, decoder.py, diffusion_transformer.py) produces for seeded
synthetic weights, inputs and noise.  Needs the reference tree (ref_harness.REF_ROOT); the tests read only the fixture.

The reference modules are imported as they are.  What they import and inference never calls is stubbed here: torchdiffeq
(flow_matching.py:12) and matcha.utils.pylogger's Lightning import.  The noise is injected by replacing torch.randn for the
call, and the line the reference prints at every estimator evaluation (flow_matching.py:183) is swallowed by redirecting
stdout.  CFM.forward fixes the guidance scale at 0.5 (flow_matching.py:61); the s = 0 cases call solve_euler, which takes it as
an argument, with forward's own z and t_span.  Each utterance goes through alone (batch 1), which is how the engine defines a
ragged batch."""
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

import stabletts_cfm_inputs as SI  # noqa: E402
from oracle import ref_harness  # noqa: E402

def import_reference_cfm():
    root = os.path.join(ref_harness.REF_ROOT, "training", "stabletts")
    if not os.path.isfile(os.path.join(root, "matcha", "models", "components", "flow_matching.py")):
        raise RuntimeError("reference tree not present at %s" % ref_harness.REF_ROOT)
    if "torchdiffeq" not in sys.modules:
        td = types.ModuleType("torchdiffeq")
        td.odeint = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("torchdiffeq is stubbed"))
        sys.modules["torchdiffeq"] = td
    # the package __init__ files and pylogger pull in Lightning, hydra, ...: register bare packages and a logger stub
    for pkg in ("matcha", "matcha.models", "matcha.models.components", "matcha.utils"):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = [os.path.join(root, *pkg.split("."))]
            sys.modules[pkg] = m
    if "matcha.utils.pylogger" not in sys.modules:
        import logging
        pl = types.ModuleType("matcha.utils.pylogger")
        pl.get_pylogger = lambda name=__name__: logging.getLogger(name)
        sys.modules["matcha.utils.pylogger"] = pl
    from matcha.models.components import flow_matching
    return flow_matching


def reference_mel(cfm, sd, mu, noise, sid, n, s, temperature):
    orig = torch.randn
    torch.randn = lambda *a, **k: noise[None].clone()
    try:
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
            mask = torch.ones(1, 1, mu.shape[1])
            spk = sd["spk_emb.weight"][sid][None]
            if s == 0.5:
                out = cfm(mu[None], mask, n, temperature, spk, None, sd["fake_speaker"], sd["fake_content"])
            else:
                z = torch.randn(1, 80, mu.shape[1]) * temperature
                t_span = 1 - torch.cos(torch.linspace(0, 1, n + 1) * 0.5 * torch.pi)
                out = cfm.solve_euler(z, t_span=t_span, mu=mu[None], mask=mask, spks=spk, cond=None, n_steps=n, guidance_scale=s,
                                      fake_speaker=sd["fake_speaker"], fake_content=sd["fake_content"])
    finally:
        torch.randn = orig
    return out[0].numpy()


def main():
    fm = import_reference_cfm()
    cfg = SI.config()
    sd = SI.model(cfg)
    cfm = fm.CFM(in_channels=336, out_channel=80, cfm_params=types.SimpleNamespace(solver="euler", sigma_min=1e-4),
                 decoder_params={}, n_spks=cfg["n_spks"], spk_emb_dim=cfg["spk_emb_dim"])
    est = {k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")}
    missing, unexpected = cfm.load_state_dict(est, strict=True)
    cfm.eval()
    out = {"seed": np.int64(SI.SEED), "cases": np.array([c[0] for c in SI.CASES])}
    for name, lens, n, s, temp, sids in SI.CASES:
        out[name + ".lengths"] = np.array(lens, np.int64)
        out[name + ".sid"] = np.array(sids, np.int64)
        out[name + ".params"] = np.array([n, s, temp], np.float64)
        for b, (T, sid) in enumerate(zip(lens, sids)):
            mu, noise = (torch.from_numpy(a) for a in SI.inputs(name + str(b), T, cfg))
            out["%s.mu%d" % (name, b)], out["%s.noise%d" % (name, b)] = mu.numpy(), noise.numpy()
            out["%s.mel%d" % (name, b)] = reference_mel(cfm, sd, mu, noise, sid, n, s, temp)
    path = os.path.join(ROOT, "tests", "golden", "ref_stabletts_cfm.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
