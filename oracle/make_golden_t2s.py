"""Writes tests/golden/ref_t2s.npz: the reference's own Text2SemanticDecoder.infer_panel (training/gpt-sovits/ar/models/
t2s_model.py:324-448), unmodified, run in float64 on the CPU on seeded models (tests/t2s_inputs.py; each state dict's SHA-1 is
stored so that a test can check it regenerates the same weights).

Three shims, none of which edits the reference: a stub torchmetrics.classification.MulticlassAccuracy (t2s_model.py imports
it; the package is not needed to infer), Tuple / Optional / Tensor made visible to patched_mha_with_cache.py for the duration
of the import (it expects them from torch.nn.functional's star import), and Tensor.exponential_ drawing the rows of a seeded
numpy stream (t2s_inputs.q_draws), one row per sampling step, so that a test can regenerate every q.

Per case: the inputs, y[:, :-1] and idx, and per sampling step the margins that decide it, from the reference's own logits
(captured by a forward hook on ar_predict_layer): the logit gap at the top-k pivot, |cum - top_p| nearest the top-p cut, the
winner's probs / q against the runner-up's (in logit units) and the gap between EOS and the largest other penalised logit;
plus which stop rule ended the loop.

    python oracle/make_golden_t2s.py /path/to/training/gpt-sovits
"""
import builtins
import contextlib
import hashlib
import os
import sys
import types
import typing

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import t2s_inputs as TI                     # noqa: E402
from oracle import t2s_oracle as O          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_t2s.npz")
FLOOR = 1e-3        # least margin of every step of a case (logit units; probability for the top-p cut)
# At the upstream width the 1025 probabilities are small enough that some step's cumulative sum always passes within 1e-3 of
# top_p; 1e-4 is still 10x the fp32 engine's measured logit error there.
FLOOR_UPSTREAM = 1e-4

# name: (model block, model seed, eos_scale, eos_logit (t2s_inputs.model), phones, (prompt length, repeating tokens?), bert?,
#        q seed, q's EOS column forced high?, early_stop_num, the stop rule the case exists for)
CASES = {
    "sampled_eos": ("SMALL", 5, 1.0, 1.0, 12, (0, False), False, 41, False, -1, "sampled"),
    "argmax_eos": ("SMALL", 5, 1.0, 1.0, 12, (0, False), False, 42, True, -1, "argmax"),
    "prompt_repeat": ("SMALL", 5, 1.6, None, 9, (15, True), False, 43, False, 59, "early"),
    "prompt_bert": ("SMALL", 5, 1.6, None, 16, (7, False), True, 44, False, 59, "early"),
    "early_stop": ("SMALL", 5, 0.0, None, 10, (4, False), False, 45, False, 25, "early"),
    "cap_1500": ("SMALL", 5, 0.0, None, 8, (0, False), False, 46, False, -1, "cap"),
    "upstream_width": ("UPSTREAM", 7, 1.0, None, 40, (20, False), True, 47, False, 49, "early"),
}


def sd_sha1(sd):
    h = hashlib.sha1()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(np.ascontiguousarray(sd[k].float().numpy()).tobytes())
    return h.hexdigest()


def case_inputs(name, qseed=None):
    """qseed: the candidate's seed (the fixture stores the one it was made with; it also picks the phones), or CASES'
    first candidate."""
    block, mseed, eos, eos_logit, T, (P, rep), with_bert, qseed0, q_eos, es, _ = CASES[name]
    qseed = qseed0 if qseed is None else int(qseed)
    sd, cfg = TI.model(getattr(TI, block), seed=mseed, eos_scale=eos, eos_logit=eos_logit)
    ph = TI.phones(cfg, T, 100 + T + qseed - qseed0)        # each candidate stream also draws its own phones
    pr = TI.prompt(cfg, P, 200 + P, repeat=rep) if P else None
    bert = np.random.default_rng(300 + T).standard_normal((T, 1024)).astype(np.float32) * 0.3 if with_bert else None
    q = TI.q_draws(cfg, 1500, qseed)
    if q_eos:
        q[:, -1] = 1e6                      # EOS is never the sample: only the penalised argmax can stop the loop
    return sd, cfg, ph, pr, bert, q, es


@contextlib.contextmanager
def reference(path):
    tm, cl = types.ModuleType("torchmetrics"), types.ModuleType("torchmetrics.classification")
    cl.MulticlassAccuracy = type("MulticlassAccuracy", (), {"__init__": lambda self, *a, **k: None})
    tm.classification = cl
    added = [n for n in ("Tuple", "Optional", "Tensor") if not hasattr(builtins, n)]
    saved = {k: sys.modules.get(k) for k in ("torchmetrics", "torchmetrics.classification")}
    sys.modules["torchmetrics"], sys.modules["torchmetrics.classification"] = tm, cl
    for n in added:
        setattr(builtins, n, torch.Tensor if n == "Tensor" else getattr(typing, n))
    sys.path.insert(0, path)
    try:
        from ar.models.t2s_model import Text2SemanticDecoder
        from ar.models import utils as U
        yield Text2SemanticDecoder, U
    finally:
        sys.path.remove(path)
        for n in added:
            delattr(builtins, n)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def run_reference(Dec, sd, cfg, block, ph, pr, bert, q, es):
    m = Dec({"model": dict(block)}).eval()
    m.load_state_dict(sd)
    m = m.double()
    logits = []
    m.ar_predict_layer.register_forward_hook(lambda mod, inp, out: logits.append(out[0].detach().clone()))
    it = iter(range(len(q)))
    orig = torch.Tensor.exponential_

    def exp_(self, lambd=1.0):
        return self.copy_(torch.from_numpy(q[next(it)][:self.shape[-1]].astype(np.float64)).reshape(self.shape))
    torch.Tensor.exponential_ = exp_
    try:
        T = len(ph)
        bf = torch.zeros(1, 1024, T, dtype=torch.float64) if bert is None else torch.from_numpy(bert.T.astype(np.float64))[None]
        with torch.no_grad():
            y, idx = m.infer_panel(torch.from_numpy(ph)[None], torch.tensor([T]), None if pr is None else torch.from_numpy(pr)[None],
                                   bf, top_k=20, top_p=0.6, early_stop_num=es, temperature=0.6)
    finally:
        torch.Tensor.exponential_ = orig
    return y[0].numpy().astype(np.int64), int(idx), logits


def margins(logits, y, P, q, V):
    """Per step the four margins of oracle.t2s_oracle.sample, the penalised argmax and the sample, on the reference's logits."""
    out, pa, tk = [], [], []
    y = list(y) + [-1]
    for i, lg in enumerate(logits):
        l = lg[:-1] if i == 0 else lg
        tok, a, mg = O.sample(l.clone(), np.array(y[:P + i], np.int64), 20, 0.6, 0.6, 1.35, q[i][:l.numel()], eos=V - 1)
        out.append(mg)
        pa.append(a)
        tk.append(tok)
    return np.array(out, np.float64), np.array(pa), np.array(tk)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/training/gpt-sovits"
    data = {}
    with reference(path) as (Dec, _):
        for name, spec in CASES.items():
            # the first q stream (from the case's seed on) whose every step is decided by at least FLOOR, so that the
            # fixture is compared on all its steps; the 1500-step case takes its first stream and is compared up to its
            # first close step
            for qseed in range(spec[7], spec[7] + 200):
                sd, cfg, ph, pr, bert, q, es = case_inputs(name, qseed)
                y, idx, logits = run_reference(Dec, sd, cfg, getattr(TI, spec[0]), ph, pr, bert, q, es)
                V, P = cfg["t2s_vocab"], 0 if pr is None else len(pr)
                mg, pa, tk = margins(logits, y, P, q, V)
                n = len(logits)
                stop = ("early" if es != -1 and n > es else "argmax" if pa[-1] == V - 1 and tk[-1] != V - 1 else
                        "sampled" if tk[-1] == V - 1 and pa[-1] != V - 1 else "both" if tk[-1] == V - 1 else "cap")
                floor = FLOOR_UPSTREAM if spec[0] == "UPSTREAM" else FLOOR
                if stop == spec[10] and (name == "cap_1500" or mg.min() >= floor):
                    break
            data[name + ".qseed"] = np.int64(qseed)
            assert np.array_equal(tk[:-1], y[P:]), name            # the restated sampler reproduces every kept sample
            assert stop == spec[10] and (name == "cap_1500" or mg.min() >= floor), (name, stop, mg.min())
            print("%-15s T %3d P %3d: %4d steps, idx %4d, stop %-7s, min margins %s" % (name, len(ph), P, n, idx, stop, mg.min(0)))
            data[name + ".y"] = y
            data[name + ".idx"] = np.int64(idx)
            data[name + ".margins"] = mg.astype(np.float32)
            data[name + ".stop"] = np.array(stop)
            data[name + ".sha1"] = np.array(sd_sha1(sd))
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
