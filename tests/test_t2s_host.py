"""GPT-SoVITS text-to-semantic decoding on the host: checkpoint loading (both layouts), the config derivation and its refusals,
the packed blob, and the float64 restatement oracle/t2s_oracle.py against the reference's infer_panel and sample where the
reference tree is present."""
import os
import numpy as np
import pytest
import torch

import t2s_inputs as TI
from oracle import t2s_oracle as O
from vosk_tts_b200 import config, weights

REF = "/root/reference/training/gpt-sovits"


def test_config_refusals():
    for k, v, msg in (("embedding_dim", 32, "embedding_dim"), ("EOS", 10, "EOS"), ("head", 3, "head widths"),
                      ("vocab_size", 5000, "block sort")):
        block = dict(TI.SMALL)
        block[k] = v
        if k == "vocab_size":
            block["EOS"] = v - 1
        with pytest.raises(ValueError, match=msg):
            config.t2s_config(block)


def test_both_checkpoint_layouts(tmp_path):
    sd, cfg = TI.model()
    conf = {"model": dict(TI.SMALL)}
    p1 = tmp_path / "lightning.ckpt"
    torch.save({"state_dict": {"model." + k: v for k, v in sd.items()}, "hyper_parameters": {"config": conf}}, p1)
    p2 = tmp_path / "half.ckpt"
    torch.save({"weight": {k: v.half() for k, v in sd.items()}, "config": conf}, p2)
    for p, tol in ((p1, 0.0), (p2, 1e-2)):
        sd2, cfg2 = weights.load_t2s(str(p))
        assert cfg2 == cfg
        assert max(float((sd2[k] - sd[k]).abs().max()) for k in sd) <= tol
    bad = dict(sd)
    bad.pop("h.layers.1.self_attn.in_proj_weight")
    with pytest.raises(ValueError):
        config.t2s_config(TI.SMALL, bad)


def test_pack_sine_table():
    sd, cfg = TI.model()
    blob, man = weights.pack_t2s(sd, cfg)
    ent = {l.split()[0]: (int(l.split()[1]), int(l.split()[2])) for l in man.splitlines()}
    o, n = ent["t2s.pe"]
    pe = blob[o:o + n].reshape(-1, cfg["cv_hidden"])
    assert pe.shape[0] == config.T2S_MAX_POSITIONS
    assert np.array_equal(pe, O.sine_table(pe.shape[0], cfg["cv_hidden"], torch.float32).numpy())
    assert "t2s.l1.ffn2.th" in ent and "t2s.pred.w" in ent


@pytest.fixture
def reference():
    """The reference's Text2SemanticDecoder and ar.models.utils, imported under the generator's scoped shims."""
    if not os.path.isdir(REF):
        pytest.skip("the reference tree is not present")
    from oracle import make_golden_t2s as G
    with G.reference(REF) as mods:
        yield mods


def test_fixture_matches_oracle():
    """The stored reference run equals the float64 restatement on every case (and the generator's seeded weights)."""
    from oracle import make_golden_t2s as G
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_t2s.npz"))
    for name in G.CASES:
        if name in ("cap_1500", "upstream_width"):
            continue                            # (1500 or 24-layer uncached passes: minutes on the CPU)
        sd, cfg, ph, pr, bert, q, es = G.case_inputs(name, gold[name + ".qseed"])
        assert G.sd_sha1(sd) == str(gold[name + ".sha1"])
        y, idx, _, _ = O.decode(sd, cfg, ph, pr, bert, q, early_stop=es)
        assert np.array_equal(y, gold[name + ".y"]) and idx == int(gold[name + ".idx"]), name


@pytest.mark.parametrize("case", [(12, 0, 1.6, 60, -1), (9, 7, 1.6, 60, -1), (10, 5, 0.0, 30, 20)])
def test_oracle_matches_reference_infer_panel(case, monkeypatch, reference):
    Dec, _ = reference
    T, P, eos, cap, es = case
    sd, cfg = TI.model(eos_scale=eos)
    m = Dec({"model": dict(TI.SMALL)}).eval()
    m.load_state_dict(sd)
    m = m.double()
    ph, pr = TI.phones(cfg, T, T), (TI.prompt(cfg, P, P, repeat=True) if P else None)
    q = TI.q_draws(cfg, 1500, 3)
    it = iter(range(1500))

    def exp_(self, lambd=1.0):
        i = next(it)
        return self.copy_(torch.from_numpy(q[i][:self.shape[-1]].astype(np.float64)).reshape(self.shape))
    monkeypatch.setattr(torch.Tensor, "exponential_", exp_)
    with torch.no_grad():
        y, idx = m.infer_panel(torch.from_numpy(ph)[None], torch.tensor([T]), None if pr is None else torch.from_numpy(pr)[None],
                               torch.zeros(1, 1024, T, dtype=torch.float64), top_k=20, top_p=0.6, early_stop_num=es, temperature=0.6)
    oy, oidx, _, _ = O.decode(sd, cfg, ph, pr, None, q, early_stop=es)
    assert np.array_equal(y[0].numpy(), oy) and idx == oidx


def test_sampler_matches_reference(reference):
    _, U = reference
    r = np.random.default_rng(0)
    for trial in range(40):
        V = int(r.integers(2, 80))
        l = torch.from_numpy(r.standard_normal(V) * 3)
        if trial % 4 == 1:
            l[r.integers(0, V, 3)] = float("-inf")
            l[0] = 1.0
        if trial % 4 == 2:
            l = torch.round(l)                            # ties
        prev = torch.from_numpy(r.integers(0, V, int(r.integers(0, 6))))
        q = r.exponential(1.0, V)
        k = int(r.integers(1, 25))
        tp = float(r.choice([0.6, 0.9, 1.0]))
        ref_l = l.clone()
        torch.manual_seed(0)
        orig = torch.Tensor.exponential_
        torch.Tensor.exponential_ = lambda self, lambd=1.0: self.copy_(torch.from_numpy(q).reshape(self.shape))
        try:
            tok, _ = U.sample(ref_l, prev[None] if prev.numel() else prev, top_k=k, top_p=tp, repetition_penalty=1.35, temperature=0.6)
        finally:
            torch.Tensor.exponential_ = orig
        otok, pa, _ = O.sample(l, prev.numpy(), k, tp, 0.6, 1.35, q)
        assert int(tok) == otok, trial
        assert pa == int(torch.argmax(ref_l))
