"""Host-side tests of the StableTTS flow-matching decoder: the oracle restatement against the reference's stored mel, the
weight packing, the config rejections and (when a CUDA device is absent these still run) the argument checks that need no
engine."""
import numpy as np
import pytest
import torch

import stabletts_cfm_inputs as SI
from oracle import stabletts_cfm_oracle as so
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import MODEL_FAMILIES, VttsConfig, make_c_config


@pytest.fixture(scope="module")
def golden():
    return np.load(SI.GOLDEN)


@pytest.fixture(scope="module")
def model():
    cfg = SI.config()
    return cfg, SI.model(cfg)


def test_fixture_holds_the_seeded_inputs(golden):
    assert int(golden["seed"]) == SI.SEED and list(golden["cases"]) == [c[0] for c in SI.CASES]
    for case in SI.CASES:
        for b, (mu, nz) in enumerate(SI.case_inputs(case)):
            assert np.array_equal(golden["%s.mu%d" % (case[0], b)], mu) and np.array_equal(golden["%s.noise%d" % (case[0], b)], nz)


@pytest.mark.parametrize("case", [c for c in SI.CASES if max(c[1]) <= 65], ids=lambda c: c[0])
def test_oracle_equals_reference(case, golden, model):
    """fp32 evaluation within 2e-5 of the reference's fp32 mel (|mel| reaches 10, and the fp32 sums' order depends on the
    host's thread count: 8.5e-6 measured at most, on the single-step case, whose dt = 1 damps nothing); the float64
    evaluation (what the GPU tests compare against) within the fp32 rounding the reference itself carries."""
    cfg, sd = model
    name, lens, n, s, temp, sids = case
    for b, (mu, nz) in enumerate(SI.case_inputs(case)):
        ref = golden["%s.mel%d" % (name, b)]
        assert ref.shape == (cfg["noise_channels"], lens[b])
        o32 = so.decode(sd, cfg, mu, sids[b], nz, n, temp, s, torch.float32)
        assert np.abs(o32 - ref).max() < 2e-5
        o64 = so.decode(sd, cfg, mu, sids[b], nz, n, temp, s, torch.float64)
        assert np.abs(o64 - ref).max() < 5e-5


def test_time_schedule_is_the_reference_loop():
    ts, dts = so.t_schedule(10)
    span = (1 - torch.cos(torch.linspace(0, 1, 11) * 0.5 * torch.pi)).numpy()
    assert ts[0] == 0 and dts[0] == span[1] and ts.dtype == np.float32
    assert abs(float(ts[-1]) + float(dts[-1]) - 1.0) < 1e-6
    assert np.allclose(ts, span[:-1], atol=1e-6)


def test_guidance_zero_is_the_conditional_branch(model):
    cfg, sd = model
    mu, nz = SI.inputs("g0", 9)
    a = so.decode(sd, cfg, mu, 1, nz, 2, 1.0, 0.0)
    sd2 = dict(sd)
    sd2["fake_content"] = sd["fake_content"] + 1.0
    assert np.array_equal(a, so.decode(sd2, cfg, mu, 1, nz, 2, 1.0, 0.0))
    assert not np.array_equal(so.decode(sd, cfg, mu, 1, nz, 2, 1.0, 0.5), so.decode(sd2, cfg, mu, 1, nz, 2, 1.0, 0.5))


def _tensors(blob, man):
    out = {}
    for line in man.strip().split("\n"):
        name, off, n = line.split()
        out[name] = blob[int(off):int(off) + int(n)]
    return out


def test_packing_round_trips(model):
    cfg, sd = model
    blob, man = weights.pack_stabletts_cfm(sd, cfg)
    t = _tensors(blob, man)
    H, F, NL, G = cfg["hidden_channels"], cfg["filter_channels"], cfg["n_layers"], cfg["spk_emb_dim"]
    e = "decoder.estimator."
    w = sd[e + "blocks.2.block.mlp.conv_1.weight"].numpy()               # [F, H, 3] -> [k][Cin][Cout]
    assert np.array_equal(t["st.l2.ffn1.w"].reshape(3, H, F), np.transpose(w, (2, 1, 0)))
    q = t["st.l1.qkv.w"].reshape(1, H, 3 * H)[0]
    for i, n in enumerate("qkv"):
        assert np.array_equal(q[:, i * H:(i + 1) * H], sd[e + "blocks.1.block.attn.conv_%s.weight" % n].numpy()[:, :, 0].T)
    assert np.array_equal(t["st.ada.w2"].reshape(NL, 6 * H, H)[5], sd[e + "blocks.5.block.adaLN_modulation.2.weight"].numpy())
    assert np.array_equal(t["st.film.w"].reshape(NL, 2 * H, H)[3], sd[e + "blocks.3.time_fusion.film.weight"].numpy()[:, :, 0])
    assert np.array_equal(t["st.lsc2.w"].reshape(3, 2 * H, H), np.transpose(sd[e + "lsc_layers.2.weight"].numpy(), (2, 1, 0)))
    assert np.array_equal(t["st.spk_emb"].reshape(-1, G), sd["spk_emb.weight"].numpy())
    assert t["st.fake_content"].shape == (cfg["cond_channels"],) and float(t["st.mel_std"][0]) == float(sd["mel_std"])
    assert all(int(line.split()[1]) % 64 == 0 for line in man.strip().split("\n"))
    bad = dict(sd)
    bad[e + "in_proj.weight"] = sd[e + "in_proj.weight"][:, :-1]
    with pytest.raises(ValueError, match="in_proj.weight has shape"):
        weights.pack_stabletts_cfm(bad, cfg)


def test_synthetic_checkpoint_has_live_gates(model):
    cfg, sd = model
    w = sd["decoder.estimator.blocks.0.block.adaLN_modulation.2.weight"]
    assert float(w.abs().max()) > 0, "a zero last adaLN linear makes every block the identity"
    again = synthetic.make_random_stabletts_cfm(cfg, SI.SEED)
    assert all(torch.equal(sd[k], again[k]) for k in sd)


@pytest.mark.parametrize("override, reason", [
    ({"use_lsc": False}, "use_lsc=false is not supported"),
    ({"n_layers": 5}, "n_layers must be even"),
    ({"n_heads": 5}, "head width"),
    ({"n_heads": 8}, "head width"),
    ({"solver": "heun"}, "only the fixed-step Euler solver"),
    ({"kernel_size": 4}, "kernel_size must be odd"),
    ({"hidden_channels": 640, "n_heads": 5}, "channel widths"),
    ({"n_spks": 0}, "n_spks must be >= 1"),
])
def test_config_rejections_carry_their_reason(override, reason):
    with pytest.raises(ValueError, match=reason):
        C.stabletts_cfm_config(override)


def test_c_config_of_the_family():
    c = make_c_config(SI.config(), precision=1)
    assert isinstance(c, VttsConfig) and c.model_family == MODEL_FAMILIES["stabletts"] == 2 and c.precision == 1
    assert (c.st_noise, c.st_cond, c.st_hidden, c.st_filter, c.st_layers, c.st_heads, c.st_kernel, c.st_spk_dim, c.st_n_spks) == \
        (80, 256, 384, 768, 6, 4, 3, 128, 2)
    assert c.hidden_channels == 0 and c.cv_layers == 0
