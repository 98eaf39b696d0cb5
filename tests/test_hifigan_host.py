"""CPU tests of the StableTTS vocoder's host side: its config, the packed layout the engine binds, the polyphase split of its
ConvTranspose1d, the weight-norm fold against the reference's remove_weight_norm, the oracle against the reference's
waveforms (tests/golden/ref_hifigan.npz), and the argument checks of the bindings."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import hifigan_inputs as HI
from oracle import hifigan_oracle as O
from vosk_tts_b200 import config, engine, weights


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(HI.GOLDEN))


@pytest.fixture(scope="module")
def sd():
    return HI.folded()


def test_config_v1_and_refusals():
    h = config.hifigan_config()
    assert h["upsample_rates"] == [8, 8, 2, 2] and h["upsample_initial_channel"] == 512 and config.hop_samples(h) == 256
    assert config.hifigan_config({"upsample_rates": [4, 4, 4, 4], "upsample_kernel_sizes": [8, 8, 8, 8], "sampling_rate": 1})["upsample_rates"] == [4, 4, 4, 4]
    for bad in ({"upsample_kernel_sizes": [15, 16, 4, 4]}, {"resblock_kernel_sizes": [3, 7, 11, 13],
                                                            "resblock_dilation_sizes": [[1]] * 4}, {"upsample_initial_channel": 200},
                {"resblock_kernel_sizes": [4, 7, 11]}, {"num_mels": 81}):
        with pytest.raises(ValueError):
            config.hifigan_config(bad)


def test_c_config_and_packing(sd):
    h = HI.config()
    cfg = dict(config.stabletts_cfm_config(), vocoder=h)
    c = engine.make_c_config(cfg, precision=1)
    assert (c.decoder_type, c.inter_channels, c.st_noise, c.n_upsamples, c.upsample_initial_channel) == (1, 80, 80, 4, 512)
    assert list(c.upsample_rates[:4]) == [8, 8, 2, 2] and list(c.upsample_kernel_sizes[:4]) == [16, 16, 4, 4]
    assert (c.resblock_type, c.n_resblock_kernels, c.n_resblock_dilations) == (1, 3, 3)
    assert engine.make_c_config(config.stabletts_cfm_config()).decoder_type == 0      # no vocoder: the fields stay 0
    blob, man = weights.pack_hifigan(sd, h)
    ent = {l.split()[0]: (int(l.split()[1]), int(l.split()[2])) for l in man.splitlines()}
    assert ent["dec.pre.w"][1] == 7 * 80 * 512 and "dec.pre.th" not in ent          # conv_pre: 80 inputs, FFMA only
    assert ent["dec.post.w"][1] == 7 * 32 * 4 and ent["dec.post.b"][1] == 4
    for i, (u, ci) in enumerate(zip([8, 8, 2, 2], [512, 256, 128, 64])):
        for r in range(u):
            assert "dec.up%d.p%d.th" % (i, r) in ent and "dec.up%d.p%d.w" % (i, r) in ent
    assert "dec.rb0.c1.0.th" in ent and "dec.rb8.c2.2.th" in ent and "dec.rb9.c1.0.th" not in ent and "dec.rb11.c2.2.w" in ent
    off, n = ent["dec.rb3.c1.1.w"]
    w = sd["resblocks.3.convs1.1.weight"].numpy()                          # [Co, Ci, k] -> [k][Ci][ldw]
    assert np.array_equal(blob[off:off + n].reshape(3, 128, 128), np.transpose(w, (2, 1, 0)))
    sdb = dict(HI.checkpoint(), **{"conv_pre.weight_v": torch.zeros(1)})
    with pytest.raises((ValueError, RuntimeError)):
        weights.pack_hifigan(weights.fold_weight_norm(sdb), h)


@pytest.mark.parametrize("u,K", [(8, 16), (2, 4), (4, 8), (3, 7)])
def test_polyphase_phases_match_conv_transpose(u, K):
    g = torch.Generator().manual_seed(u * 31 + K)
    ci, co, T = 5, 3, 11
    x = torch.randn(1, ci, T, generator=g, dtype=torch.float64)
    w = torch.randn(ci, co, K, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, w, stride=u, padding=(K - u) // 2)
    out = torch.zeros(1, co, u * T, dtype=torch.float64)
    for r, (pad, js) in enumerate(weights.convt_phases(u, K, (K - u) // 2)):
        wr = torch.stack([w[:, :, j] for j in js], -1).permute(1, 0, 2)
        out[:, :, r::u] = F.conv1d(F.pad(x, (pad, len(js) - 1 - pad)), wr)
    n = min(ref.shape[-1], u * T)
    assert torch.allclose(out[..., :n], ref[..., :n], atol=1e-12)


def test_weight_norm_fold_matches_reference(golden, sd):
    assert str(golden["sha1_checkpoint"]) == HI.sha1_state(HI.checkpoint())
    for k in ("conv_post.weight", "ups.3.weight"):
        np.testing.assert_allclose(sd[k].numpy(), golden["folded." + k], rtol=2e-6, atol=1e-9)


@pytest.mark.parametrize("case", HI.CASES, ids=lambda c: c[0])
def test_oracle_matches_reference(golden, sd, case):
    for b, m in enumerate(HI.case_mels(case)):
        assert np.array_equal(m, golden["%s.mel%d" % (case[0], b)])
        ref = golden["%s.wav%d" % (case[0], b)]
        y32 = O.generator(sd, HI.config(), m, torch.float32).numpy()
        y64 = O.generator(sd, HI.config(), m, torch.float64).numpy()
        assert ref.shape == (256 * m.shape[1],) and 0.1 < np.abs(ref).max() < 0.99
        assert np.abs(y32 - ref).max() < 1e-5
        assert np.abs(y64 - ref).max() < 1e-5


class _FakeLib:
    def __getattr__(self, name):
        raise AssertionError("the library must not be called")


def test_binding_argument_checks():
    e = engine.Engine.__new__(engine.Engine)
    e.cfg, e.lib, e.h = dict(config.stabletts_cfm_config()), _FakeLib(), None
    with pytest.raises(ValueError, match="no vocoder"):
        e.hifigan_vocode(np.zeros((4, 80), np.float32))
    e.cfg["vocoder"] = HI.config()
    with pytest.raises(ValueError, match="frame-major"):
        e.hifigan_vocode(np.zeros((4, 81), np.float32))
