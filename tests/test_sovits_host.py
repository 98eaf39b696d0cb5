"""GPT-SoVITS prompt tokens on the host: the float64 restatement of extract_latent against the reference's own, the s2
checkpoint loader (both layouts) and its refusals, the prompt pad and length limits, and the packed layout."""
import os
import pickle

import numpy as np
import pytest
import torch

import sovits_inputs as SI
from oracle import sovits_oracle as O
from vosk_tts_b200 import config as C, synthetic, weights

GPT_SOVITS = os.path.join(os.environ.get("VTTS_REFERENCE_ROOT", "/root/reference"), "training", "gpt-sovits")


def _s2():
    return synthetic.make_random_sovits(SI.hubert())      # the quick codebook: no HuBERT run


def _reference_available():
    try:
        import einops  # noqa: F401
    except Exception:
        return False
    return os.path.isfile(os.path.join(GPT_SOVITS, "module", "models.py"))


@pytest.mark.skipif(not _reference_available(), reason="the reference tree is not present")
def test_restatement_equals_reference_extract_latent():
    from oracle.make_golden_sovits import reference_synthesizer
    sd = _s2()
    net = reference_synthesizer(GPT_SOVITS, sd)
    for name in ("f_odd", "f_even"):
        x = SI.feats(name)
        with torch.no_grad():
            ref = net.extract_latent(torch.from_numpy(x).double().T[None])
        assert tuple(ref.shape) == (1, 1, x.shape[0] // 2)
        codes, margin, _ = O.extract_latent(x, sd)
        assert np.array_equal(codes, ref[0, 0].numpy()) and margin.min() > 0


class HParams:
    """Stands in for GPT-SoVITS's utils.HParams, pickled beside `weight` in its exports."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _save(tmp_path, obj, name):
    path = str(tmp_path / name)
    torch.save(obj, path)
    return path


def test_both_layouts_load(tmp_path):
    sd = _s2()
    full = dict(sd, **{"enc_p.proj.weight": torch.zeros(3), "quantizer.vq.layers.0._codebook.cluster_size": torch.zeros(1024)})
    a = _save(tmp_path, {"model": full, "iteration": 3, "optimizer": None, "learning_rate": 1e-4}, "G_3.pth")
    b = _save(tmp_path, {"weight": {k: v.half() for k, v in full.items()}, "config": HParams(data=HParams(sampling_rate=32000)),
                         "info": "e8"}, "s2G488k.pth")
    for path in (a, b):
        got, cfg = weights.load_sovits(path, SI.S2_24K)
        assert set(got) == {"ssl_proj.weight", "ssl_proj.bias", "quantizer.vq.layers.0._codebook.embed",
                            "quantizer.vq.layers.0._codebook.inited"}
        assert all(v.dtype == torch.float32 for v in got.values())
        assert cfg["model_family"] == "sovits" and cfg["sv_codebook"] == 1024 and cfg["cv_hidden"] == 768
        assert cfg["sampling_rate"] == 24000 and cfg["sovits_pad"] == 7200          # from the config, not the pickled object
    tol = dict(rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(weights.load_sovits(b, SI.S2_32K)[0]["ssl_proj.weight"], sd["ssl_proj.weight"], **tol)


def test_refusals(tmp_path):
    cfg = SI.cfg()
    sd = _s2()
    bad = dict(sd, **{"ssl_proj.weight": torch.zeros(768, 768, 1)})
    with pytest.raises(ValueError, match="50 Hz"):
        weights.pack_sovits(bad, cfg, SI.hubert())
    bad = dict(sd, **{"quantizer.vq.layers.0._codebook.embed": torch.zeros(1024, 512)})
    with pytest.raises(ValueError, match=r"expected \[K, 768\]"):
        weights.pack_sovits(bad, cfg, SI.hubert())
    bad = dict(sd, **{"quantizer.vq.layers.0._codebook.inited": torch.zeros(1)})
    with pytest.raises(ValueError, match="never initialised"):
        weights.pack_sovits(bad, cfg, SI.hubert())
    with pytest.raises(ValueError, match="neither"):
        weights.load_sovits(_save(tmp_path, {"state_dict": sd}, "x.pth"), SI.S2_32K)
    with pytest.raises(ValueError, match="has no tensor"):
        weights.load_sovits(_save(tmp_path, {"weight": {"ssl_proj.weight": sd["ssl_proj.weight"]}}, "y.pth"), SI.S2_32K)
    with pytest.raises(ValueError, match="sampling_rate"):
        C.sovits_config({"model": {}})
    with pytest.raises(ValueError, match="conv_bias"):
        C.sovits_config(SI.S2_32K, {"conv_bias": True})


def test_loader_runs_nothing_the_file_names(tmp_path):
    class Boom:
        def __reduce__(self):
            return (os.system, ("exit 3",))
    path = str(tmp_path / "evil.pth")
    torch.save({"weight": _s2(), "config": Boom()}, path, pickle_protocol=pickle.HIGHEST_PROTOCOL)
    assert weights.load_sovits(path, SI.S2_32K)[1]["sv_codebook"] == 1024


def test_pad_and_limits():
    assert C.sovits_pad(32000) == 9600 and C.sovits_pad(24000) == 7200 and C.sovits_pad(48000) == 14400
    assert (C.SOVITS_PROMPT_MIN, C.SOVITS_PROMPT_MAX) == (48000, 320000)
    assert C.SOVITS_PROMPT_MESSAGE == "Prompt audio length must be longer than 3 seconds and shorter than 20 seconds!"
    f = np.load(SI.FIXTURE)
    for name in SI.WAVE:
        assert int(f[name + "/samples"]) == SI.padded(name).size
        assert int(f[name + "/frames"]) == C.contentvec_frames(SI.padded(name).size)
        assert f[name + "/codes"].size == int(f[name + "/frames"]) // 2
    assert [int(f[n + "/frames"]) for n in ("w48000", "w48320", "w10s", "w20s")] == [179, 180, 529, 1029]


def test_pack_layout():
    sd = _s2()
    cfg = SI.cfg()
    blob, man = weights.pack_sovits(sd, cfg, SI.hubert(), tc=False)
    ent = {n: (int(o), int(c)) for n, o, c in (line.split() for line in man.strip().splitlines())}
    get = lambda n: blob[ent[n][0]:ent[n][0] + ent[n][1]]
    assert "cv.c0.w" in ent and "cv.fp.th" not in ent
    w, b = sd["ssl_proj.weight"].numpy(), sd["ssl_proj.bias"].numpy()
    pw = get("sv.proj.w").reshape(1, 2 * 768, 768)          # [k][Cin][ldw]: input channel j < 768 is tap 0, else tap 1
    assert np.array_equal(pw[0, :768], w[:, :, 0].T) and np.array_equal(pw[0, 768:], w[:, :, 1].T)
    assert np.array_equal(get("sv.proj.b"), b)
    E = sd["quantizer.vq.layers.0._codebook.embed"].numpy().astype(np.float64)
    assert np.array_equal(get("sv.score.w").reshape(768, 1024), (2 * E).T.astype(np.float32))
    np.testing.assert_array_equal(get("sv.score.b"), (-(E * E).sum(1)).astype(np.float32))
    # argmax of x.2E - |E|^2 is the argmax of -|x - E|^2
    x = SI.feats("f_even")
    p = O.project(x, w, b)
    s = p @ (2 * E).T - (E * E).sum(1)
    assert np.array_equal(s.argmax(1), O.extract_latent(x, sd)[0])
