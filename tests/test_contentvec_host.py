"""ContentVec on the host: the oracle against the reference HubertModel (vc/contentvec.py) and its fixture
(tests/golden/ref_contentvec.npz, oracle/make_golden_contentvec.py), the frame count, the positional conv's weight-norm fold in
both spellings, the configuration refusals, the packed blob and the C entry points."""
import numpy as np
import pytest
import torch

import contentvec_inputs as CI
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from oracle import contentvec_oracle as O
from vosk_tts_b200 import config as C, engine as E, weights

REF = np.load(CI.GOLDEN + "/ref_contentvec.npz")
needs_ref = pytest.mark.skipif(not CI.reference_available(), reason="reference vc/contentvec.py or transformers not present")


@pytest.fixture(scope="module")
def net():
    return CI.build_reference(CI.model())


@pytest.mark.parametrize("n", CI.LENGTHS + (CI.LONG,))
def test_oracle_reproduces_fixture(n):
    x = CI.speech(n, n)
    st = {}
    u = O.contentvec_units(CI.folded(), CI.cv(), x, torch.float32, st).numpy()
    assert u.shape[0] == int(REF["s%d/frames" % n]) == C.contentvec_frames(n)
    err = float(np.abs(u[CI.kept_frames(u.shape[0])] - REF["s%d/units" % n]).max())
    print(n, err)
    assert err < 1e-5
    if n == 16000:
        assert np.abs(st["feat"].numpy() - REF["s16000/feat"]).max() < 1e-5
        assert np.abs(st["enc_in"].numpy() - REF["s16000/enc_in"]).max() < 1e-5


@needs_ref
@pytest.mark.parametrize("make", [CI.speech, CI.dc_offset])
def test_oracle_matches_reference(make, net):
    """fp32 within 1e-5 of the reference; float64 within the fp32 reference's own distance from the reference run in float64
    (which recomputes the weight norm in float64)."""
    x = make(32000, 3)
    with torch.no_grad():
        r32 = net.extract(torch.from_numpy(x)[None])[0].numpy()
        r64 = net.double().extract(torch.from_numpy(x).double()[None])[0].numpy()
        net.float()
    o32 = O.contentvec_units(CI.folded(), CI.cv(), x, torch.float32).numpy()
    o64 = O.contentvec_units(CI.folded(), CI.cv(), x, torch.float64).numpy()
    print(make.__name__, "fp32 %.3g, fp64 %.3g, reference fp32 vs fp64 %.3g" % (np.abs(o32 - r32).max(), np.abs(o64 - r64).max(),
                                                                               np.abs(r32 - r64).max()))
    assert np.abs(o32 - r32).max() < 1e-5
    assert np.abs(o64 - r64).max() <= np.abs(r32 - r64).max()


@needs_ref
def test_frame_count_matches_reference(net):
    n = np.arange(400, 4001)
    ref = net._get_feat_extract_output_lengths(torch.from_numpy(n)).numpy()
    assert [C.contentvec_frames(int(v)) for v in n] == list(ref)
    for v in (160000, 960000):
        assert C.contentvec_frames(v) == int(net._get_feat_extract_output_lengths(torch.tensor(v)))
    assert C.contentvec_frames(399) == 0 and C.contentvec_frames(960000) == 2999 and C.contentvec_frames(160000) == 499


@needs_ref
def test_weight_norm_fold_both_spellings(net):
    eff = net.encoder.pos_conv_embed.conv.weight.detach()
    k = weights.CV_POS + "weight"
    assert torch.equal(weights.fold_contentvec_pos_conv(CI.model())[k], eff)                       # weight_g / weight_v
    sd = {n: t.detach().clone() for n, t in net.state_dict().items()}                              # parametrizations.*
    assert any("original0" in n for n in sd)
    assert torch.equal(weights.fold_contentvec_pos_conv(sd)[k], eff)


def test_weight_norm_fold_is_per_tap():
    """The norm is over dims 0 and 1 for every tap (dim=2), not fold_weight_norm's per output channel."""
    sd = CI.model()
    w = weights.fold_contentvec_pos_conv(sd)[weights.CV_POS + "weight"]
    g = sd[weights.CV_POS + "weight_g"].reshape(-1)
    assert torch.allclose(w.norm(dim=(0, 1)), g, rtol=1e-5)


@pytest.mark.parametrize("key,val,msg", [
    ("feat_extract_norm", "layer", "feat_extract_norm"), ("do_stable_layer_norm", True, "do_stable_layer_norm"),
    ("conv_bias", True, "conv_bias"), ("hidden_act", "relu", "hidden_act"), ("feat_extract_activation", "gelu_new", "gelu"),
    ("conv_stride", [5, 2, 2, 3, 2, 2, 2], "strides"), ("num_attention_heads", 16, "head dim"),
    ("num_conv_pos_embeddings", 127, "even")])
def test_config_refusals(key, val, msg):
    with pytest.raises(ValueError, match=msg):
        C.contentvec_config({key: val})


def test_config_defaults_and_json(tmp_path):
    cv = C.contentvec_config()
    assert (cv["cv_layers"], cv["cv_hidden"], cv["cv_heads"], cv["cv_ffn"], cv["cv_pos_k"], cv["cv_pos_groups"]) == (12, 768, 12, 3072, 128, 16)
    p = tmp_path / "config.json"
    p.write_text('{"num_hidden_layers": 2, "layer_norm_eps": 1e-6, "architectures": ["HubertModel"]}')
    cv = C.contentvec_config(str(p))
    assert cv["cv_layers"] == 2 and cv["cv_ln_eps"] == 1e-6


def test_load_contentvec(tmp_path):
    sd = {"hubert." + k: v for k, v in CI.model().items()}       # some exports prefix the model
    torch.save(sd, tmp_path / "pytorch_model.bin")
    (tmp_path / "config.json").write_text('{"conv_bias": false, "classifier_proj_size": 256}')
    got, cv = weights.load_contentvec(str(tmp_path))
    assert cv == C.contentvec_config()
    assert torch.equal(got[weights.CV_POS + "weight"], CI.folded()[weights.CV_POS + "weight"])
    assert weights.CV_POS + "weight_g" not in got


def test_pack_without_contentvec_unchanged():
    sd = weights.fold_weight_norm(QC.model())
    b0, m0 = weights.pack_quickvc(sd, QI.config())
    b1, m1 = weights.pack_quickvc(sd, QI.config(), contentvec=CI.model())
    assert m1.startswith(m0) and np.array_equal(b1[:b0.size], b0)
    names = [l.split()[0] for l in m1[len(m0):].splitlines()]
    assert names[0] == "cv.c0.w" and all(n.startswith("cv.") for n in names)
    fp32 = 3 + 2 * 6 + 4 + 2 + 2 + 12 * 12
    assert "cv.l11.ln2.b" in names and len(names) == fp32 + 2 + 12 * 4 * 2         # + the split-bf16 copies (.th / .tl)
    assert "cv.l11.ffn2.th" in names and "cv.fp.tl" in names
    b2, m2 = weights.pack_quickvc(sd, QI.config(), precision=0, contentvec=CI.model())
    assert len(m2.splitlines()) - len(weights.pack_quickvc(sd, QI.config(), precision=0)[1].splitlines()) == fp32


def test_pack_layout():
    """Layers 1.. are 1x1 convs over k consecutive rows, tap-major; the positional conv is [half][group][tap][in][out]."""
    sd = CI.folded()
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    ent = {l.split()[0]: (int(l.split()[1]), int(l.split()[2])) for l in man.splitlines()}
    get = lambda n: blob[ent[n][0]:ent[n][0] + ent[n][1]]
    w1 = sd["feature_extractor.conv_layers.1.conv.weight"].numpy()            # [512, 512, 3]
    p1 = get("cv.c1.w").reshape(3 * 512, 512)
    assert np.array_equal(p1[2 * 512 + 7], w1[:, 7, 2])
    pw = sd[weights.CV_POS + "weight"].numpy()                                # [768, 48, 128]
    pp = get("cv.pos.w").reshape(2, 16, 64, 48, 48)
    assert np.array_equal(pp[1, 3, 5, 6], pw[3 * 48:4 * 48, 6, 64 + 5])


def test_abi_exports():
    assert "vtts_content_units" in E.EXPORTS and "vtts_quickvc_convert_wav" in E.EXPORTS
    names = [f[0] for f in E.VttsConfig._fields_]
    assert names[-12:] == ["cv_layers", "cv_hidden", "cv_heads", "cv_ffn", "cv_conv_dim", "cv_n_conv", "cv_conv_kernel",
                           "cv_conv_stride", "cv_pos_k", "cv_pos_groups", "cv_ln_eps", "cv_gn_eps"]
    cfg = dict(QI.config(), contentvec=CI.cv())
    c = E.make_c_config(cfg)
    assert c.cv_n_conv == 7 and list(c.cv_conv_kernel)[:7] == [10, 3, 3, 3, 3, 2, 2] and c.cv_gn_eps == pytest.approx(1e-5)
    assert E.make_c_config(QI.config()).cv_layers == 0


def test_flops_per_frame():
    assert O.flops_per_frame(CI.cv(), 499) / 1e6 == pytest.approx(296.7, abs=0.1)


def test_cli_source_needs_contentvec(tmp_path, capsys):
    from vosk_tts_b200 import quickvc
    with pytest.raises(SystemExit):
        quickvc.main(["--config", "x.json", "--checkpoint", "G.pth", "--source", "a.wav", "--target", "t.wav", "--out-dir", str(tmp_path)])
    with pytest.raises(SystemExit):
        quickvc.main(["--config", "x.json", "--checkpoint", "G.pth", "--source", "a.wav", "--units", "a.npy", "--target", "t.wav",
                      "--out-dir", str(tmp_path)])
