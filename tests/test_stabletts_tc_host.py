"""CPU tests of precision mode 2's StableTTS packing: the split-bf16 copies of the decoder convs the tensor cores take, the
pipe of each conv, and blobs of the other modes left as they were."""
import hashlib

import numpy as np
import pytest

import stabletts_cfm_inputs as SI
import stabletts_inputs as TI
from vosk_tts_b200 import config as C, weights

# SHA-1 of (blob bytes + manifest) as packed before precision mode 2 existed, for the seeded decoder-only and text models
SHA1 = {"cfm": "b2400ab9b39df4c38a6c23d32f82c063e4053708", "text": "af39c71258240a12ecbb3edd0f140417eb681248"}


def sha1(packed):
    blob, man = packed
    return hashlib.sha1(np.ascontiguousarray(blob).tobytes() + man.encode()).hexdigest()


def tensors(packed):
    blob, man = packed
    out = {}
    it = iter(man.split())
    for name, off, n in zip(it, it, it):
        out[name] = blob[int(off):int(off) + int(n)]
    return out


@pytest.fixture(scope="module")
def cfm():
    cfg = SI.config()
    return cfg, SI.model(cfg)


def conv_weight(sd, cfg, name):
    """[Co, Ci, k] of a decoder conv, from the state dict"""
    e = "decoder.estimator."
    if name.startswith("st.cp"):
        return sd[e + "cond_proj.%d.weight" % (2 * int(name[5:]))].numpy()
    if name.startswith("st.lsc"):
        return sd[e + "lsc_layers.%d.weight" % int(name[6:])].numpy()
    l, kind = name[4:].split(".")
    b = e + "blocks.%s.block." % l
    if kind == "qkv":
        return np.concatenate([sd[b + "attn.conv_%s.weight" % n].numpy() for n in "qkv"], 0)
    if kind == "o":
        return sd[b + "attn.conv_o.weight"].numpy()
    return sd[b + "mlp.conv_%d.weight" % (1 if kind == "ffn1" else 2)].numpy()


@pytest.mark.parametrize("precision", [None, 0, 1, 3])
def test_other_modes_pack_the_blob_they_packed_before(cfm, precision):
    cfg, sd = cfm
    kw = {} if precision is None else {"precision": precision}
    assert sha1(weights.pack_stabletts_cfm(sd, cfg, **kw)) == SHA1["cfm"]
    tcfg = TI.config()
    assert sha1(weights.pack_stabletts(TI.model(tcfg), tcfg, **kw)) == SHA1["text"]


def test_mode2_planes_reconstruct_each_weight(cfm):
    cfg, sd = cfm
    t1, t2 = tensors(weights.pack_stabletts_cfm(sd, cfg, precision=1)), tensors(weights.pack_stabletts_cfm(sd, cfg, precision=2))
    names = weights.stabletts_tc_convs(cfg)
    assert set(t2) - set(t1) == {n + s for n in names for s in (".th", ".tl")}
    for n in t1:                                   # every fp32 tensor as before
        assert np.array_equal(t1[n], t2[n]), n
    for n in names:
        w = conv_weight(sd, cfg, n)
        co, ci, k = w.shape
        hi = weights.from_bf16_bits(t2[n + ".th"].view(np.uint16)).reshape(k, co, ci)
        lo = weights.from_bf16_bits(t2[n + ".tl"].view(np.uint16)).reshape(k, co, ci)
        wt = np.transpose(w, (2, 0, 1)).astype(np.float64)
        err = np.abs(hi.astype(np.float64) + lo - wt)
        assert (err <= np.abs(wt) * 2.0 ** -16).all(), n


def test_text_blob_of_mode2_adds_only_decoder_planes():
    cfg = TI.config()
    sd = TI.model(cfg)
    t1, t2 = tensors(weights.pack_stabletts(sd, cfg, precision=1)), tensors(weights.pack_stabletts(sd, cfg, precision=2))
    extra = set(t2) - set(t1)
    assert extra == {n + s for n in weights.stabletts_tc_convs(cfg) for s in (".th", ".tl")}
    assert not any(n.startswith("st.enc") for n in extra)        # the text encoder stays fp32 in every mode


def test_pipe_of_each_conv_at_the_reference_widths():
    cfg = C.stabletts_cfm_config()
    assert (cfg["noise_channels"], cfg["cond_channels"], cfg["hidden_channels"], cfg["filter_channels"]) == (80, 256, 384, 768)
    names = weights.stabletts_tc_convs(cfg)
    want = ["st.cp0", "st.cp1", "st.cp2"] + ["st.l%d.%s" % (l, n) for l in range(cfg["n_layers"]) for n in ("qkv", "o", "ffn1", "ffn2")]
    want += ["st.lsc%d" % j for j in range(cfg["n_layers"] // 2)]
    assert names == want
    assert "st.in" not in names and "st.final" not in names     # 464 inputs; 80 outputs (and x, v stay fp32)


def test_pipe_falls_back_to_ffma_for_widths_off_the_tile():
    """filter 720 (a multiple of 16, not of 64): cond_proj and the FFN convs stay on the FFMA pipe, qkv / o / long skips not."""
    cfg = C.stabletts_cfm_config({"filter_channels": 720})
    names = weights.stabletts_tc_convs(cfg)
    assert not any(n.startswith("st.cp") or n.endswith(".ffn1") or n.endswith(".ffn2") for n in names)
    assert names == ["st.l%d.%s" % (l, n) for l in range(cfg["n_layers"]) for n in ("qkv", "o")] + ["st.lsc%d" % j for j in range(3)]
    # hidden 352 (11 heads of 32): only the two cond_proj convs that neither read nor write the hidden width
    cfg = C.stabletts_cfm_config({"hidden_channels": 352, "n_heads": 11})
    assert weights.stabletts_tc_convs(cfg) == ["st.cp0", "st.cp1"]


def test_precision_is_checked(cfm):
    cfg, sd = cfm
    with pytest.raises(ValueError, match="precision"):
        weights.pack_stabletts_cfm(sd, cfg, precision=4)
