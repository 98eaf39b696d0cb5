"""A multistream voice's model.onnx (matcha/onnx/export.py's MatchaWithVocoder graph) read back on the host: every tensor, the
configs and the step count against what the test graph was exported from (oracle/make_golden_stabletts_onnx.py, rebuilt by
tests/stabletts_onnx_inputs.py), the refusals of what is not such a graph, and Model over a deployed directory without a checkpoint."""
import json
import os
import shutil

import numpy as np
import pytest
import torch

import stabletts_onnx_inputs as SI
from vosk_tts_b200 import config as C, engine as E, onnx_weights as O, synthetic, weights as W
from vosk_tts_b200.model import Model

GOLDEN = SI.GOLDEN
NOT_BUILT = "the exported graph is not built as matcha/onnx/export.py builds it"


@pytest.fixture(scope="module")
def fix():
    return dict(np.load(os.path.join(GOLDEN, "ref_stabletts_onnx.npz")))


@pytest.fixture(scope="module")
def graph_path(tmp_path_factory, fix):
    return SI.write_graph(tmp_path_factory.mktemp("stabletts_onnx"), fix)


@pytest.fixture(scope="module")
def graph(graph_path):
    return O.stabletts_from_onnx(graph_path)


def test_every_tensor_equals_the_checkpoint(graph):
    sd = SI.model_state_dict()
    got = graph["state_dict"]
    # the mel encoder feeds only encoder_outputs, which the graph does not return: the exporter drops it
    assert sorted(k for k in sd if k not in got) == sorted(k for k in sd if k.startswith("encoder.encoder."))
    assert not [k for k in got if k not in sd]
    for k, v in got.items():
        assert v.dtype == np.float32 and np.array_equal(v, sd[k]), k
    # bert_proj.1 is the one Linear on 3-D input: a MatMul with the transposed weight, recovered through its bias's Add
    assert got["encoder.bert_proj.1.weight"].shape == (32, 768)
    voc = SI.vocoder_state_dict()
    assert sorted(graph["vocoder"]) == sorted(voc)
    for k, v in graph["vocoder"].items():
        assert v.dtype == np.float32 and np.array_equal(v, voc[k]), k


def test_configs_and_steps_are_the_exported_ones(fix, graph):
    assert graph["config"] == C.stabletts_config(json.loads(str(fix["config"])))
    assert graph["vocoder_config"] == C.hifigan_config(json.loads(str(fix["vocoder_config"])))
    assert graph["n_timesteps"] == int(fix["n_timesteps"]) == 3
    assert C.hop_samples(graph["vocoder_config"]) == 256          # export.py's wav_lengths = mel_lengths * 256


def test_recovered_conditioning_gives_torch_rows(fix, graph):
    """The FiLM rows of every step and the guidance branch's adaLN rows, which the reference computes from time_mlp, the film
    convs and fake_speaker, follow from the recovered weights (fp32, as the engine's dit_time_kernel / dit_ada_kernel run)."""
    sd = {k: torch.from_numpy(np.array(v)) for k, v in graph["state_dict"].items()}
    e, n, H = "decoder.estimator.", graph["n_timesteps"], graph["config"]["hidden_channels"]
    t_span = 1 - torch.cos(torch.linspace(0, 1, n + 1) * 0.5 * torch.pi)
    t, dt = t_span[0], t_span[1] - t_span[0]
    half = H // 2
    freq = torch.exp(torch.arange(half).float() * -(np.log(10000) / (half - 1)))
    lin = lambda x, p: x @ sd[p + ".weight"].T + sd[p + ".bias"]
    for s in range(n):
        a = 1000 * t.reshape(1, 1) * freq[None]
        te = lin(torch.nn.functional.silu(lin(torch.cat([a.sin(), a.cos()], -1), e + "time_mlp.layer.0")), e + "time_mlp.layer.2")
        for l in range(graph["config"]["n_layers"]):
            f = e + "blocks.%d.time_fusion.film." % l
            row = te @ sd[f + "weight"][:, :, 0].T + sd[f + "bias"]
            assert np.allclose(row[0].numpy(), fix["film"][s, l], rtol=1e-5, atol=1e-5), (s, l)
        t = t + dt
        if s + 1 < n:
            dt = t_span[s + 2] - t
    for l in range(graph["config"]["n_layers"]):
        p = e + "blocks.%d.block.adaLN_modulation." % l
        row = lin(torch.nn.functional.silu(lin(sd["fake_speaker"], p + "0")), p + "2")
        assert np.allclose(row[0].numpy(), fix["ada_uncond"][l], rtol=1e-5, atol=1e-5), l


def _pb(fno, payload):
    """One length-delimited protobuf field."""
    key, n, out = bytearray(), len(payload), bytearray()
    for v, dst in ((fno << 3 | 2, key), (n, out)):
        while True:
            dst.append((v & 0x7F) | (0x80 if v > 0x7F else 0))
            v >>= 7
            if not v:
                break
    return bytes(key) + bytes(out) + payload


def _graph_bytes(tensors, external=False):
    """A ModelProto whose graph holds only the given float32 initializers."""
    inits = b""
    for name, a in tensors.items():
        t = b"".join(bytes([0x08]) + bytes([d]) for d in a.shape) + bytes([0x10, 1]) + _pb(8, name.encode())
        t += bytes([0x70, 1]) if external else _pb(9, np.ascontiguousarray(a, np.float32).tobytes())
        inits += _pb(5, t)
    return _pb(7, inits)


@pytest.mark.parametrize("case", ["one_byte", "truncated", "vits", "mel_only", "no_vocoder", "single_speaker", "external", "folded"])
def test_refusals(tmp_path, graph_path, case):
    p = tmp_path / "model.onnx"
    z = lambda *s: np.zeros(s, np.float32)
    blob = open(graph_path, "rb").read()
    data, reason = {
        "one_byte": (b"\0", "readable"),
        "truncated": (blob[:len(blob) // 2], "readable"),
        "vits": (open(os.path.join(GOLDEN, "tiny_model.onnx"), "rb").read(), "VITS"),
        "mel_only": (_graph_bytes({"encoder.emb.weight": z(4, 8), "spk_emb.weight": z(2, 4)}), "mel-only export without the vocoder"),
        "no_vocoder": (_graph_bytes({"matcha.encoder.emb.weight": z(4, 8)}), "no vocoder.conv_pre.weight"),
        "single_speaker": (_graph_bytes({"matcha.encoder.emb.weight": z(4, 8), "vocoder.conv_pre.weight": z(8, 80, 7)}), "single-speaker"),
        "external": (_graph_bytes({"matcha.encoder.emb.weight": z(4, 8)}, external=True), "external data"),
        "folded": (_graph_bytes({"matcha.encoder.emb.weight": z(4, 8), "vocoder.conv_pre.weight": z(8, 80, 7),
                                 "matcha.spk_emb.weight": z(2, 4)}), "time_mlp.layer.0.weight is missing"),
    }[case]
    p.write_bytes(data)
    with pytest.raises(ValueError) as e:
        O.stabletts_from_onnx(str(p))
    assert NOT_BUILT in str(e.value) and reason in str(e.value), str(e.value)


class _FakeEngine:
    """Stands in for the CUDA engine: records what the host packs for it."""
    made = []

    def __init__(self, cfg, blob, man, device=0, precision=1):
        self.cfg, self.blob, self.man = cfg, blob, man
        _FakeEngine.made.append(self)

    def close(self):
        pass


def _deployed_dir(tmp_path):
    """config.json, dictionary, bert/ (vocab.txt, config.json, a synthetic 768-wide BERT) and the exported model.onnx, nothing else."""
    fixj = json.load(open(os.path.join(GOLDEN, "multistream_front.json"), encoding="utf-8"))
    d = tmp_path / "voice"
    (d / "bert").mkdir(parents=True)
    cfg = {"model_type": "multistream_v3", "phoneme_id_map": {k: v % 40 for k, v in fixj["phoneme_id_map"].items()},
           "inference": {"noise_level": 0.667, "speech_rate": 1.0, "duration_noise_level": 0.8, "scale": 1.0}}
    (d / "config.json").write_text(json.dumps(cfg), encoding="utf-8")
    (d / "dictionary").write_text("".join("%s 1.0 %s\n" % (w, p) for w, p in fixj["dictionary"].items()), encoding="utf-8")
    vocab = os.path.join(GOLDEN, "multistream_vocab.txt")
    shutil.copyfile(vocab, str(d / "bert" / "vocab.txt"))
    bcfg = {"hidden_size": 768, "num_attention_heads": 12, "intermediate_size": 768, "num_hidden_layers": 3,
            "vocab_size": len(open(vocab, encoding="utf-8").read().splitlines())}
    (d / "bert" / "config.json").write_text(json.dumps(bcfg))
    torch.save(synthetic.make_random_bert(C.bert_config(bcfg), 5), str(d / "bert" / "pytorch_model.bin"))
    SI.write_graph(d)
    return d


def test_model_loads_the_deployed_directory(tmp_path, monkeypatch, graph):
    monkeypatch.setattr(E, "Engine", _FakeEngine)
    for name in ("load_lightning_state_dict", "load_hifigan", "load_checkpoint"):
        monkeypatch.setattr(W, name, lambda *a, **k: pytest.fail("a checkpoint was read"))
    d = _deployed_dir(tmp_path)
    _FakeEngine.made.clear()
    m = Model(model_path=d)
    assert m.onnx.multistream and m.onnx.n_timesteps == 3 and m.onnx.tts.n_timesteps == 3 and m.tokenizer is not None
    eng = _FakeEngine.made[-1]
    assert eng.cfg["n_spks"] == 3 and eng.cfg["vocoder"] == graph["vocoder_config"] and eng.cfg["bert"]["cv_hidden"] == 768
    assert "st.enc.dp.proj" in str(eng.man) and "st.enc.mel.proj" not in str(eng.man)
    assert Model(model_path=d, n_timesteps=3).onnx.n_timesteps == 3
    with pytest.raises(ValueError, match="unrolls 3 flow-matching steps; n_timesteps=5"):
        Model(model_path=d, n_timesteps=5)
