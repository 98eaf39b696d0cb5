"""BERT's host side without a GPU: the float64 / float32 oracle against transformers' BertModel as bert-export.py calls it,
the Hugging Face checkpoint loader, the bt.* packing and the shapes the engine refuses."""
import json
import os

import numpy as np
import pytest
import torch

import bert_inputs as BI
from oracle import bert_oracle as O
from vosk_tts_b200 import config as C, weights
from vosk_tts_b200.engine import make_c_config


def _hf_model(bt, sd):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.BertConfig(hidden_size=bt["cv_hidden"], num_hidden_layers=bt["cv_layers"] + 2,
                                  num_attention_heads=bt["cv_heads"], intermediate_size=bt["cv_ffn"], vocab_size=bt["bt_vocab"],
                                  max_position_embeddings=bt["bt_max_pos"], type_vocab_size=bt["bt_type_rows"])
    m = transformers.BertModel(cfg, add_pooling_layer=False).eval()
    m.load_state_dict(sd, strict=True)
    return m


def _reference(m, ids):
    """bert-export.py's OurBert.forward: cat(hidden_states[-3:-2]).squeeze(0) on one sentence, mask ones, token types 0."""
    x = torch.as_tensor(ids)[None]
    with torch.no_grad():
        out = m(input_ids=x, attention_mask=torch.ones_like(x), token_type_ids=torch.zeros_like(x), output_hidden_states=True)
    return torch.cat(out["hidden_states"][-3:-2], -1).squeeze(0)


@pytest.mark.parametrize("shape", ["tiny", "production"])
def test_oracle_matches_transformers(shape):
    bt = getattr(BI, shape)()
    sd = BI.model(bt)
    m = _hf_model(bt, sd)
    for L in (2, 7, 64) if shape == "production" else BI.LENGTHS:
        ids = BI.sentence(bt, L)
        ref = _reference(m, ids)
        assert float((O.bert_features(sd, bt, ids, torch.float32) - ref).abs().max()) < 1e-5
        # float64 against the float32 model: within the model's own rounding
        assert float((O.bert_features(sd, bt, ids) - ref.double()).abs().max()) < 1e-4
    m64 = m.double()
    ids = BI.sentence(bt, 64)
    assert float((O.bert_features(sd, bt, ids) - _reference(m64, ids)).abs().max()) < 1e-12


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_load_bert_directory(tmp_path, fmt):
    bt = BI.tiny()
    sd = BI.model(bt)
    cfg = {"hidden_size": 128, "num_attention_heads": 4, "intermediate_size": 512, "num_hidden_layers": 4, "vocab_size": 300,
           "max_position_embeddings": 512, "type_vocab_size": 2, "layer_norm_eps": 1e-12, "hidden_act": "gelu"}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    prefixed = {"bert." + k: v for k, v in sd.items()}          # a BertForMaskedLM checkpoint's names
    prefixed["cls.predictions.bias"] = torch.zeros(300)
    if fmt == "safetensors":
        from safetensors.torch import save_file
        save_file(prefixed, str(tmp_path / "model.safetensors"))
    else:
        torch.save(prefixed, str(tmp_path / "pytorch_model.bin"))
    got, gbt = weights.load_bert(str(tmp_path))
    assert gbt == bt and gbt["cv_layers"] == 2
    for k, v in sd.items():
        assert torch.equal(torch.as_tensor(got[k]), v), k
    assert not any(k.startswith("cls.") or k.startswith("bert.") for k in got if k in sd)
    with pytest.raises(ValueError):
        weights.load_bert(str(tmp_path / "config.json"))


def test_pack_bert_layout():
    bt = BI.tiny()
    sd = BI.model(bt)
    blob, man = weights.pack_bert(sd, bt, tc=True)
    ents = {n: (int(o), int(c)) for n, o, c in (ln.split() for ln in man.strip().split("\n"))}
    H, Fh = bt["cv_hidden"], bt["cv_ffn"]
    assert ents["bt.emb.word"][1] == bt["bt_vocab"] * H and ents["bt.emb.pos"][1] == bt["bt_max_pos"] * H
    o, n = ents["bt.emb.type"]
    assert np.array_equal(blob[o:o + n].reshape(-1, H), sd["embeddings.token_type_embeddings.weight"].numpy())
    # the layers that run, and not the two bert-export.py drops
    assert "bt.l1.ffn2.th" in ents and "bt.l2.qkv.b" not in ents
    o, n = ents["bt.l1.qkv.w"]
    w = blob[o:o + n].reshape(H, 3 * H)                            # [k=1][Cin][ldw]
    q = sd["encoder.layer.1.attention.self.query.weight"].numpy()
    v = sd["encoder.layer.1.attention.self.value.weight"].numpy()
    assert np.array_equal(w[:, :H], q.T) and np.array_equal(w[:, 2 * H:], v.T)
    assert ents["bt.l0.ffn1.th"][1] == Fh * H // 2
    _, man0 = weights.pack_bert(sd, bt, tc=False)
    assert ".th " not in man0


def test_pack_refuses_wrong_shapes():
    bt = BI.tiny()
    sd = dict(BI.model(bt))
    sd["embeddings.position_embeddings.weight"] = sd["embeddings.position_embeddings.weight"][:100]
    with pytest.raises(ValueError, match="position_embeddings"):
        weights.pack_bert(sd, bt)


@pytest.mark.parametrize("over, match", [
    ({"hidden_size": 120, "num_attention_heads": 4}, "head widths"),
    ({"hidden_size": 768, "num_attention_heads": 16}, "head widths"),
    ({"hidden_act": "relu"}, "gelu"),
    ({"position_embedding_type": "relative_key"}, "absolute"),
    ({"num_hidden_layers": 2}, "no BERT layer"),
    ({"intermediate_size": 100}, "intermediate_size"),
])
def test_config_refusals(over, match):
    with pytest.raises(ValueError, match=match):
        C.bert_config(over)


def test_c_config_fields():
    bt = BI.production()
    cfg = C.stabletts_cfm_config()
    cfg["bert"] = bt
    c = make_c_config(cfg, precision=1)
    assert (c.cv_layers, c.cv_hidden, c.cv_heads, c.cv_ffn) == (10, 768, 12, 3072)
    assert abs(c.cv_ln_eps - 1e-12) < 1e-18
    assert make_c_config(C.stabletts_cfm_config(), 1).cv_layers == 0


def test_flops_count():
    bt = BI.production()
    # about 142 MFLOP per word piece for the 10 layers (the GEMMs; attention adds 4 L H per piece per layer)
    assert abs(O.flops(bt, 1) / 1e6 - 141.6) < 0.1


class _ExportBert(torch.nn.Module):
    """BertModel's modules under BertModel's names, with all cv_layers + 2 layers as a checkpoint holds them, whose forward
    returns the output of layer cv_layers (hidden_states[-3]) as bert-export.py's OurBert does.  The installed transformers
    cannot be traced by torch's TorchScript exporter, so this restatement stands in for it when writing the graph."""

    def __init__(self, bt, sd):
        super().__init__()
        nn, H, Fh = torch.nn, bt["cv_hidden"], bt["cv_ffn"]
        self.bt = bt
        self.embeddings = nn.Module()
        self.embeddings.word_embeddings = nn.Embedding(bt["bt_vocab"], H)
        self.embeddings.position_embeddings = nn.Embedding(bt["bt_max_pos"], H)
        self.embeddings.token_type_embeddings = nn.Embedding(bt["bt_type_rows"], H)
        self.embeddings.LayerNorm = nn.LayerNorm(H, eps=bt["cv_ln_eps"])
        self.encoder = nn.Module()
        self.encoder.layer = nn.ModuleList()
        for _ in range(bt["cv_layers"] + 2):
            m = nn.Module()
            m.attention = nn.Module()
            m.attention.self = nn.Module()
            for n in ("query", "key", "value"):
                setattr(m.attention.self, n, nn.Linear(H, H))
            m.attention.output = nn.Module()
            m.attention.output.dense = nn.Linear(H, H)
            m.attention.output.LayerNorm = nn.LayerNorm(H, eps=bt["cv_ln_eps"])
            m.intermediate = nn.Module()
            m.intermediate.dense = nn.Linear(H, Fh)
            m.output = nn.Module()
            m.output.dense = nn.Linear(Fh, H)
            m.output.LayerNorm = nn.LayerNorm(H, eps=bt["cv_ln_eps"])
            self.encoder.layer.append(m)
        self.load_state_dict(sd, strict=True)

    def forward(self, input_ids, attention_mask, token_type_ids):
        e, nh = self.embeddings, self.bt["cv_heads"]
        L = input_ids.shape[1]
        pos = torch.arange(L).unsqueeze(0)
        x = e.LayerNorm(e.word_embeddings(input_ids) + e.token_type_embeddings(token_type_ids) + e.position_embeddings(pos))
        hs = [x]
        for m in self.encoder.layer:
            s = m.attention.self
            sh = lambda t: t.reshape(1, L, nh, -1).transpose(1, 2)
            q, k, v = sh(s.query(x)), sh(s.key(x)), sh(s.value(x))
            a = torch.softmax(q @ k.transpose(2, 3) / (q.shape[-1] ** 0.5), -1) @ v
            x = m.attention.output.LayerNorm(x + m.attention.output.dense(a.transpose(1, 2).reshape(1, L, -1)))
            x = m.output.LayerNorm(x + m.output.dense(torch.nn.functional.gelu(m.intermediate.dense(x))))
            hs.append(x)
        return torch.cat(hs[-3:-2], -1).squeeze(0)


def _export(tmp_path, bt, sd, name="model.onnx"):
    """Writes the graph the way bert-export.py does (inputs input_ids / attention_mask / token_type_ids, output logits,
    dynamic batch and sequence axes, constant folding, opset 17), with torch's TorchScript exporter.  The onnx package is not
    installed; the exporter imports it only to attach onnxscript functions, of which there are none, so that step is bypassed."""
    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils
    m = _ExportBert(bt, sd).eval()
    ids = torch.tensor([[2, 17, 45, 99, 3]])
    orig = onnx_proto_utils._add_onnxscript_fn
    onnx_proto_utils._add_onnxscript_fn = lambda proto, custom_opsets: proto
    try:
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            torch.onnx.export(m, (ids, torch.ones_like(ids), torch.zeros_like(ids)), str(tmp_path / name),
                              input_names=["input_ids", "attention_mask", "token_type_ids"], output_names=["logits"],
                              dynamic_axes={"input_ids": {0: "batch_size", 1: "sequence"}, "attention_mask": {0: "batch_size", 1: "sequence"},
                                            "token_type_ids": {0: "batch_size", 1: "sequence"}, "logits": {0: "batch_size", 1: "sequence"}},
                              do_constant_folding=True, opset_version=17, dynamo=False)
    finally:
        onnx_proto_utils._add_onnxscript_fn = orig
    return m


def test_load_bert_onnx_equals_seeded_weights(tmp_path):
    bt = BI.tiny()
    sd = BI.model(bt)
    m = _export(tmp_path, bt, sd)
    ids = BI.sentence(bt, 40)
    with torch.no_grad():
        ref = m(torch.as_tensor(ids)[None], torch.ones(1, 40, dtype=torch.long), torch.zeros(1, 40, dtype=torch.long))
    assert float((O.bert_features(sd, bt, ids, torch.float32) - ref).abs().max()) < 1e-5
    got, gbt = weights.load_bert(str(tmp_path / "model.onnx"), heads=4)
    assert gbt == bt and gbt["cv_layers"] == 2
    # layers 3-4 (indices 2, 3) do not reach hidden_states[-3]: the exporter drops them and the loader does not invent them
    assert not any(k.startswith("encoder.layer.2.") or k.startswith("encoder.layer.3.") for k in got)
    for k, v in sd.items():
        if k.startswith("encoder.layer.2.") or k.startswith("encoder.layer.3."):
            continue
        assert np.array_equal(np.asarray(got[k]), v.numpy()), k
    # a directory holding model.onnx (a multistream model's bert/), heads from a config.json beside it
    (tmp_path / "config.json").write_text(json.dumps({"num_attention_heads": 4}))
    got2, gbt2 = weights.load_bert(str(tmp_path))
    assert gbt2 == bt and all(np.array_equal(got2[k], got[k]) for k in got)
    # the ONNX path and the Hugging Face path pack the same blob
    assert np.array_equal(weights.pack_bert(got, gbt)[0], weights.pack_bert(sd, bt)[0])


def test_load_bert_refuses_other_graphs(tmp_path):
    with pytest.raises(ValueError, match="not a BERT graph"):
        weights.load_bert(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_model.onnx"))
