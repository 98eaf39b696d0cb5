"""The multistream StableTTS front end on the host, against what the reference's own Synth fed its graphs
(tests/golden/multistream_front.json, oracle/make_golden_multistream.py): the WordPiece tokenizer, g2p_multistream*,
get_word_bert's selection, Synth.synth_audio's feeds over a stub session, and the refusals."""
import json
import os
import random
import shutil

import numpy as np
import pytest

from vosk_tts_b200.model import Model
from vosk_tts_b200.synth import Synth
from vosk_tts_b200.wordpiece import BertWordPieceTokenizer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
VOCAB = os.path.join(GOLDEN, "multistream_vocab.txt")
MODEL_TYPES = {"v1": "multistream_v1", "v2": "multistream_v2", "v3": "multistream_v3", "v2_nobert": "multistream_v2"}


def _fixture():
    with open(os.path.join(GOLDEN, "multistream_front.json"), encoding="utf-8") as f:
        return json.load(f)


FIX = _fixture()


class _StubSession:
    """A multistream session that records what Synth sends; BERT's row i holds i, as the fixture's stub."""
    multistream = True

    def __init__(self):
        self.calls = []

    def bert_features(self, ids):
        return np.repeat(np.arange(len(ids), dtype=np.float32)[:, None], 2, 1)

    def run(self, output_names, feeds):
        self.calls.append(("run", feeds, None, None))
        return [np.full((1, 300), 0.4, np.float32), np.array([300])]

    def run_pieces(self, feeds, pieces, bert_rows):
        assert "bert" not in feeds
        self.calls.append(("pieces", feeds, pieces, bert_rows))
        return [np.full((1, 300), 0.4, np.float32), np.array([300])]


def _model_dir(tmp_path, variant, fix=FIX, vocab=True):
    d = tmp_path / variant
    d.mkdir()
    cfg = {"model_type": MODEL_TYPES[variant], "phoneme_id_map": fix["phoneme_id_map"],
           "inference": {"noise_level": 0.667, "speech_rate": 1.0, "duration_noise_level": 0.8, "scale": 1.0}}
    (d / "config.json").write_text(json.dumps(cfg), encoding="utf-8")
    (d / "dictionary").write_text("".join("%s 1.0 %s\n" % (w, p) for w, p in fix["dictionary"].items()), encoding="utf-8")
    if vocab and variant != "v2_nobert":
        (d / "bert").mkdir()
        shutil.copyfile(VOCAB, str(d / "bert" / "vocab.txt"))
    return d


def _sub(tmp_path, name):
    (tmp_path / name).mkdir()
    return tmp_path / name


def test_tokenizer_matches_the_reference_tokens():
    tok = BertWordPieceTokenizer(VOCAB, unk_token="[UNK]", lowercase=True)
    for d in FIX["direct"]:
        enc = tok.encode(d["text"].replace("+", "").replace("_", ""))
        assert enc.tokens == d["tokens"] and enc.ids == d["ids"], d["text"]
        assert enc.attention_mask == [1] * len(enc.ids) and enc.type_ids == [0] * len(enc.ids)
    assert tok.normalize("Мой ЕЩЁ") == "мои еще"        # accents stripped, as lowercase=True does


def test_tokenizer_matches_the_library_on_generated_strings():
    tokenizers = pytest.importorskip("tokenizers")
    ref = tokenizers.BertWordPieceTokenizer(VOCAB, unk_token="[UNK]", lowercase=True)
    tok = BertWordPieceTokenizer(VOCAB, unk_token="[UNK]", lowercase=True)
    rng = random.Random(11)
    alphabet = ("приветмойеёщизадомЁЙПРИМabcXYZ ,.-\"!?()—…_+;:'`~$€«»„“%&*#@\\|/<>[]{}\t\n\r\x0b\x0c\x85\xa0　 "
                "​­́�\x00\x01中文ﬁİΣß\u2065\ud7ff\u0378\U0010ffff\U000e0001\ue000")   # unassigned, tag, private use
    words = [w for w in (l.rstrip("\n") for l in open(VOCAB, encoding="utf-8")) if not w.startswith("[")]
    for n in range(400):
        parts = [rng.choice(alphabet) if rng.random() < 0.6 else rng.choice(words).lstrip("#") for _ in range(rng.randint(0, 12))]
        text = "".join(parts) if n % 50 else "я" * (95 + n // 50)
        a, b = tok.encode(text), ref.encode(text)
        assert (a.tokens, a.ids) == (b.tokens, b.ids), repr(text)


def test_g2p_multistream_wrappers_match_the_reference(tmp_path):
    s = Synth(Model(model_path=_model_dir(tmp_path, "v2"), session=_StubSession()))
    emb = np.arange(200, dtype=np.int64)[:, None]
    for d in FIX["direct"]:
        for key, fn in (("g2p_multistream", lambda: s.g2p_multistream(d["text"], emb)),
                        ("g2p_multistream_pos", lambda: s.g2p_multistream(d["text"], emb, word_pos=True)),
                        ("g2p_multistream_scales", lambda: s.g2p_multistream_scales(d["text"], emb))):
            want = d[key]
            if "error" in want:
                with pytest.raises(ValueError, match="phoneme_id_map"):
                    fn()
                continue
            r = fn()
            assert [list(x) for x in r[0]] == want["ids"], (key, d["text"])
            assert [int(x[0]) for x in r[1]] == want["rows"], (key, d["text"])
            if want["extra"] is not None:
                assert list(r[2]) == want["extra"], (key, d["text"])
        if "ids" in d["g2p_multistream"]:         # without BERT rows: the same ids, no rows
            assert s.g2p_multistream(d["text"], None) == ([tuple(x) for x in d["g2p_multistream"]["ids"]], [])
        for nopunc, key in ((False, "selected"), (True, "selected_nopunc")):
            assert s.get_word_bert(d["text"], nopunc=nopunc)[:, 0].astype(int).tolist() == d[key], d["text"]
        assert s.add_pos(["a"]) == ["a_S"] and s.add_pos(["a", "b", "c"]) == ["a_B", "b_I", "c_E"]


@pytest.mark.parametrize("variant", sorted(MODEL_TYPES))
def test_synth_audio_sends_the_reference_feeds(tmp_path, variant):
    sess = _StubSession()
    s = Synth(Model(model_path=_model_dir(tmp_path, variant), session=sess))
    assert (s.model.tokenizer is None) == (variant == "v2_nobert")
    for c in (c for c in FIX["cases"] if c["variant"] == variant):
        if c["error"]:
            with pytest.raises(ValueError):
                s.synth_audio(c["text"], **c["args"])
            continue
        audio = s.synth_audio(c["text"], **c["args"])
        kind, feeds, pieces, rows = sess.calls[-1]
        assert kind == ("run" if variant == "v2_nobert" else "pieces"), c["text"]
        assert feeds["input"].dtype == np.int64 and feeds["input"][0].T.tolist() == c["input"], c["text"]
        assert feeds["input_lengths"].tolist() == c["input_lengths"]
        assert np.array_equal(feeds["scales"], np.array(c["scales"], np.float32)) and feeds["scales"].dtype == np.float32
        assert feeds["sid"].tolist() == c["sid"]
        if c["phone_duration_extra"] is None:
            assert feeds["phone_duration_extra"] is None
        else:
            assert feeds["phone_duration_extra"][0].tolist() == c["phone_duration_extra"]
        if variant == "v2_nobert":
            assert list(feeds["bert"].shape) == c["bert_shape"] and not feeds["bert"].any()
        else:
            text = c["text"].strip().replace("—", "-")           # synth_audio's text, lowercased by v3 (synth.py:58-65)
            assert [p.tolist() for p in pieces] == [s.model.tokenizer.encode((text.lower() if variant == "v3" else text)
                                                                             .replace("+", "").replace("_", "")).ids]
            assert rows.dtype == np.int32 and rows[0].tolist() == c["rows"], c["text"]
        assert audio.dtype == np.int16 and audio.size == c["audio_len"] and audio[:4].tolist() == c["audio"]
        chunks = list(s.synth_audio_stream(c["text"], **c["args"]))
        assert len(chunks) == 1 and np.array_equal(chunks[0], audio)


def test_multistream_refusals(tmp_path):
    # a multistream model refuses a session that is not a multistream one
    class _Vits:
        def run(self, names, feeds):
            return [np.zeros((1, 1, 1, 10), np.float32)]
    with pytest.raises(ValueError, match="multistream session"):
        Model(model_path=_model_dir(tmp_path, "v1"), session=_Vits())
    # the deployed graph alone: reading StableTTS weights out of model.onnx is not built
    d = _model_dir(tmp_path, "v3")
    (d / "model.onnx").write_bytes(b"\0")
    with pytest.raises(ValueError, match="exported graph is not built"):
        Model(model_path=d)
    d = _model_dir(tmp_path, "v2_nobert")
    with pytest.raises(FileNotFoundError):
        Model(model_path=d)
    # v1 / v3 need the tokenizer
    s = Synth(Model(model_path=_model_dir(_sub(tmp_path, "x"), "v1", vocab=False), session=_StubSession()))
    with pytest.raises(ValueError, match="tokenizer"):
        s.synth_audio("привет")
    # conversion and alignment stay VITS-only
    s = Synth(Model(model_path=_model_dir(_sub(tmp_path, "y"), "v2"), session=_StubSession()))
    with pytest.raises(ValueError, match="not a VITS2 graph"):
        s.convert_audio(np.zeros(512, np.int16), 0, 1)
    with pytest.raises(ValueError, match="not a VITS2 graph"):
        s.align_audio("привет", np.zeros(512, np.int16))
    # a phone missing from the map is named
    fix = dict(FIX, phoneme_id_map={k: v for k, v in FIX["phoneme_id_map"].items() if k != "m_S"})
    s = Synth(Model(model_path=_model_dir(_sub(tmp_path, "z"), "v1", fix), session=_StubSession()))
    s.synth_audio("мир")                              # (m_S is not a phone of this word)
    fix = dict(FIX, phoneme_id_map={k: v for k, v in FIX["phoneme_id_map"].items() if k != "$"})
    s = Synth(Model(model_path=_model_dir(_sub(tmp_path, "w"), "v1", fix), session=_StubSession()))
    with pytest.raises(ValueError, match="'\\$'"):
        s.synth_audio("мир")
    # BERT-conditioned VITS graphs (a tokenizer, model_type not multistream_*) keep being refused
    d = _model_dir(_sub(tmp_path, "v"), "v1")
    cfg = json.loads((d / "config.json").read_text(encoding="utf-8"))
    cfg["model_type"] = "vits2"
    (d / "config.json").write_text(json.dumps(cfg), encoding="utf-8")
    with pytest.raises(ValueError, match="^bert-conditioned / multistream models are not VITS2 graphs: not supported by this engine$"):
        Model(model_path=d, session=_StubSession())


class _HydraConfigLike(dict):
    """Stands for the omegaconf DictConfig a Lightning checkpoint's hyper_parameters hold: a class outside torch."""


class _RunsOnLoad:
    def __init__(self, path):
        self.path = path

    def __reduce__(self):
        return (open, (self.path, "w"))


def _lightning_checkpoint(path, sd, marker):
    """What the reference's training (MatchaTTS.save_hyperparameters, Lightning's ModelCheckpoint) writes: the state dict
    beside hyper_parameters holding a functools.partial of the optimizer and Hydra configs, optimizer states and loops."""
    import functools
    import torch
    torch.save({"state_dict": sd, "epoch": 12, "global_step": 3400, "pytorch-lightning_version": "2.1.0",
                "hyper_parameters": {"optimizer": functools.partial(torch.optim.Adam, lr=1e-4, weight_decay=0.0),
                                     "encoder": _HydraConfigLike(n_feats=80, n_spks=3), "tamper": _RunsOnLoad(marker)},
                "optimizer_states": [{"state": {0: {"exp_avg": torch.ones(3)}}, "param_groups": [{"lr": 1e-4}]}],
                "loops": {"fit_loop": {"state_dict": {}}}, "callbacks": {}}, str(path))


def test_lightning_checkpoint_loads_its_state_dict_only(tmp_path):
    import torch
    from vosk_tts_b200 import weights
    sd = {"encoder.emb.weight": torch.randn(7, 4), "spk_emb.weight": torch.randn(3, 2), "mel_mean": torch.tensor(-5.5),
          "conv.weight_g": torch.rand(4, 1, 1) + 0.5, "conv.weight_v": torch.randn(4, 2, 3)}
    marker = tmp_path / "ran"
    _lightning_checkpoint(tmp_path / "model.ckpt", sd, str(marker))
    with pytest.raises(Exception):
        torch.load(str(tmp_path / "model.ckpt"), weights_only=True)   # what a plain safe load does with it
    out = weights.load_lightning_state_dict(str(tmp_path / "model.ckpt"))
    assert not marker.exists()                                        # nothing the file names was called
    assert sorted(out) == ["conv.weight", "encoder.emb.weight", "mel_mean", "spk_emb.weight"]
    assert torch.equal(out["encoder.emb.weight"], sd["encoder.emb.weight"])
    assert torch.allclose(out["conv.weight"], weights.fold_weight_norm(sd)["conv.weight"])
    torch.save(sd, str(tmp_path / "plain.ckpt"))                      # a file holding the state dict alone
    assert sorted(weights.load_lightning_state_dict(str(tmp_path / "plain.ckpt"))) == sorted(out)
    torch.save({"state_dict": {"a": _HydraConfigLike()}}, str(tmp_path / "bad.ckpt"))
    with pytest.raises(ValueError, match="no state dict"):
        weights.load_lightning_state_dict(str(tmp_path / "bad.ckpt"))


def test_single_speaker_checkpoint_is_refused_with_the_reason(tmp_path):
    import torch
    d = _model_dir(tmp_path, "v2_nobert")
    _lightning_checkpoint(d / "model.ckpt", {"encoder.emb.weight": torch.randn(7, 4)}, str(tmp_path / "ran"))
    (d / "generator_v1").write_bytes(b"")
    with pytest.raises(ValueError, match="single-speaker"):
        Model(model_path=d)
    assert not (tmp_path / "ran").exists()
