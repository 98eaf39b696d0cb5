"""Multistream StableTTS from word pieces on the GPU (vtts_stabletts_synthesise_pieces_wav): BERT's rows computed and gathered
in the text phase's graph must give the bits of the unfused composition -- vtts_bert_features, the same gather on the host,
vtts_stabletts_synthesise_wav -- in modes 0 and 1, alone and in ragged batches, eager and replayed; its refusals; and
Model / Synth end to end over a model directory of synthetic checkpoints."""
import ctypes as C
import functools
import json
import os
import shutil
import subprocess
import sys
import wave

import numpy as np
import pytest
import torch

import bert_inputs as BI
import hifigan_inputs as HI
import stabletts_inputs as TI
from vosk_tts_b200 import config as Cfg, synthetic
from vosk_tts_b200.model import Model
from vosk_tts_b200.stabletts import StableTTS
from vosk_tts_b200.synth import Synth

pytestmark = pytest.mark.gpu
ERR_INVALID = -1
SEED = 8642


def _config(bert_dim):
    return Cfg.stabletts_config({"n_vocab": 120, "bert_dim": bert_dim})


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "mode1"])
def tts(request):
    bt = BI.tiny()
    cfg = _config(bt["cv_hidden"])
    t = StableTTS({"n_vocab": 120, "bert_dim": bt["cv_hidden"]}, synthetic.make_random_stabletts(cfg, SEED), device=0,
                  precision=request.param, vocoder=HI.checkpoint(), bert=(BI.model(bt), bt))
    t.precision = request.param
    yield t
    t.close()


def _batch(bt, n_piece_lengths, salt=0):
    """Utterances (ids [5, T], pieces, rows [T], pause [T], noise, sid): rows point at [CLS] and [SEP], repeat, and skip pieces."""
    rng = np.random.default_rng(SEED + salt)
    out = []
    for i, L in enumerate(n_piece_lengths):
        T = int(rng.integers(2, 48))
        ids = rng.integers(0, 120, (5, T)).astype(np.int64)
        rows = np.sort(rng.integers(0, L, T)).astype(np.int32)
        rows[0], rows[-1] = 0, L - 1
        pause = np.where(rng.random(T) < 0.1, 3.0, 0.0).astype(np.float32)
        noise = rng.standard_normal((80, TI.MAX_FRAMES)).astype(np.float32)
        out.append((ids, BI.sentence(bt, L, salt=100 * salt + i), rows, pause, noise, i % 2))
    return out


def _fused(t, us, **kw):
    return t.synthesise([u[0] for u in us], None, [u[5] for u in us], [u[3] for u in us], n_timesteps=3,
                        noise=[u[4] for u in us], pieces=[u[1] for u in us], bert_rows=[u[2] for u in us], **kw)


def _composed(t, us):
    feats = t.bert_features([u[1] for u in us])
    berts = [np.ascontiguousarray(f[u[2]].T) for f, u in zip(feats, us)]
    return t.synthesise([u[0] for u in us], berts, [u[5] for u in us], [u[3] for u in us], n_timesteps=3,
                        noise=[u[4] for u in us], return_wav=True)


def _same(a, b, i, j=None):
    j = i if j is None else j
    for k in ("durations", "mel", "decoder_outputs", "wav"):
        assert np.array_equal(a[k][i], b[k][j]), (k, i, j)
    assert a["mel_lengths"][i] == b["mel_lengths"][j] and a["wav_lengths"][i] == b["wav_lengths"][j]


@pytest.mark.parametrize("lengths", [[9], [2, 512, 37, 5, 300, 64, 3, 128]], ids=["B1", "ragged8"])
def test_fused_equals_composition(tts, lengths):
    us = _batch(BI.tiny(), lengths, salt=len(lengths))
    fused, comp = _fused(tts, us), _composed(tts, us)
    for b in range(len(us)):
        _same(fused, comp, b)
    again = _fused(tts, us)                      # both phases replay their graphs
    for b in range(len(us)):
        _same(again, fused, b)
    if len(us) > 1:
        for b in (0, 1, 4):
            alone = _fused(tts, [us[b]])
            if tts.precision == 0:               # (modes >= 1: the vocoder's split-K plans follow the batch, DESIGN.md 4.n)
                _same(alone, fused, 0, b)
            else:
                for k in ("durations", "mel"):
                    assert np.array_equal(alone[k][0], fused[k][b]), (k, b)


def test_padded_pieces_take_their_lengths(tts):
    us = _batch(BI.tiny(), [5, 23, 9], salt=4)
    pieces = np.zeros((3, 30), np.int64)              # zero-padded past each sentence: [PAD] rows BERT must not see
    for b, u in enumerate(us):
        pieces[b, :u[1].size] = u[1]
    T = max(u[0].shape[1] for u in us)
    ids, rows = np.zeros((3, 5, T), np.int64), np.zeros((3, T), np.int32)
    for b, u in enumerate(us):
        ids[b, :, :u[0].shape[1]], rows[b, :u[2].size] = u[0], u[2]
    noise = [np.ascontiguousarray(u[4].T) for u in us]
    kw = dict(lengths=[u[0].shape[1] for u in us], n_timesteps=3, noise=noise)
    padded = tts.engine.stabletts_synthesise(ids, None, [u[5] for u in us], pieces=pieces, bert_rows=rows,
                                             piece_lengths=[u[1].size for u in us], **kw)
    listed = tts.engine.stabletts_synthesise(ids, None, [u[5] for u in us], pieces=[u[1] for u in us], bert_rows=rows, **kw)
    for k in ("durations", "mel", "wav", "mel_lengths"):
        assert np.array_equal(padded[k], listed[k]), k
    with pytest.raises(ValueError):
        tts.engine.stabletts_synthesise(ids, None, 0, pieces=pieces, bert_rows=rows, piece_lengths=[5, 31, 9], **kw)


def test_eager_equals_replay(tts):
    us = _batch(BI.tiny(), [17, 40, 6], salt=9)
    tts.engine.set_graphs(False)
    try:
        eager = _fused(tts, us)
    finally:
        tts.engine.set_graphs(True)
    r0 = tts.engine.graph_replays()
    _fused(tts, us)
    replayed = _fused(tts, us)
    assert tts.engine.graph_replays() >= r0 + 2
    for b in range(len(us)):
        _same(replayed, eager, b)


def _raw(t, ids, rows, pieces, plen, T=None):
    T = ids.shape[2] if T is None else T
    B = ids.shape[0]
    lens, sid = np.full(B, T, np.int64), np.zeros(B, np.int64)
    mel_len, wl = np.zeros(B, np.int64), np.zeros(B, np.int64)
    wav = np.zeros((B, 1 << 20), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    t.engine.set_graphs(False)
    try:
        n0 = t.engine.kernel_launches()
        rc = t.engine.lib.vtts_stabletts_synthesise_pieces_wav(t.engine.h, p(ids), p(lens), B, ids.shape[2], p(pieces), p(plen),
                                                               pieces.shape[1], p(rows), None, p(sid), 2, 1.0, 1.0, 0.5, None, 0, 0,
                                                               None, 0, p(mel_len), None, None, 1, p(wav), wav.shape[1], p(wl))
        return rc, t.engine.kernel_launches() - n0
    finally:
        t.engine.set_graphs(True)


def test_refusals(tts):
    bt = BI.tiny()
    ids = np.ascontiguousarray(np.random.default_rng(1).integers(0, 120, (1, 5, 6)), np.int64)
    pieces = BI.sentence(bt, 5)[None].copy()
    plen = np.array([5], np.int64)
    ok = np.array([[0, 1, 2, 3, 4, 4]], np.int32)
    assert _raw(tts, ids, ok, pieces, plen)[0] == 0
    for rows in (np.array([[0, 1, 2, 3, 4, 5]], np.int32), np.array([[-1, 1, 2, 3, 4, 4]], np.int32)):
        assert _raw(tts, ids, rows, pieces, plen) == (ERR_INVALID, 0)           # a row outside the sentence
    bad = pieces.copy()
    bad[0, 2] = bt["bt_vocab"]
    assert _raw(tts, ids, ok, bad, plen) == (ERR_INVALID, 0)                  # an id outside BERT's vocabulary
    assert _raw(tts, ids, ok, pieces, np.array([0], np.int64)) == (ERR_INVALID, 0)
    long = np.full((1, 600), 5, np.int64)
    assert _raw(tts, ids, ok, long, np.array([600], np.int64)) == (ERR_INVALID, 0)   # past the position table
    with pytest.raises(ValueError):
        tts.engine.stabletts_synthesise(ids, None, 0, pieces=pieces, bert_rows=ok[:, :5])
    with pytest.raises(ValueError):
        tts.engine.stabletts_synthesise(ids, np.zeros((1, 6, bt["cv_hidden"]), np.float32), 0, pieces=pieces, bert_rows=ok)
    # no BERT in the blob, and a bert_dim that is not BERT's width
    cfg = _config(bt["cv_hidden"])
    t = StableTTS({"n_vocab": 120, "bert_dim": bt["cv_hidden"]}, synthetic.make_random_stabletts(cfg, SEED), device=0, precision=0,
                  vocoder=HI.checkpoint())
    try:
        assert _raw(t, ids, ok, pieces, plen) == (ERR_INVALID, 0)
    finally:
        t.close()
    cfg = _config(64)
    t = StableTTS({"n_vocab": 120, "bert_dim": 64}, synthetic.make_random_stabletts(cfg, SEED), device=0, precision=0,
                  vocoder=HI.checkpoint(), bert=(BI.model(bt), bt))
    try:
        assert _raw(t, ids, ok, pieces, plen) == (ERR_INVALID, 0)
    finally:
        t.close()


GOLDEN = os.path.dirname(HI.GOLDEN)


def _fixture():
    with open(os.path.join(GOLDEN, "multistream_front.json"), encoding="utf-8") as f:
        return json.load(f)


def _model_dir(root, variant, fix):
    """A multistream_* directory: config.json, dictionary, bert/ (vocab.txt, config.json, pytorch_model.bin), model.ckpt and
    generator_v1, from the synthetic StableTTS, HiFi-GAN and BERT helpers with the fixture's vocabulary and map."""
    d = root / variant
    (d / "bert").mkdir(parents=True)
    model_type = {"v1": "multistream_v1", "v2": "multistream_v2", "v3": "multistream_v3", "v2_nobert": "multistream_v2"}[variant]
    cfg = {"model_type": model_type, "phoneme_id_map": fix["phoneme_id_map"],
           "inference": {"noise_level": 0.667, "speech_rate": 1.0, "duration_noise_level": 0.8, "scale": 1.0}}
    (d / "config.json").write_text(json.dumps(cfg), encoding="utf-8")
    (d / "dictionary").write_text("".join("%s 1.0 %s\n" % (w, p) for w, p in fix["dictionary"].items()), encoding="utf-8")
    vocab = os.path.join(GOLDEN, "multistream_vocab.txt")
    n_vocab = len(open(vocab, encoding="utf-8").read().splitlines())
    if variant != "v2_nobert":
        shutil.copyfile(vocab, str(d / "bert" / "vocab.txt"))
        bcfg = {"hidden_size": 768, "num_attention_heads": 12, "intermediate_size": 3072, "num_hidden_layers": 4, "vocab_size": n_vocab}
        (d / "bert" / "config.json").write_text(json.dumps(bcfg))
        torch.save(synthetic.make_random_bert(Cfg.bert_config(bcfg), SEED), str(d / "bert" / "pytorch_model.bin"))
    scfg = Cfg.stabletts_config({"n_vocab": max(fix["phoneme_id_map"].values()) + 1, "n_spks": 3})
    # Lightning's layout, as the reference's training writes it: hyper_parameters hold a functools.partial of the optimizer
    torch.save({"state_dict": synthetic.make_random_stabletts(scfg, SEED), "epoch": 7,
                "hyper_parameters": {"optimizer": functools.partial(torch.optim.Adam, lr=1e-4)}}, str(d / "model.ckpt"))
    torch.save({"generator": HI.checkpoint()}, str(d / "generator_v1"))
    return d


@pytest.mark.parametrize("variant", ["v1", "v2", "v3", "v2_nobert"])
def test_synth_end_to_end(tmp_path, variant):
    fix = _fixture()
    d = _model_dir(tmp_path, variant, fix)
    text, speaker = "Привет, мир! Ещё \"раз\" из-за дом_ - да...", 2      # words of the fixture, whose phones the map holds
    if variant != "v3":                          # "_" is a pause mark of v3's front end only (the reference's __E KeyError)
        text = text.replace("_", "")
    model = Model(model_path=d, precision=0)
    try:
        s = Synth(model)
        out = str(tmp_path / "out.wav")
        s.synth(text, out, speaker_id=speaker)
        with wave.open(out, "rb") as w:
            assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 22050)
            pcm = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)
        # the composition with the seed of the synth call: the session's call counter, which the seed follows, is put back
        sess = model.onnx
        t = text.strip().replace("—", "-")
        mt = model.config["model_type"]
        scales = np.array([0.667, 1.0, 0.8], np.float32)
        if model.tokenizer is None:
            ids, rows, extra = s._multistream(t, True, False)
            bert = np.zeros((1, 768, len(ids)), np.float32)
        else:
            enc, keep = s._word_pieces(t.lower() if mt == "multistream_v3" else t, nopunc=True)
            ids, rows, extra = s._multistream(t, mt != "multistream_v1", mt == "multistream_v3", len(keep))
            feats = sess.bert_features(enc.ids)
            bert = np.ascontiguousarray(feats[[keep[r] for r in rows]].T[None])
        feeds = {"input": np.array(ids, np.int64).T[None], "input_lengths": np.array([len(ids)], np.int64), "scales": scales,
                 "sid": np.array([speaker], np.int64), "bert": bert,
                 "phone_duration_extra": np.array([extra], np.float32) if mt == "multistream_v3" else None}
        sess._calls -= 1                          # replay the seed of the synth call
        wav, wl = sess.run(None, feeds)
        ref = s.audio_float_to_int16(wav[0, :int(wl[0])] * 1.0)
        assert pcm.size == ref.size and np.array_equal(pcm, ref)
        assert np.abs(pcm).max() > 0
    finally:
        model.onnx.close()


def test_cli_writes_a_wav(tmp_path):
    d = _model_dir(tmp_path, "v3", _fixture())
    out = tmp_path / "out.wav"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "vosk_tts_b200.cli", "-m", str(d), "-i", "Привет, мир!", "-o", str(out)], cwd=root,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    with wave.open(str(out), "rb") as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 22050) and w.getnframes() > 0
