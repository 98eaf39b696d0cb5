"""CPU: forced alignment host side -- the oracle (oracle/align_oracle.py) against the reference's stored SynthesizerTrn.forward
alignment (tests/golden/ref_alignment.npz, oracle/make_golden_align.py), the float64 2-best MAS against brute force, the
phoneme segments of Synth.align_audio on a stub session, the CLI, and the C ABI declarations / exports."""
import ctypes as C
import itertools
import json
import math
import os
import re

import numpy as np
import pytest

import align_inputs as AI
import golden_ref as GR
from oracle import align_oracle as ao
from vosk_tts_b200 import cli, config as CF, synthetic, weights
from vosk_tts_b200.model import Model
from vosk_tts_b200.synth import Synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c[0]: c for c in AI.CASES}


def _ref():
    return GR.load("ref_alignment.npz")


def _weights(model):
    cfg = CF.from_training_json(AI.training_json(model), n_vocab=AI.n_vocab(model))
    return cfg, weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, AI.SEEDS[model], posterior=True))


def fp32_bound(z_p, m_p, logs_p, idx, t_x):
    """Error bound of the reference's float32 neg_cent (models.py:1645-1651, four terms, two of them fp32 GEMMs over the I
    channels) at the flat cells `idx` of [t_y, t_x]: every term is a sum of I products, each rounded, so the total is within
    (I + 8) * 2^-23 * S of the exact value, S = sum_d (|-0.5 log 2pi - logs| + 0.5 z^2 s + |z m s| + 0.5 m^2 s) with
    s = exp(-2 logs) (the 8 covers the rounding of s, of the four-term sum and of the products' operands)."""
    z, m, lg = (np.asarray(a, np.float64) for a in (z_p, m_p, logs_p))
    j, i = idx // t_x, idx % t_x
    s = np.exp(-2 * lg)
    S = (np.abs(-0.5 * math.log(2 * math.pi) - lg[:, i]) + 0.5 * z[:, j] ** 2 * s[:, i] + np.abs(z[:, j] * m[:, i] * s[:, i]) +
         0.5 * m[:, i] ** 2 * s[:, i]).sum(0)
    return (z.shape[0] + 8) * 2.0 ** -23 * S


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_reference_alignment(case):
    ref = _ref()
    p = case + "/"
    _, clip, model, sid, _ = CASES[case]
    cfg, w = _weights(model)
    ids = AI.ids(case)
    assert np.array_equal(ref[p + "ids"], ids)
    spec = AI.ref_spec(case)
    r = ao.align(w, cfg, ids, spec, sid, AI.eps_q(case, cfg["inter_channels"], spec.shape[1]))
    for nm in ("z_p", "m_p", "logs_p"):
        assert float(np.abs(r[nm] - ref[p + nm]).max()) <= 1e-4 * max(1.0, float(np.abs(ref[p + nm]).max())), nm
    assert np.array_equal(r["token_of_frame"], ref[p + "token_of_frame"])
    assert np.array_equal(r["durations"], ref[p + "w"])
    assert r["durations"].sum() == spec.shape[1] and r["durations"].min() >= 1
    # the float64 direct form on the reference's own operands is within the reference's fp32 rounding of its samples
    t_y, t_x = (int(v) for v in ref[p + "neg_cent_shape"])
    nc = ao.neg_cent(ref[p + "z_p"], ref[p + "m_p"], ref[p + "logs_p"]).reshape(-1)
    idx = ref[p + "neg_cent_idx"]
    err = np.abs(nc[idx] - ref[p + "neg_cent"])
    assert (err <= fp32_bound(ref[p + "z_p"], ref[p + "m_p"], ref[p + "logs_p"], idx, t_x)).all(), float(err.max())
    best, second = ao.two_best(ao.neg_cent(ref[p + "z_p"], ref[p + "m_p"], ref[p + "logs_p"]), t_y, t_x)
    assert (t_x == 1 or t_x == t_y) == (second == -np.inf)


def _all_paths(t_y, t_x):
    """Every monotonic path as the token of each frame: starts at token 0, ends at t_x - 1, steps of 0 or 1."""
    for steps in itertools.combinations(range(1, t_y), t_x - 1):
        tof, x = [], 0
        for y in range(t_y):
            if y in steps:
                x += 1
            tof.append(x)
        yield tof


@pytest.mark.parametrize("seed", range(40))
def test_two_best_equals_brute_force(seed):
    rng = np.random.RandomState(seed)
    t_y = rng.randint(1, 10)
    t_x = rng.randint(1, min(5, t_y) + 1)
    # small integers: float64 sums are exact, and equal scores of different paths (ties) are frequent
    nc = rng.randint(-3, 3, size=(t_y, t_x)).astype(np.float64) if seed % 2 else rng.randn(t_y, t_x)
    scores = sorted((ao.path_score(nc, p) for p in _all_paths(t_y, t_x)), reverse=True)
    best, second = ao.two_best(nc, t_y, t_x)
    assert best == scores[0]
    assert second == (scores[1] if len(scores) > 1 else -np.inf)
    # MAS itself picks a best path
    from oracle import mas_oracle
    path = mas_oracle.maximum_path(nc.astype(np.float32)[None], [t_y], [t_x])[0]
    tof, dur = ao.path_of(path)
    assert dur.min() >= 1 and dur.sum() == t_y
    assert abs(ao.path_score(nc, tof) - best) <= 1e-5 * (1 + abs(best))


class _StubSession:
    def __init__(self, hop=256, sr=22050):
        self.cfg = {"sampling_rate": sr, "hop_length": hop}
        self.calls = []

    def align(self, ids, wav, sid=0, noise=None, noise_scale=1.0):
        self.calls.append((ids, wav, sid, noise_scale))
        dur = (np.arange(ids.size) % 3 + 1).astype(np.int32)       # 1, 2, 3, 1, 2, 3, ... frames per id
        return dur, np.repeat(np.arange(ids.size), dur).astype(np.int32), -12.5


def _model(tmp_path, id_map):
    (tmp_path / "config.json").write_text(json.dumps({"phoneme_id_map": id_map}), encoding="utf-8")
    sess = _StubSession()
    return Model(str(tmp_path), session=sess), sess


def test_align_audio_phoneme_segments(tmp_path):
    id_map = {"^": [1], "$": [2], "a": [3], "b": [4, 5], ",": [6], " ": [7], "_": [0]}
    model, sess = _model(tmp_path, id_map)
    model.dic = {"ab": "a b", "ba": "b a"}
    s = Synth(model)
    audio = (np.arange(5000) % 100 - 50).astype(np.int16) * 100
    ent = s.align_audio("ab, ba", audio, speaker_id=3)
    ids, wav, sid, ns = sess.calls[-1]
    assert sid == 3 and ns == 1.0 and np.array_equal(wav, audio.astype(np.float32) / 32768.0)
    phon = ["^", "a", "b", ",", " ", "b", "a", "$"]
    assert list(ids) == [1, 0, 3, 0, 4, 5, 0, 6, 0, 7, 0, 4, 5, 0, 3, 0, 2]
    assert [e["phoneme"] for e in ent] == [phon[0]] + [x for p in phon[1:] for x in (None, p)]
    dur = np.arange(len(ids)) % 3 + 1
    cum = np.concatenate([[0], np.cumsum(dur)]) * 256 / 22050.0
    # entries tile [0, frames * hop / sr) exactly, in order
    assert ent[0]["start"] == 0.0 and ent[-1]["end"] == cum[-1]
    assert all(a["end"] == b["start"] for a, b in zip(ent, ent[1:]))
    # the two ids of "b" are merged: entry 4 is the first "b" (ids 4, 5 at positions 4 and 5)
    assert ent[4]["phoneme"] == "b" and ent[4]["start"] == cum[4] and ent[4]["end"] == cum[6]
    # every blank is one id
    for e in ent:
        if e["phoneme"] is None:
            assert round((e["end"] - e["start"]) * 22050 / 256) in (1, 2, 3)
    assert s.last_score == -12.5
    with pytest.raises(ValueError):
        s.align_audio("ab", np.zeros((2, 10), np.int16))
    with pytest.raises(ValueError):
        s.align_audio("ab", np.array([0.5, 1.5], np.float32))


def test_align_reads_wav_with_convert_checks(tmp_path):
    import wave
    model, sess = _model(tmp_path, {"^": 1, "$": 2, "_": 0})
    s = Synth(model)

    def write(path, sr):
        with wave.open(str(path), "w") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(sr)
            f.writeframes(np.zeros(3000, np.int16).tobytes())

    write(tmp_path / "a.wav", 22050)
    ent = s.align(str(tmp_path / "a.wav"), "", 0)
    assert [e["phoneme"] for e in ent] == ["^", None, "$"]
    write(tmp_path / "b.wav", 16000)
    with pytest.raises(ValueError, match="resample"):
        s.align(str(tmp_path / "b.wav"), "", 0)


def test_cli_align_arguments(monkeypatch, capsys):
    seen = {}

    class _M:
        def __init__(self, *a, **k):
            seen["model"] = k

    class _S:
        def __init__(self, m):
            pass

        def align(self, wav, text, speaker_id=None):
            seen["align"] = (wav, text, speaker_id)
            return [{"phoneme": "^", "start": 0.0, "end": 0.1}]

    monkeypatch.setattr(cli, "Model", _M)
    monkeypatch.setattr(cli, "Synth", _S)
    assert cli.main(["-m", "x", "--align", "in.wav", "-i", "hello", "-s", "2"]) == 0
    assert seen["align"] == ("in.wav", "hello", 2) and seen["model"]["voice_conversion"] is True
    assert json.loads(capsys.readouterr().out) == [{"phoneme": "^", "start": 0.0, "end": 0.1}]
    with pytest.raises(SystemExit):
        cli.main(["-m", "x", "--align", "in.wav"])


def test_c_abi_declares_and_exports_align():
    with open(os.path.join(ROOT, "include", "vtts.h")) as f:
        h = f.read()
    for nm in ("vtts_align", "vtts_align_spec"):
        assert re.search(r"\bint %s\(vtts_handle h, const int64_t\* ids, const int64_t\* id_lengths, int t_max" % nm, h), nm
    from vosk_tts_b200 import engine
    lib = C.CDLL(engine.lib_path())
    for nm in ("vtts_align", "vtts_align_spec"):
        assert hasattr(lib, nm) and nm in engine.EXPORTS
