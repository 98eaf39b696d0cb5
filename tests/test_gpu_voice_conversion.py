"""Voice conversion on the GPU (vtts_convert / vtts_convert_spec) against the reference's SynthesizerTrn.voice_conversion,
stored by oracle/make_golden_vc.py in tests/golden/ref_voice_conversion.npz (speech input, injected posterior noise)."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

import golden_ref as GR
import vc_inputs as VI
from vosk_tts_b200 import config as CF, synthetic, weights

pytestmark = pytest.mark.gpu

_PACKED, _ENGINES = {}, {}
CASES = {c[0]: c for c in VI.CASES}


def _cfg(model):
    return CF.from_training_json(VI.training_json(model), n_vocab=62 if model == "mel" else GR.N_VOCAB)


def _packed(model):
    if model not in _PACKED:
        cfg = _cfg(model)
        sd = synthetic.make_random_checkpoint(cfg, VI.SEEDS[model], posterior=True)
        _PACKED[model] = (cfg,) + weights.pack(weights.fold_weight_norm(sd), cfg, posterior=True)
    return _PACKED[model]


def _engine(model, precision):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    key = (model, precision)
    if key not in _ENGINES:
        cfg, blob, man = _packed(model)
        _ENGINES[key] = Engine(cfg, blob, man, device=0, precision=precision)
    return _ENGINES[key]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


def _ref():
    return GR.load("ref_voice_conversion.npz")


def _rows(e, name, C_, F):
    return e.debug_read(name).reshape(F, C_)


def _run(e, case, from_spec, precision):
    """One conversion of a fixture case with the reference's eps; returns the engine's stages as reference-shaped arrays."""
    c, clip, s, t, model = CASES[case]
    cfg = e.cfg
    ref = _ref()
    I = cfg["inter_channels"]
    spec_ref = ref[c + "/spec"]
    F = spec_ref.shape[1]
    eps = VI.eps_q(c, I, F).numpy()
    e.debug_flags(1)
    try:
        if from_spec:
            o, fr = e.convert_spec(spec_ref[None], s, t, noise=eps)
        else:
            o, fr = e.convert(VI.wav_float(VI.speech()[clip]), s, t, noise=eps)
        assert int(fr[0]) == F
        out = {"o_hat": o[:, None, :]}
        sp = (cfg["spec_channels"] + 15) // 16 * 16
        out["spec"] = _rows(e, "vc_spec", sp, F)[:, : cfg["spec_channels"]].T
        for nm, dbg in (("z", "vc_z"), ("z_p", "vc_z_p"), ("z_hat", "vc_z_hat")):
            out[nm] = _rows(e, dbg, I, F).T[None]
    finally:
        e.debug_flags(0)
    return out


def _err(out, case, nm):
    ref = _ref()
    v = out[nm].reshape(-1)
    assert v.size == int(np.prod(ref[case + "/" + nm + "_shape"]))
    return float(np.abs(v[ref[case + "/" + nm + "_idx"]] - ref[case + "/" + nm]).max())


@pytest.mark.parametrize("case", ["c0", "c2"])
def test_front_end_matches_reference_spectrogram(case):
    """Reflect padding, framing, |STFT| (and mel + log) of the CUDA front end against mel_processing.py."""
    model = CASES[case][4]
    out = _run(_engine(model, 0), case, False, 0)
    ref = _ref()[case + "/spec"]
    err = float(np.abs(out["spec"] - ref).max())
    if model == "mel":
        assert err <= 1e-3, err                       # log domain
    else:
        assert err <= 1e-5 * float(np.abs(ref).max()), (err, float(np.abs(ref).max()))


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("case", ["c0", "c1", "c2"])
def test_convert_spec_matches_reference(case, precision):
    """The model part alone (vtts_convert_spec on the reference's own spectrogram): enc_q, flow forward, flow reverse,
    decoder.  Per-stage errors are printed (-s) for the precision report."""
    model = CASES[case][4]
    if precision == 1 and not weights.tc_supported(_cfg(model)):
        pytest.skip("tiny widths: no tensor-core path")
    out = _run(_engine(model, precision), case, True, precision)
    errs = {nm: _err(out, case, nm) for nm in ("z", "z_p", "z_hat", "o_hat")}
    print("convert_spec %s precision %d max abs error: %s" % (case, precision, errs))
    if precision == 0:
        assert errs["z"] <= 1e-4, errs
    assert errs["o_hat"] <= 1e-3, errs


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("case", ["c0", "c1", "c2"])
def test_convert_wav_matches_reference(case, precision):
    model = CASES[case][4]
    if precision == 1 and not weights.tc_supported(_cfg(model)):
        pytest.skip("tiny widths: no tensor-core path")
    out = _run(_engine(model, precision), case, False, precision)
    errs = {nm: _err(out, case, nm) for nm in ("z", "z_p", "z_hat", "o_hat")}
    print("convert %s precision %d max abs error: %s" % (case, precision, errs))
    assert errs["o_hat"] <= 1e-3, errs


@pytest.mark.parametrize("precision", [0, 1])
def test_same_speaker_round_trip_is_identity(precision):
    """sid_src == sid_tgt: the reverse flow undoes the forward flow (both recompute m from bit-identical x0)."""
    out = _run(_engine("mel", precision), "c1", False, precision)
    assert float(np.abs(out["z_hat"] - out["z"]).max()) <= 1e-5 * float(np.abs(out["z"]).max())


@pytest.mark.parametrize("precision", [0, 1])
def test_ragged_batch_equals_single_clips(precision):
    e = _engine("mel", precision)
    sp = VI.speech()
    clips = [VI.wav_float(sp["a"]), VI.wav_float(sp["b"]), VI.wav_float(sp["a"][7000:7000 + 5000])]
    L = max(len(c) for c in clips)
    wav = np.zeros((3, L + 100), np.float32)
    for i, c in enumerate(clips):
        wav[i, :len(c)] = c
    lens = np.array([len(c) for c in clips])
    frames = e.convert_frames(lens)
    I = e.cfg["inter_channels"]
    eps = np.random.RandomState(4).randn(3, I, int(frames.max()) + 3).astype(np.float32)
    src, tgt = np.array([3, 5, 9]), np.array([7, 5, 0])
    o, fr = e.convert(wav, src, tgt, lengths=lens, noise=eps)
    assert np.array_equal(fr, frames)
    for i, c in enumerate(clips):
        o1, f1 = e.convert(c, src[i], tgt[i], noise=eps[i:i + 1, :, : frames[i]])
        n = int(f1[0]) * e.hop
        assert float(np.abs(o[i, :n] - o1[0, :n]).max()) <= 1e-4
        assert not np.any(o[i, n:])


def test_graph_replay_equals_eager_bitwise():
    e = _engine("mel", 1)
    wav = VI.wav_float(VI.speech()["b"])[:20000]
    e.set_graphs(False)
    eager, _ = e.convert(wav, 2, 8, seed=11)
    e.set_graphs(True)
    r0 = e.graph_replays()
    first, _ = e.convert(wav, 2, 8, seed=11)                     # eager run + capture
    second, _ = e.convert(wav, 2, 8, seed=11)                    # replay
    assert e.graph_replays() > r0
    assert np.array_equal(first, eager) and np.array_equal(second, eager)


def test_same_seed_same_output():
    e = _engine("mel", 0)
    wav = VI.wav_float(VI.speech()["b"])[:12000]
    a, _ = e.convert(wav, 1, 4, seed=5)
    b, _ = e.convert(wav, 1, 4, seed=5)
    c, _ = e.convert(wav, 1, 4, seed=6)
    d, _ = e.convert(wav, 1, 4, seed=6, noise_scale=0.0)
    f, _ = e.convert(wav, 1, 4, seed=7, noise_scale=0.0)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    assert np.array_equal(d, f)                                   # noise_scale 0: z = m, no seed dependence


def test_mode2_equals_mode1_bitwise():
    wav = VI.wav_float(VI.speech()["a"])
    I = _cfg("mel")["inter_channels"]
    eps = VI.eps_q("c0", I, len(wav) // 256).numpy()
    a, _ = _engine("mel", 1).convert(wav, 3, 7, noise=eps)
    b, _ = _engine("mel", 2).convert(wav, 3, 7, noise=eps)
    assert np.array_equal(a, b)


def _code(fn):
    from vosk_tts_b200.engine import VttsError
    with pytest.raises(VttsError) as ei:
        fn()
    return ei.value.code, str(ei.value)


def test_invalid_requests():
    e = _engine("mel", 0)
    wav = VI.wav_float(VI.speech()["b"])
    assert _code(lambda: e.convert(wav, 0, 200))[0] == -1                 # speaker id out of range
    assert _code(lambda: e.convert(wav, -1, 3))[0] == -1
    assert _code(lambda: e.convert(wav[:384], 0, 3))[0] == -1             # reflect padding needs > 384 samples
    o, fr = e.convert(wav[:385], 0, 3)
    assert int(fr[0]) == 1 and o.shape[1] == 256
    # output capacity
    lens = np.array([len(wav)], np.int64)
    out = np.zeros(256, np.float32)
    frames = np.zeros(1, np.int64)
    s = np.zeros(1, np.int64)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = e.lib.vtts_convert(e.h, P(wav), P(lens), 1, len(wav), P(s), P(s), 1.0, None, 0, 0, P(out), 256, P(frames))
    assert rc == -4


def test_invalid_models():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200 import onnx_weights
    from vosk_tts_b200.engine import Engine
    wav = VI.wav_float(VI.speech()["b"])
    # a TTS blob (no enc_q): the default pack, and a model read from model.onnx
    cfg, _, _ = _packed("lin")
    sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, VI.SEEDS["lin"], posterior=True))
    blob, man = weights.pack(sd, cfg)
    e = Engine(cfg, blob, man, precision=0)
    code, msg = _code(lambda: e.convert(wav, 0, 1))
    assert code == -1 and "enc_q" in msg
    e.close()
    path = os.path.join(GR.GOLDEN, "tiny_model.onnx")
    ocfg = onnx_weights.config_from_onnx(path)
    oblob, oman = weights.pack(onnx_weights.state_dict_from_onnx(path), ocfg)
    e = Engine(ocfg, oblob, oman, precision=0)
    code, msg = _code(lambda: e.convert(wav, 0, 1))
    assert code == -1 and "enc_q" in msg
    e.close()
    # single-speaker model
    c1 = copy.deepcopy(cfg)
    c1["n_speakers"] = 0
    sd1 = weights.fold_weight_norm(synthetic.make_random_checkpoint(c1, 3, posterior=True))
    b1, m1 = weights.pack(sd1, c1, posterior=True)
    e = Engine(c1, b1, m1, precision=0)
    assert _code(lambda: e.convert(wav, 0, 0))[0] == -1
    e.close()
    # odd flow count (checked before anything else: the packer refuses to add enc_q to such a model)
    c3 = copy.deepcopy(cfg)
    c3["flow_n_flows"] = 3
    b3, m3 = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(c3, 3)), c3)
    e = Engine(c3, b3, m3, precision=0)
    code, msg = _code(lambda: e.convert(wav, 0, 1))
    assert code == -1 and "flow_n_flows" in msg
    e.close()
