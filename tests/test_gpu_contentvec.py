"""ContentVec on the GPU (vtts_content_units, vtts_quickvc_convert_wav) against the float64 oracle, which matches the reference
HubertModel (tests/test_contentvec_host.py), in precision modes 0 and 1."""
import ctypes as C

import numpy as np
import pytest
import torch

import contentvec_inputs as CI
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from oracle import contentvec_oracle as O
from vosk_tts_b200 import weights

pytestmark = pytest.mark.gpu

_ENGINES = {}
_REF = {}


def _cfg():
    cfg = dict(QI.config())
    cfg["contentvec"] = CI.cv()
    return cfg


def _engine(precision):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    if precision not in _ENGINES:
        blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
        _ENGINES[precision] = Engine(_cfg(), blob, man, device=0, precision=precision)
    return _ENGINES[precision]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


def _oracle(x, stages=None):
    return O.contentvec_units(CI.folded(), CI.cv(), x, torch.float64, stages).numpy()


def _ref(name, x):
    if name not in _REF:
        st = {}
        u = _oracle(x, st)
        _REF[name] = (u, st["feat"].numpy(), st["enc_in"].numpy())
    return _REF[name]


CLIPS = [(n, "s%d" % n) for n in CI.LENGTHS + (CI.LONG,)]


@pytest.mark.parametrize("precision", [0, 1])
def test_units_match_oracle(precision):
    """Units within 1e-3 of float64; the feature encoder's output and the transformer's input within 1e-3 too."""
    eng = _engine(precision)
    eng.debug_flags(1)
    try:
        for n, name in CLIPS:
            x = CI.speech(n, n)
            u_ref, f_ref, e_ref = _ref(name, x)
            units, frames = eng.content_units(x)
            T = u_ref.shape[0]
            assert frames[0] == T
            feat = eng.debug_read("cv_feat").reshape(-1, 512)[:T]
            enc_in = eng.debug_read("cv_enc_in").reshape(-1, 768)[:T]
            errs = (float(np.abs(units[0, :T] - u_ref).max()), float(np.abs(feat - f_ref).max()), float(np.abs(enc_in - e_ref).max()))
            print("mode %d, %d samples, %d frames: units %.3g, feature encoder %.3g, encoder input %.3g" % ((precision, n, T) + errs))
            assert max(errs) < 1e-3, errs
    finally:
        eng.debug_flags(0)


@pytest.mark.parametrize("precision", [0, 1])
def test_groupnorm_variance_on_dc_offset(precision):
    """On a clip with a DC offset the error stays that of a speech-like clip: the whole-clip GroupNorm's variance is centred."""
    eng = _engine(precision)
    n = 48000
    sp, dc = CI.speech(n, 7), CI.dc_offset(n, 7)
    e_sp = float(np.abs(eng.content_units(sp)[0][0] - _oracle(sp)).max())
    e_dc = float(np.abs(eng.content_units(dc)[0][0] - _oracle(dc)).max())
    print("mode %d: speech-like %.3g, DC offset %.3g" % (precision, e_sp, e_dc))
    assert e_dc <= 2 * e_sp and e_dc < 5.3e-4


def tone_3200(n, seed):
    """0.5 * cos(2 pi 3200 t) + 0.001 * speech: the 3200 Hz tone repeats every 5 samples, the layer-0 stride, so every channel
    gets a constant offset that the clip's sample mean (about 0) does not remove, 500 times the size of its signal."""
    k = np.arange(n)
    return (0.5 * np.cos(2 * np.pi * k / 5) + 0.001 * CI.speech(n, seed)).astype(np.float32)


@pytest.mark.parametrize("precision", [0, 1])
def test_groupnorm_variance_is_centred(precision):
    """Layer 0's per-channel variance on the device against float64, on a clip whose channels sit far from zero: relative error
    below 1e-4, where a one-pass E[v^2] - E[v]^2 in fp32 loses about 1e-2 (eps * (offset / signal)^2)."""
    eng = _engine(precision)
    n = 48000
    x = tone_3200(n, 8)
    eng.debug_flags(1)
    try:
        _, frames = eng.content_units(x)
        sq = eng.debug_read("cv_gn_sq").reshape(-1, 512)
    finally:
        eng.debug_flags(0)
    w0 = CI.folded()["feature_extractor.conv_layers.0.conv.weight"].double()
    v = torch.nn.functional.conv1d(torch.from_numpy(x).double()[None, None], w0, stride=5)[0]       # [512, L0]
    L0 = v.shape[1]
    nch = (L0 + 255) // 256
    var_gpu = sq[:nch].astype(np.float64).sum(0) / L0
    var_ref = v.var(dim=1, unbiased=False).numpy()
    offset = float((v.mean(dim=1).abs() / v.std(dim=1)).median())
    rel = float(np.abs(var_gpu / var_ref - 1).max())
    print("mode %d: channel offset / std (median) %.0f, variance relative error %.3g" % (precision, offset, rel))
    assert offset > 100 and rel < 1e-4


@pytest.mark.parametrize("precision", [0, 1])
def test_convert_wav_matches_reference(precision):
    """Waveform to waveform within 1e-3 of reference ContentVec followed by the reference QuickVC infer (same noise)."""
    eng = _engine(precision)
    ref = np.load(CI.GOLDEN + "/ref_contentvec.npz")
    for i, (n, _) in enumerate(CI.E2E):
        x = CI.speech(n, 500 + i)
        o = ref["e2e%d/o" % i]
        T = o.size // 320
        wav, frames = eng.quickvc_convert_wav(x, ref["e2e%d/g" % i], noise=QC.eps(T, 500 + i)[None])
        err = float(np.abs(wav[0, :o.size] - o).max())
        print("mode %d, e2e %d (%d frames): %.3g, peak %.3g" % (precision, i, T, err, float(np.abs(o).max())))
        assert frames[0] == T and err < 1e-3


def test_mode_1_runs_the_tensor_core_path():
    x = CI.speech(24000, 9)
    u0, u1 = _engine(0).content_units(x)[0], _engine(1).content_units(x)[0]
    assert not np.array_equal(u0, u1) and np.abs(u0 - u1).max() < 1e-3


@pytest.mark.parametrize("precision", [0, 1])
def test_ragged_batch_equals_single(precision):
    eng = _engine(precision)
    ns = [400, 16000, 160000, 719, 52345]
    clips = [CI.speech(n, 100 + i) for i, n in enumerate(ns)]
    units, frames = eng.content_units(clips)
    for b, x in enumerate(clips):
        one, f1 = eng.content_units(x)
        assert frames[b] == f1[0]
        T = int(f1[0])
        err = float(np.abs(units[b, :T] - one[0, :T]).max())
        assert err < 1e-4, (b, err)
        assert not units[b, T:].any()


@pytest.mark.parametrize("precision", [0, 1])
def test_long_clip(precision):
    """60 s (2999 frames) against float64 on the frames at both ends and in the middle."""
    eng = _engine(precision)
    x = CI.speech(960000, 60)
    u_ref = _oracle(x)
    units, frames = eng.content_units(x)
    assert frames[0] == 2999 == u_ref.shape[0]
    keep = CI.kept_frames(2999)
    err = float(np.abs(units[0][keep] - u_ref[keep]).max())
    print("mode %d, 60 s: %.3g" % (precision, err))
    assert err < 1e-3


@pytest.mark.parametrize("precision", [0, 1])
def test_graph_replay_equals_eager(precision):
    eng = _engine(precision)
    x = [CI.speech(33333, 5), CI.speech(20000, 6)]
    a = eng.content_units(x)[0]
    b = eng.content_units(x)[0]          # replays the graph captured behind the first call
    eng.set_graphs(False)
    try:
        c = eng.content_units(x)[0]
    finally:
        eng.set_graphs(True)
    assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.parametrize("precision", [0, 1])
def test_convert_wav_equals_two_calls(precision):
    """One call equals units then conversion, bit for bit, for the same noise."""
    eng = _engine(precision)
    clips = [CI.speech(32000, 11), CI.speech(9000, 12)]
    g = np.stack([np.load(QI.GOLDEN + "/ref_quickvc_convert.npz")["T37/g"]] * 2)
    units, frames = eng.content_units(clips)
    T = int(frames.max())
    noise = np.random.RandomState(3).randn(2, 192, T).astype(np.float32)
    w2, f2 = eng.quickvc_convert([units[b, :frames[b]] for b in range(2)], g, noise=noise)
    w1, f1 = eng.quickvc_convert_wav(clips, g, noise=noise)
    assert np.array_equal(f1, f2) and np.array_equal(w1, w2)
    assert np.abs(w1).max() > 0.01


def test_modes_2_3_equal_mode_1():
    from vosk_tts_b200.engine import Engine
    x = CI.speech(24000, 9)
    u1 = _engine(1).content_units(x)[0]
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    for p in (2, 3):
        e = Engine(_cfg(), blob, man, device=0, precision=p)
        try:
            assert np.array_equal(e.content_units(x)[0], u1)
        finally:
            e.close()


def test_refusals():
    from vosk_tts_b200.engine import Engine, VttsError
    eng = _engine(0)
    with pytest.raises(VttsError) as ex:
        eng.content_units(np.zeros(399, np.float32))
    assert ex.value.code == -1 and "too short" in str(ex.value)
    wav = np.zeros((1, 16000), np.float32)
    lens = np.array([16000], np.int64)
    units = np.zeros((1, 10, 768), np.float32)
    fr = np.zeros(1, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert eng.lib.vtts_content_units(eng.h, p(wav), p(lens), 0, 16000, p(units), 10, p(fr)) == -1
    assert eng.lib.vtts_content_units(eng.h, p(wav), p(lens), 1, 16000, p(units), 10, p(fr)) == -4      # 49 frames > 10
    out = np.zeros((1, 320 * 49), np.float32)
    g = np.zeros((1, 256), np.float32)
    noise = np.zeros((1, 192, 10), np.float32)
    assert eng.lib.vtts_quickvc_convert_wav(eng.h, p(wav), p(lens), 1, 16000, p(g), 1.0, p(noise), 10, 0, p(out), out.shape[1], p(fr)) == -4
    assert eng.lib.vtts_quickvc_convert_wav(eng.h, p(wav), p(lens), 1, 16000, p(g), 1.0, None, 0, 0, p(out), 320 * 10, p(fr)) == -4
    # a blob without cv.*
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config())
    e = Engine(_cfg(), blob, man, device=0, precision=0)
    try:
        with pytest.raises(VttsError) as ex:
            e.content_units(wav)
        assert ex.value.code == -1 and "cv.*" in str(ex.value)
    finally:
        e.close()
    # conversion from waveforms on a speaker-encoder-only blob with ContentVec
    blob, man = weights.pack_quickvc(QI.speaker_encoder(), QI.config(), contentvec=CI.model())
    e = Engine(_cfg(), blob, man, device=0, precision=0)
    try:
        assert e.content_units(wav)[1][0] == 49
        with pytest.raises(VttsError) as ex:
            e.quickvc_convert_wav(wav, g)
        assert ex.value.code == -1
    finally:
        e.close()
