"""QuickVC conversion on the GPU (vtts_quickvc_convert) against the reference's SynthesizerTrn.infer
(tests/golden/ref_quickvc_convert.npz) and the float64 oracle, in precision modes 0 and 1."""
import ctypes as C

import numpy as np
import pytest

import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from oracle import quickvc_convert_oracle as O
from vosk_tts_b200 import weights

pytestmark = pytest.mark.gpu

REF = np.load(QI.GOLDEN + "/ref_quickvc_convert.npz")
CASES = [("T%d" % T, i, T) for i, (T, _) in enumerate(QC.CASES)]
_ENGINES = {}
_FOLDED = {}


def _folded():
    if not _FOLDED:
        _FOLDED["sd"] = weights.fold_weight_norm(QC.model())
    return _FOLDED["sd"]


def _engine(precision):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    if precision not in _ENGINES:
        cfg = QI.config()
        blob, man = weights.pack_quickvc(_folded(), cfg)
        _ENGINES[precision] = Engine(cfg, blob, man, device=0, precision=precision)
    return _ENGINES[precision]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


@pytest.mark.parametrize("precision", [0, 1])
def test_matches_reference(precision):
    """Waveform within 1e-3 of the reference on every case (z_p and z from the debug buffers within 1e-4 / 1e-3)."""
    eng = _engine(precision)
    worst = {}
    eng.debug_flags(1)
    try:
        for case, i, T in CASES:
            wav, frames = eng.quickvc_convert(QC.units(T, i), REF[case + "/g"], noise=QC.eps(T, i)[None])
            assert frames[0] == T and wav.shape == (1, 320 * T)
            o = REF[case + "/o"]
            err = float(np.abs(wav[0] - o).max())
            keep = QC.kept_frames(T)
            zp = eng.debug_read("vc_z").reshape(-1, 192)[:T].T[:, keep]
            z = eng.debug_read("vc_z_hat").reshape(-1, 192)[:T].T[:, keep]
            ezp, ez = float(np.abs(zp - REF[case + "/z_p"]).max()), float(np.abs(z - REF[case + "/z"]).max())
            worst[case] = (err, ezp, ez)
            assert err < 1e-3 and ezp < 1e-4 and ez < 1e-3, (case, err, ezp, ez)
    finally:
        eng.debug_flags(0)
    print("precision %d: max |wav - ref|, |z_p - ref|, |z - ref| per case: %s" % (precision, worst))


@pytest.mark.parametrize("precision", [0, 1])
def test_ragged_batch_equals_single_clips(precision):
    eng = _engine(precision)
    clips = [QC.units(T, i) for _, i, T in CASES]
    Tm = max(T for _, _, T in CASES)
    noise = np.zeros((len(CASES), 192, Tm), np.float32)
    g = np.stack([REF[c + "/g"] for c, _, _ in CASES])
    for b, (_, i, T) in enumerate(CASES):
        noise[b, :, :T] = QC.eps(T, i)
    wav, frames = eng.quickvc_convert(clips, g, noise=noise)
    assert list(frames) == [T for _, _, T in CASES]
    for b, (case, i, T) in enumerate(CASES):
        one, _ = eng.quickvc_convert(clips[b], g[b], noise=noise[b:b + 1, :, :T])
        assert float(np.abs(wav[b, :320 * T] - one[0]).max()) < 1e-4, case
        assert not np.any(wav[b, 320 * T:])


@pytest.mark.parametrize("precision", [0, 1])
def test_graph_replay_equals_eager(precision):
    eng = _engine(precision)
    u, g, e = QC.units(37, 2), REF["T37/g"], QC.eps(37, 2)[None]
    eng.set_graphs(False)
    try:
        eager, _ = eng.quickvc_convert(u, g, noise=e)
    finally:
        eng.set_graphs(True)
    r0 = eng.graph_replays()
    first, _ = eng.quickvc_convert(u, g, noise=e)
    again, _ = eng.quickvc_convert(u, g, noise=e)
    assert eng.graph_replays() > r0
    assert np.array_equal(eager, first) and np.array_equal(eager, again)


@pytest.mark.parametrize("precision", [0, 1])
def test_noise(precision):
    eng = _engine(precision)
    u, g = QC.units(37, 2), REF["T37/g"]
    a, _ = eng.quickvc_convert(u, g, noise_scale=0.0, seed=1)
    b, _ = eng.quickvc_convert(u, g, noise_scale=0.0, seed=2)
    c, _ = eng.quickvc_convert(u, g, noise=np.zeros((1, 192, 37), np.float32))
    assert np.array_equal(a, b) and np.array_equal(a, c)
    d, _ = eng.quickvc_convert(u, g, seed=1)
    e, _ = eng.quickvc_convert(u, g, seed=1)
    f, _ = eng.quickvc_convert(u, g, seed=2)
    assert np.array_equal(d, e) and not np.array_equal(d, f) and not np.array_equal(a, d)
    with pytest.raises(ValueError, match="noise"):          # the engine reads inter_channels rows of every clip
        eng.quickvc_convert(u, g, noise=np.zeros((1, 191, 37), np.float32))


HALO = 32


@pytest.mark.parametrize("precision", [0, 1])
def test_long_clip_against_oracle(precision):
    """A 3000-frame (60 s) clip: z over every frame, the audio of the first and last 2 s (100 frames).  The oracle decodes
    each 100-frame window with HALO = 32 frames of z on its inner side.  The decoder's receptive field is under 24 frames
    each way: conv_pre (3 frames), the first upsampler (16 taps at rate 5: 2 frames), the first MRF (ResBlock1 k=11 with
    dilations 1, 3, 5: 5 + 15 + 25 + 3 * 5 = 60 samples at rate 5, 12 frames), the second upsampler and MRF (1 + 3 frames),
    conv_post (7 taps at rate 20) and the inverse STFT with its 63-tap filter (both under a frame)."""
    eng = _engine(precision)
    T = 3000
    u, e, g = QC.units(T, 7), QC.eps(T, 7), REF["T250/g"]
    eng.debug_flags(1)
    try:
        wav, _ = eng.quickvc_convert(u, g, noise=e[None])
        z = eng.debug_read("vc_z_hat").reshape(-1, 192)[:T].T
    finally:
        eng.debug_flags(0)
    sd = O.as_float64(_folded())
    cfg = QI.config()
    _, _, z_p = O.content_encoder(u, sd, cfg, e)
    z_ref = O.flow_reverse(z_p, g, sd, cfg)
    ez = float(np.abs(z - z_ref).max())
    W = 100
    head = O.decode(z_ref[:, :W + HALO], g, sd, cfg)[:320 * W]
    tail = O.decode(z_ref[:, T - W - HALO:], g, sd, cfg)[-320 * W:]
    eh, et = float(np.abs(wav[0, :320 * W] - head).max()), float(np.abs(wav[0, -320 * W:] - tail).max())
    print("precision %d, 3000 frames: max |z - oracle| %.2e, audio first 2 s %.2e, last 2 s %.2e" % (precision, ez, eh, et))
    assert ez < 1e-3 and eh < 1e-3 and et < 1e-3


def _raw(eng, units, lengths, B, ld, g, noise=None, noise_ld=0, out_ld=None):
    out_ld = 320 * ld if out_ld is None else out_ld
    wav = np.zeros((max(B, 1), max(out_ld, 1)), np.float32)
    frames = np.zeros(max(B, 1), np.int64)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    rc = eng.lib.vtts_quickvc_convert(eng.h, p(units), p(lengths), B, ld, p(g), 1.0, p(noise), noise_ld, 0, p(wav), out_ld, p(frames))
    return rc, eng.lib.vtts_last_error(eng.h).decode()


def test_refusals():
    eng = _engine(0)
    u = np.zeros((2, 10, 768), np.float32)
    g = np.zeros((2, 256), np.float32)
    ln = lambda *v: np.array(v, np.int64)
    assert _raw(eng, u, ln(10, 10), 2, 10, g)[0] == 0
    assert _raw(eng, u, ln(10, 10), 0, 10, g)[0] == -1
    assert _raw(eng, u, ln(0, 10), 2, 10, g)[0] == -1
    assert _raw(eng, u, ln(10, 11), 2, 10, g)[0] == -1
    rc, msg = _raw(eng, u, ln(10, 10), 2, 10, None)
    assert rc == -1 and "g" in msg
    rc, msg = _raw(eng, u, ln(10, 10), 2, 10, g, out_ld=320 * 10 - 1)
    assert rc == -4 and "out_ld" in msg
    rc, msg = _raw(eng, u, ln(10, 10), 2, 10, g, noise=np.zeros((2, 192, 9), np.float32), noise_ld=9)
    assert rc == -4 and "noise" in msg


def test_speaker_encoder_only_blob_refuses_conversion():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine, VttsError
    cfg = QI.config()
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QI.speaker_encoder()), cfg)
    eng = Engine(cfg, blob, man, device=0, precision=1)
    try:
        g = eng.speaker_embedding(QI.wav_float(QI.targets()["short"]))
        assert abs(float(np.linalg.norm(g)) - 1.0) < 0.2
        with pytest.raises(VttsError, match="speaker encoder"):
            eng.quickvc_convert(QC.units(5, 0), g[0])
    finally:
        eng.close()


def test_vits2_engine_refuses():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200 import config as Cf, synthetic
    from vosk_tts_b200.engine import Engine, VttsError
    cfg = Cf.DEFAULT_CONFIG
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234)), cfg, precision=0)
    eng = Engine(cfg, blob, man, device=0, precision=0)
    try:
        eng.cfg = dict(cfg, gin_channels=256)
        with pytest.raises(VttsError, match="QuickVC"):
            eng.quickvc_convert(QC.units(5, 0), np.zeros(256, np.float32))
    finally:
        eng.close()


@pytest.mark.parametrize("precision", [2, 3])
def test_modes_2_and_3_run_as_mode_1(precision):
    """Modes 2 and 3 differ from mode 1 only in the VITS2 text encoder, which QuickVC has none of: bit for bit mode 1."""
    eng = _engine(precision)
    u, g, e = QC.units(37, 2), REF["T37/g"], QC.eps(37, 2)[None]
    a, _ = eng.quickvc_convert(u, g, noise=e)
    b, _ = _engine(1).quickvc_convert(u, g, noise=e)
    assert np.array_equal(a, b)
