"""QuickVC speaker encoder on the GPU (vtts_speaker_embedding / _mel) against the reference's g (tests/golden/ref_quickvc.npz)
and the LSTM recurrence kernel alone against a float64 recurrence on the engine's own projected inputs."""
import numpy as np
import pytest

import quickvc_inputs as QI
from oracle import quickvc_oracle as O
from vosk_tts_b200 import weights

pytestmark = pytest.mark.gpu

REF = np.load(QI.GOLDEN + "/ref_quickvc.npz")
KEYS = [k for k, _, _, _ in QI.TARGETS]
_ENGINES = {}
U = 2.0 ** -24


def _engine(precision):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    if precision not in _ENGINES:
        cfg = QI.config()
        blob, man = weights.pack_quickvc(weights.fold_weight_norm(QI.speaker_encoder()), cfg)
        _ENGINES[precision] = Engine(cfg, blob, man, device=0, precision=precision)
    return _ENGINES[precision]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


def recurrence_bound(xp, whh, h_gpu):
    """float64 LSTM layer on the kernel's own inputs, teacher-forced: step t reads the kernel's h_{t-1} (h_gpu [T][G]) and
    the float64 c_{t-1}.  Returns that recurrence's h [T][G] and an elementwise bound on |h_gpu - h| [T][G].

    The kernel forms each gate pre-activation z_r = xp_r + sum_k W_rk h_k in fp32: a 32-term FMA chain per warp, then the
    8 warp partials and xp added in turn, at most K = 41 roundings deep, so with the same h the error is
    |dz_r| <= gamma_K (|xp_r| + sum_k |W_rk| |h_k|), gamma_K = K u / (1 - K u).  The gates follow through sigma' <= 1/4 and
    tanh' <= 1, each activation adding 4 u (expf / tanhf and the division).  The cell state is the only error carried from
    step to step: e_c <= |f| e_c + |c_{t-1}| df + |g| di + |i| dg + df e_c + di dg + 2 u (|f c| + |i g|), a contraction as
    |f| < 1; and h = o tanh(c) gives e_h <= |tanh c| do + (|o| + do) (e_c + 4 u) + u |h|."""
    xp = np.asarray(xp, np.float64)
    W = np.asarray(whh, np.float64)
    hg = np.asarray(h_gpu, np.float64)
    aW = np.abs(W)
    G = W.shape[1]
    K = 41
    gam = K * U / (1 - K * U)
    c, ec = np.zeros(G), np.zeros(G)
    H, E = np.zeros((xp.shape[0], G)), np.zeros((xp.shape[0], G))
    sg = lambda x: 1.0 / (1.0 + np.exp(-x))
    for t in range(xp.shape[0]):
        hp = hg[t - 1] if t else np.zeros(G)
        z = xp[t] + W @ hp
        dz = gam * (np.abs(xp[t]) + aW @ np.abs(hp))
        i, f, g, o = sg(z[:G]), sg(z[G:2 * G]), np.tanh(z[2 * G:3 * G]), sg(z[3 * G:])
        di, df, dg, do = dz[:G] / 4 + 4 * U, dz[G:2 * G] / 4 + 4 * U, dz[2 * G:3 * G] + 4 * U, dz[3 * G:] / 4 + 4 * U
        cn = f * c + i * g
        ec = f * ec + np.abs(c) * df + np.abs(g) * di + i * dg + df * ec + di * dg + 2 * U * (np.abs(f * c) + np.abs(i * g))
        c = cn
        tc = np.tanh(c)
        h = o * tc
        H[t] = h
        E[t] = np.abs(tc) * do + (o + do) * (ec + 4 * U) + U * np.abs(h)
    return H, E


def _slice_rows(frames):
    """(clip, start, length, first slice row) of every slice, packed as the engine packs them (8 rows between slices)."""
    out, off = [], 0
    for b, T in enumerate(frames):
        for s, L in O.slices(T):
            out.append((b, s, L, off))
            off += L + 8
    return out


def _check_recurrence(eng, frames, pick=None):
    sd = QI.speaker_encoder()
    fo = np.concatenate([[0], np.cumsum(np.asarray(frames) + 8)])[:-1]
    rows = _slice_rows(frames)
    sel = range(len(rows)) if pick is None else pick(len(rows))
    worst = widest = 0.0
    for l in range(3):
        x = eng.debug_read("spk_x%d" % l).reshape(-1, 1024)
        h = eng.debug_read("spk_h%d" % l).reshape(-1, 256)
        whh = sd["enc_spk.lstm.weight_hh_l%d" % l].numpy()
        for si in sel:
            b, s, L, off = rows[si]
            xr = fo[b] + s if l == 0 else off
            ref, bound = recurrence_bound(x[xr:xr + L], whh, h[off:off + L])
            err = np.abs(h[off:off + L] - ref)
            assert np.all(err <= bound), (l, si, float(err.max()), float(bound[err > bound].min()))
            assert bound.max() < 1e-3                      # h is in (-1, 1): the bound stays meaningful over the whole slice
            worst = max(worst, float((err / bound).max()))
            widest = max(widest, float(bound.max()))
    print("recurrence: largest error / bound = %.3g, largest bound %.3g" % (worst, widest))
    return worst


@pytest.mark.parametrize("precision", [0, 1])
def test_recurrence_kernel_alone(precision):
    """Every slicing case (T <= 128, 129, the 64-frame grid boundaries, long clips) in one ragged batch."""
    eng = _engine(precision)
    frames = [1, 81, 128, 129, 191, 192, 193, 431, 3000]
    rng = np.random.default_rng(7)
    mel = rng.normal(-4.0, 2.0, (len(frames), 80, max(frames))).astype(np.float32)
    eng.speaker_embedding_mel(mel, frames)
    _check_recurrence(eng, frames)


@pytest.mark.parametrize("precision", [0, 1])
def test_recurrence_many_clusters(precision):
    """64 clips of 431 frames: 384 slices, more clusters than fit the GPU at once, 8 sequences per cluster."""
    eng = _engine(precision)
    rng = np.random.default_rng(11)
    frames = [431] * 64
    mel = rng.normal(-4.0, 2.0, (64, 80, 431)).astype(np.float32)
    g = eng.speaker_embedding_mel(mel, frames)
    _check_recurrence(eng, frames, pick=lambda n: [0, 1, 7, 8, 100, 191, 200, n - 2, n - 1])
    for b in (0, 33, 63):
        g1 = eng.speaker_embedding_mel(mel[b:b + 1], frames[b:b + 1])
        assert np.array_equal(g1[0], g[b])


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("key", KEYS)
def test_g_matches_reference(precision, key):
    eng = _engine(precision)
    ref = REF[key + "/g"]
    g_mel = eng.speaker_embedding_mel(REF[key + "/mel"])[0]
    g_wav = eng.speaker_embedding(QI.wav_float(QI.targets()[key]))[0]
    print("%s: |g_mel - ref| %.3g, |g_wav - ref| %.3g" % (key, np.abs(g_mel - ref).max(), np.abs(g_wav - ref).max()))
    # measured: at most 1.8e-7 from either input, on g entries of up to 0.21
    assert np.abs(g_mel - ref).max() < 1e-6
    assert np.abs(g_wav - ref).max() < 1e-6
    fl = eng.debug_read("vc_spec").reshape(-1, 80)[:REF[key + "/mel"].shape[1]]
    assert np.abs(fl.T - REF[key + "/mel"]).max() < 2e-2


def test_ragged_targets_equal_single_clips():
    eng = _engine(1)
    t = QI.targets()
    wavs = [QI.wav_float(t[k]) for k in KEYS]
    L = max(w.size for w in wavs)
    batch = np.zeros((len(wavs), L), np.float32)
    for b, w in enumerate(wavs):
        batch[b, :w.size] = w
    g = eng.speaker_embedding(batch, [w.size for w in wavs])
    for b, w in enumerate(wavs):
        assert np.array_equal(eng.speaker_embedding(w)[0], g[b])
    assert np.array_equal(eng.speaker_embedding(batch, [w.size for w in wavs]), g)


def test_refusals():
    from vosk_tts_b200.engine import VttsError
    eng = _engine(0)
    with pytest.raises(VttsError) as e:
        eng.convert(np.zeros((1, 4096), np.float32), 0, 1)
    assert e.value.code == -1 and "QuickVC" in str(e.value)
    with pytest.raises(VttsError) as e:
        eng.durations(np.ones((1, 5), np.int64), [5], [0], (0.667, 1.0, 0.8))
    assert e.value.code == -1
    with pytest.raises(VttsError) as e:
        eng.speaker_embedding(np.zeros(400, np.float32))          # shorter than the reflect padding (480 samples)
    assert e.value.code == -1


def test_profiler_counts_the_projection_launches():
    """The conv profiler serves a QuickVC engine, and counts the layer-1/2 projections over the slices (not the clips)."""
    eng = _engine(0)
    frames = [81, 129, 431]
    mel = np.random.default_rng(3).normal(-4.0, 2.0, (3, 80, 431)).astype(np.float32)
    eng.speaker_embedding_mel(mel, frames)           # (warm)
    eng.profile(1)
    try:
        eng.speaker_embedding_mel(mel, frames)
        r = eng.profile_read()
    finally:
        eng.profile(0)
    rows = sum(L for T in frames for _, L in O.slices(T))
    assert r["conv_launches"] == 3
    assert r["conv_flops"] == 2.0 * sum(frames) * 80 * 1024 + 2 * 2.0 * rows * 256 * 1024


def test_vits2_engine_refuses_embedding():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200 import config as CF, synthetic
    from vosk_tts_b200.engine import Engine, VttsError
    cfg = CF.DEFAULT_CONFIG
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 1234)), cfg)
    eng = Engine(cfg, blob, man, device=0, precision=0)
    try:
        with pytest.raises(VttsError) as e:
            eng.speaker_embedding(np.zeros(16000, np.float32))
        assert e.value.code == -1 and "QuickVC" in str(e.value)
    finally:
        eng.close()
