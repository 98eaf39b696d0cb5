"""CPU: the float64 references of tests/spectral_ref.py pinned to the oracles and torch, the envelope claim of
istft_pqmf_kernel, and the sharpness of every bound: each plausible kernel mistake must break its bound on an input the GPU
tests (test_gpu_spectral.py) run."""
import numpy as np
import pytest
import torch

import golden_ref as GR
import spectral_ref as S
from oracle import quickvc_convert_oracle as qo, vc_oracle, vits_oracle as vo
from vosk_tts_b200 import config as C, weights


@pytest.mark.parametrize("nfft,hop", [(1024, 256), (1280, 320), (64, 16), (1024, 512), (2048, 512)])
@pytest.mark.parametrize("kind", ["noise", "tone", "nyquist"])
def test_magnitude_matches_torch_stft(nfft, hop, kind):
    rng = np.random.default_rng(nfft + hop)
    for L in [S.min_clip(nfft, hop), S.length_for_frames(3, nfft, hop, hop - 1), 5 * nfft + 7]:
        x = S.signal(kind, L, nfft, rng)
        mag, bound = S.magnitude(x, nfft, hop)
        ref = vc_oracle.spectrogram(torch.from_numpy(x.astype(np.float64))[None], nfft, hop, nfft)[0].numpy().T
        assert mag.shape == ref.shape and mag.shape[0] == S.frames_of(L, nfft, hop) >= 1
        # (the oracle's window is torch.hann_window's fp32 one: within the bound, which covers fp32 windowed basis values)
        assert np.all(np.abs(mag - ref) <= bound)


def test_min_clip_is_where_torch_stft_starts_to_frame():
    for nfft, hop in [(1024, 256), (1024, 512), (1280, 320), (64, 16), (3072, 768)]:
        lo = S.min_clip(nfft, hop)
        pad = (nfft - hop) // 2
        assert S.frames_of(lo, nfft, hop) == 1
        x = torch.zeros(1, lo - 1, dtype=torch.float64)
        if lo - 1 > pad:        # long enough for the reflect padding, too short for one frame: torch refuses it
            with pytest.raises(RuntimeError):
                vc_oracle.spectrogram(x, nfft, hop, nfft)


@pytest.mark.parametrize("sr,nfft,hop", [(22050, 1024, 256), (16000, 1280, 320), (22050, 64, 16)])
def test_log_mel_matches_oracle(sr, nfft, hop):
    rng = np.random.default_rng(5)
    x = np.concatenate([S.signal("noise", 3000, nfft, rng), np.zeros(3000, np.float32)])
    mag, _ = S.magnitude(x, nfft, hop)
    fb = weights.mel_basis(sr, nfft, 80, 0.0, None)
    v, lo, hi = S.log_mel(mag, fb)
    ref = vc_oracle.mel_spectrogram(torch.from_numpy(x.astype(np.float64))[None], nfft, 80, sr, hop, nfft, 0.0, None)[0].numpy().T
    assert np.abs(v - ref).max() < 1e-5
    assert np.all(lo <= v) and np.all(v <= hi)


def _post_tensor(P):
    return torch.from_numpy(P.T[None].copy())


@pytest.mark.parametrize("flag,kind", GR.DECODER_VARIANTS)
def test_tail_matches_decoder_oracle(flag, kind, monkeypatch):
    cfg = C.from_training_json(GR.training_json(flag), n_vocab=GR.N_VOCAB)
    sb = 1 if kind == "istft" else cfg["subbands"]
    rng = np.random.default_rng(3)
    P = S.post_values("normal", 16 * 5 + 1, sb * 18, rng)
    bank = {"mb_istft": weights.pqmf_synthesis_filter(sb), "istft": np.eye(1, 63, 31, dtype=np.float32),
            "ms_istft": rng.standard_normal((sb, 63)).astype(np.float32) * 0.1}[kind]
    monkeypatch.setattr(vo, "decoder_trunk", lambda z, w, cfg: torch.zeros(1, 1, 2))
    monkeypatch.setattr(vo, "conv", lambda x, w, name, padding=0: _post_tensor(P))
    w = {"dec.multistream_conv_post.weight": torch.from_numpy(bank[None])}
    with torch.no_grad():
        wav, _ = vo.decoder_mb_istft(None, w, dict(cfg, decoder=kind))
    wav = wav.reshape(-1).numpy().astype(np.float64)
    out, bound = S.tail(P, weights.istft_inverse_basis(16, 4), bank, 4)
    assert wav.shape == out.shape
    assert np.abs(wav - out).max() <= 2e-5 * np.abs(out).max() + bound.max()


def test_tail_matches_torch_istft():
    """QuickVC's TorchSTFT.inverse (torch.istft, divided by the window envelope) per band, then the multistream filter."""
    rng = np.random.default_rng(4)
    sb, L1 = 4, 20 * 3 + 1
    P = S.post_values("normal", L1, sb * 18, rng)
    bank = rng.standard_normal((sb, 63)).astype(np.float32) * 0.1
    p = torch.from_numpy(P.astype(np.float64)).reshape(L1, sb, 18).permute(1, 2, 0)
    y = qo.istft(torch.exp(p[:, :9]), np.pi * torch.sin(p[:, 9:]), 16, 4)               # [sb][4 (L1 - 1)]
    up = torch.zeros(1, sb, sb * y.shape[1], dtype=torch.float64)
    up[0, :, ::sb] = sb * y
    ref = torch.nn.functional.conv1d(up, torch.from_numpy(bank[:, None].astype(np.float64)).reshape(1, sb, 63), padding=31)[0, 0].numpy()
    out, bound = S.tail(P, weights.istft_inverse_basis(16, 4), bank, 4, w2=weights.hann_squared(16))
    # (the blob's basis is fp32, torch's window float64: within the bound, which covers the fp32 operands)
    assert np.all(np.abs(ref - out) <= bound)


def test_envelope_is_at_least_1_25_on_every_kept_sample():
    w2 = weights.hann_squared(16).astype(np.float64)
    for L1 in range(2, 70):
        env = S.envelope(L1, w2, 4)
        assert env.min() >= 1.25 - 1e-12 and len(env) == 4 * (L1 - 1)
    assert abs(S.envelope(40, w2, 4)[20] - 1.5) < 1e-12


# ---------------------------------------------------------------------------------------------------- sharpness
def _breaks(mut, ref, bound):
    return bool(np.any(np.abs(mut - ref) > bound))


@pytest.mark.parametrize("mutate,kind", [("symmetric", "noise"), ("hop+1", "noise"), ("swap_dc_nyquist", "dc"),
                                         ("swap_dc_nyquist", "nyquist"), ("no_eps", "silence")])
def test_magnitude_bound_catches(mutate, kind):
    for _, nfft, hop, _, _ in S.FRONT_CONFIGS:
        rng = np.random.default_rng(0)
        x = S.signal(kind, S.length_for_frames(65, nfft, hop), nfft, rng)
        ref, bound = S.magnitude(x, nfft, hop)
        mut, _ = S.magnitude(x, nfft, hop, mutate=mutate)
        assert _breaks(mut, ref, bound), (mutate, kind, nfft, hop)


def test_log_mel_bound_catches_a_floor_at_1e_6():
    """Silence: every magnitude is sqrt(1e-6); the 64-point configuration has mel filters between bins (empty), whose sum is
    exactly 0 and so at the floor."""
    mag = np.full((3, 33), np.float32(np.sqrt(np.float32(1e-6))), np.float32)
    fb = weights.mel_basis(22050, 64, 80, 0.0, None)
    _, lo, hi = S.log_mel(mag, fb)
    mut, _, _ = S.log_mel(mag, fb, floor=float(np.float32(1e-6)))
    assert np.any((mut < lo) | (mut > hi))
    assert np.any(fb.sum(1) == 0)


@pytest.mark.parametrize("mutate", ["drop_last_frame", "pqmf_shift", "no_envelope"])
@pytest.mark.parametrize("Ty", [1, 17])
def test_tail_bound_catches(mutate, Ty):
    rng = np.random.default_rng(Ty)
    sb, up = 4, 16
    P = S.post_values("normal", Ty * up + 1, sb * 18, rng)
    bank = weights.pqmf_synthesis_filter(sb)
    w2 = weights.hann_squared(16)
    ref, bound = S.tail(P, weights.istft_inverse_basis(16, 4), bank, 4, w2=w2)
    mut, _ = S.tail(P, weights.istft_inverse_basis(16, 4), bank, 4, w2=w2, mutate=mutate)
    assert _breaks(mut, ref, bound)
    if mutate == "drop_last_frame":          # only the last samples change
        assert not _breaks(mut[:-16 * sb], ref[:-16 * sb], bound[:-16 * sb])


def test_tail_bound_is_far_below_the_waveform():
    rng = np.random.default_rng(9)
    P = S.post_values("normal", 16 * 64 + 1, 72, rng)
    out, bound = S.tail(P, weights.istft_inverse_basis(16, 4), weights.pqmf_synthesis_filter(4), 4)
    assert np.median(bound / (np.abs(out).max())) < 1e-4
