"""CPU restatement of SynthesizerTrn.voice_conversion (training/vits2/models.py:1710-1718) and of the spectrogram front end
it is fed with (mel_processing.py:53-125), in the op order of the reference lines cited per function.  Shares the flow,
encoder and decoder restatements of ``vits_oracle``; pinned to the unmodified reference by
tests/test_voice_conversion_host.py through tests/golden/ref_voice_conversion.npz (oracle/make_golden_vc.py)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.vits_oracle import conv, decoder_hifigan, decoder_mb_istft, encoder, flow_reverse, sequence_mask, wn


# --------------------------------------------------------------------------- voice conversion
def spectrogram(y, n_fft, hop, win):
    """spectrogram_torch (mel_processing.py:53-77), center=False: y float [B, L] -> [B, n_fft//2+1, frames]."""
    pad = int((n_fft - hop) / 2)
    y = F.pad(y.unsqueeze(1), (pad, pad), mode="reflect").squeeze(1)
    spec = torch.stft(y, n_fft, hop_length=hop, win_length=win, window=torch.hann_window(win).to(y.dtype), center=False,
                      pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
    spec = torch.view_as_real(spec)
    return torch.sqrt(spec.pow(2).sum(-1) + 1e-6)


def mel_basis(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    """librosa.filters.mel with its defaults (Slaney mel scale and Slaney area normalisation), float64 -> float32."""
    fmax = sr / 2.0 if fmax is None else float(fmax)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0

    def hz_to_mel(f):
        return min_log_mel + math.log(f / min_log_hz) / logstep if f >= min_log_hz else f / f_sp

    m = np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2)
    mel_f = np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)
    freqs = np.linspace(0.0, sr / 2.0, n_fft // 2 + 1)
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - freqs[None, :]
    weights = np.zeros((n_mels, n_fft // 2 + 1))
    for i in range(n_mels):
        weights[i] = np.maximum(0.0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


def mel_spectrogram(y, n_fft, n_mels, sr, hop, win, fmin, fmax):
    """mel_spectrogram_torch (mel_processing.py:93-125): log(clamp(mel @ |STFT|, 1e-5))."""
    spec = spectrogram(y, n_fft, hop, win)
    mel = torch.matmul(torch.from_numpy(mel_basis(sr, n_fft, n_mels, fmin, fmax)).to(spec.dtype), spec)
    return torch.log(torch.clamp(mel, min=1e-5))


def _wn_stack(x, x_mask, g, w, p, H, ks, dil_rate, nl):
    """modules.py:148-176 for any layer count (weight norm folded)."""
    out = torch.zeros_like(x)
    gc = conv(g, w, p + ".cond_layer") if g is not None else None
    for i in range(nl):
        dil = dil_rate ** i
        x_in = conv(x, w, "%s.in_layers.%d" % (p, i), dilation=dil, padding=int((ks * dil - dil) / 2))
        if gc is not None:
            x_in = x_in + gc[:, i * 2 * H:(i + 1) * 2 * H, :]
        acts = torch.tanh(x_in[:, :H]) * torch.sigmoid(x_in[:, H:])
        rs = conv(acts, w, "%s.res_skip_layers.%d" % (p, i))
        if i < nl - 1:
            x = (x + rs[:, :H]) * x_mask
            out = out + rs[:, H:]
        else:
            out = out + rs
    return out * x_mask


def posterior_encoder(y, y_lengths, g, w, eps):
    """PosteriorEncoder.forward (models.py:836-842: 1x1 pre, 16-layer WN with kernel 5, 1x1 proj); eps [B, inter, >=T]
    replaces the torch.randn_like of :841."""
    H = w["enc_q.pre.weight"].shape[0]
    x_mask = sequence_mask(y_lengths, y.size(2)).unsqueeze(1).to(y.dtype)
    x = conv(y, w, "enc_q.pre") * x_mask
    x = _wn_stack(x, x_mask, g, w, "enc_q.enc", H, 5, 1, 16)
    stats = conv(x, w, "enc_q.proj") * x_mask
    m, logs = torch.split(stats, stats.shape[1] // 2, dim=1)
    z = (m + eps[:, :, : y.size(2)] * torch.exp(logs)) * x_mask
    return z, m, logs, x_mask


def coupling_forward(x, x_mask, g, w, p, cfg):
    """models.py:374-389 (mean_only) with reverse=False: x1 <- m + x1 * mask."""
    half = cfg["inter_channels"] // 2
    x0, x1 = x[:, :half], x[:, half:]
    h = conv(x0, w, p + ".pre") * x_mask
    if cfg["use_transformer_flows"]:
        h = h + encoder(h * x_mask, x_mask, w, p + ".pre_transformer", 1, 2, cfg["flow_kernel_size"], cfg["window_size"])
    h = wn(h, x_mask, g, w, p + ".enc", cfg)
    m = conv(h, w, p + ".post") * x_mask
    x1 = m + x1 * x_mask
    return torch.cat([x0, x1], 1)


def flow_forward(z, y_mask, g, w, cfg):
    """models.py:750-753: [L1, Flip, ..., Ln, Flip] in order."""
    for f in range(cfg["flow_n_flows"]):
        z = coupling_forward(z, y_mask, g, w, "flow.flows.%d" % (2 * f), cfg)
        z = torch.flip(z, [1])
    return z


def voice_conversion(w, cfg, y, y_lengths, sid_src, sid_tgt, eps_q):
    """SynthesizerTrn.voice_conversion (models.py:1710-1718) on features y [B, spec_channels, T]; eps_q [B, inter, >=T]."""
    g_src = F.embedding(sid_src, w["emb_g.weight"]).unsqueeze(-1)
    g_tgt = F.embedding(sid_tgt, w["emb_g.weight"]).unsqueeze(-1)
    z, m_q, logs_q, y_mask = posterior_encoder(y, y_lengths, g_src, w, eps_q)
    z_p = flow_forward(z, y_mask, g_src, w, cfg)
    z_hat = flow_reverse(z_p, y_mask, g_tgt, w, cfg)
    zin = z_hat * y_mask
    if cfg["decoder"] in ("mb_istft", "ms_istft", "istft"):
        o, o_mb = decoder_mb_istft(zin, w, cfg)
    else:
        o, o_mb = decoder_hifigan(zin, w, cfg, g_tgt)
    return dict(o_hat=o, o_hat_mb=o_mb, y_mask=y_mask, z=z, z_p=z_p, z_hat=z_hat, m_q=m_q, logs_q=logs_q)
