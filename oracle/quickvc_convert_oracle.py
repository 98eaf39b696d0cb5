"""CPU restatement, in float64, of QuickVC's conversion: SynthesizerTrn.infer (vc/models.py:862-872) with g given -- the
content encoder enc_p, the reverse flow and the Multistream_iSTFT_Generator decoder (:416-501) with QuickVC's upsampling
pads (config.convt_pad), its conv_pre(z) + cond(g) and the torch.istft tail.  The WN stack, the coupling flow and the
resblocks are vits_oracle's (vc/modules.py restates them unchanged); the speaker encoder is quickvc_oracle's.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import vits_oracle as vo
from vosk_tts_b200.config import convt_pad

ENC_P_LAYERS, ENC_P_KERNEL = 16, 5          # PosteriorEncoder(768, I, H, 5, 1, 16) (models.py:825)


def as_float64(sd):
    """float64 tensors of a (folded) state dict; a dict that already is one is returned as it is."""
    return {k: v if isinstance(v, torch.Tensor) and v.dtype == torch.float64 else torch.as_tensor(np.asarray(v), dtype=torch.float64)
            for k, v in sd.items()}


def content_encoder(units, sd, cfg, eps, noise_scale=1.0):
    """enc_p on units [T][768] (ContentVec's frame-major rows): (m, logs, z_p), each [I][T].  eps [I][T] stands in for
    torch.randn_like (models.py:270); z_p = m + eps * exp(logs) * noise_scale."""
    w = as_float64(sd)
    c = torch.as_tensor(np.asarray(units, np.float64)).T[None]
    mask = torch.ones(1, 1, c.shape[2], dtype=torch.float64)
    x = vo.conv(c, w, "enc_p.pre")
    wcfg = dict(cfg, flow_kernel_size=ENC_P_KERNEL, flow_wn_layers=ENC_P_LAYERS, flow_dilation_rate=1)
    x = vo.wn(x, mask, None, w, "enc_p.enc", wcfg)
    m, logs = torch.split(vo.conv(x, w, "enc_p.proj"), cfg["inter_channels"], dim=1)
    z_p = m + torch.as_tensor(np.asarray(eps, np.float64))[None] * torch.exp(logs) * noise_scale
    return m[0].numpy(), logs[0].numpy(), z_p[0].numpy()


def flow_reverse(z_p, g, sd, cfg):
    """z = flow(z_p, mask, g, reverse=True) (models.py:869): [I][T]."""
    w = as_float64(sd)
    z = torch.as_tensor(np.asarray(z_p, np.float64))[None]
    mask = torch.ones(1, 1, z.shape[2], dtype=torch.float64)
    gg = torch.as_tensor(np.asarray(g, np.float64)).reshape(1, -1, 1)
    return vo.flow_reverse(z, mask, gg, w, cfg)[0].numpy()


def istft(spec, phase, n_fft, hop):
    """TorchSTFT.inverse (vc/stft.py:197-202): torch.istft(spec * exp(i phase)) with the periodic Hann window, which divides
    by the window envelope sum_f w^2.  spec, phase: [rows][n_fft/2 + 1][L] -> [rows][hop * (L - 1)]."""
    win = torch.hann_window(n_fft, periodic=True, dtype=torch.float64)
    return torch.istft(spec * torch.exp(phase * 1j), n_fft, hop, n_fft, window=win)


def decoder_trunk(z, w, cfg, g):
    """x = conv_pre(z) + cond(g), then per stage leaky ReLU, ConvTranspose1d with QuickVC's padding and output_padding
    (models.py:428-430), and the mean of the MRF resblocks (:463-481)."""
    x = vo.conv(z, w, "dec.conv_pre", padding=3) + vo.conv(g, w, "dec.cond")
    nk = len(cfg["resblock_kernel_sizes"])
    for i, u in enumerate(cfg["upsample_rates"]):
        p, op = convt_pad(cfg, i)
        x = F.leaky_relu(x, vo.LRELU_SLOPE)
        x = F.conv_transpose1d(x, w["dec.ups.%d.weight" % i], w["dec.ups.%d.bias" % i], stride=u, padding=p, output_padding=op)
        xs = None
        for j in range(nk):
            r = vo.resblock1(x, w, "dec.resblocks.%d" % (i * nk + j), cfg["resblock_kernel_sizes"][j], cfg["resblock_dilation_sizes"][j])
            xs = r if xs is None else xs + r
        x = xs / nk
    return x


def decode(z, g, sd, cfg):
    """o = dec(z, g) (Multistream_iSTFT_Generator.forward, models.py:459-501): z [I][T] -> [320 T] samples."""
    w = as_float64(sd)
    gg = torch.as_tensor(np.asarray(g, np.float64)).reshape(1, -1, 1)
    x = decoder_trunk(torch.as_tensor(np.asarray(z, np.float64))[None], w, cfg, gg)
    x = F.leaky_relu(x)
    x = F.pad(x, (1, 0), mode="reflect")
    x = vo.conv(x, w, "dec.subband_conv_post", padding=3)
    sb, nfft, hop = cfg["subbands"], cfg["gen_istft_n_fft"], cfg["gen_istft_hop_size"]
    x = x.reshape(1, sb, x.shape[1] // sb, x.shape[-1])
    nb = nfft // 2 + 1
    y = istft(torch.exp(x[0, :, :nb]), math.pi * torch.sin(x[0, :, nb:]), nfft, hop)[None]
    updown = torch.zeros(sb, sb, sb, dtype=torch.float64)
    for k in range(sb):
        updown[k, k, 0] = 1.0
    up = F.conv_transpose1d(y, updown * sb, stride=sb)
    return F.conv1d(up, w["dec.multistream_conv_post.weight"], None, padding=31)[0, 0].numpy()


def infer(units, g, sd, cfg, eps, noise_scale=1.0):
    """SynthesizerTrn.infer(c, mel=...) of one clip with its g given: dict of m_p, logs_p, z_p, z ([I][T]) and o ([320 T])."""
    sd = as_float64(sd)
    m, logs, z_p = content_encoder(units, sd, cfg, eps, noise_scale)
    z = flow_reverse(z_p, g, sd, cfg)
    return dict(m_p=m, logs_p=logs, z_p=z_p, z=z, o=decode(z, g, sd, cfg))
