"""The StableTTS vocoder's forward (the HiFi-GAN Generator of training/stabletts/matcha/hifigan/models.py:148-206, ResBlock1
:13-88 and ResBlock2 :91-130), restated with torch's functional convs in any float dtype (float64 for the tests' reference),
from a state dict with the weight norm folded and a config of vosk_tts_b200.config.hifigan_config."""
import torch
import torch.nn.functional as F

LRELU_SLOPE = 0.1


def generator(sd, h, mel, dtype=torch.float64):
    """mel [80, T] (or [B, 80, T]), denormalised -> waveform [T * hop] (or [B, T * hop]) in `dtype`; clamp(-1, 1) after
    tanh as the reference's caller (cli.py:126) does."""
    w = {k: torch.as_tensor(v).to(dtype) for k, v in sd.items()}
    x = torch.as_tensor(mel).to(dtype)
    single = x.dim() == 2
    if single:
        x = x[None]
    x = F.conv1d(x, w["conv_pre.weight"], w["conv_pre.bias"], padding=3)
    nk = len(h["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, LRELU_SLOPE)
        x = F.conv_transpose1d(x, w["ups.%d.weight" % i], w["ups.%d.bias" % i], stride=u, padding=(k - u) // 2)
        xs = None
        for j, (ks, dils) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            n, y = i * nk + j, x
            for d, dl in enumerate(dils):
                if h["resblock"] == "1":
                    p = "resblocks.%d.convs%%d.%d." % (n, d)
                    t = F.conv1d(F.leaky_relu(y, LRELU_SLOPE), w[p % 1 + "weight"], w[p % 1 + "bias"], dilation=dl, padding=dl * (ks - 1) // 2)
                    t = F.conv1d(F.leaky_relu(t, LRELU_SLOPE), w[p % 2 + "weight"], w[p % 2 + "bias"], padding=(ks - 1) // 2)
                else:
                    p = "resblocks.%d.convs.%d." % (n, d)
                    t = F.conv1d(F.leaky_relu(y, LRELU_SLOPE), w[p + "weight"], w[p + "bias"], dilation=dl, padding=dl * (ks - 1) // 2)
                y = t + y
            xs = y if xs is None else xs + y
        x = xs / nk
    x = F.conv1d(F.leaky_relu(x), w["conv_post.weight"], w["conv_post.bias"], padding=3)
    x = torch.tanh(x).clamp(-1, 1)[:, 0]
    return x[0] if single else x
