"""CPU restatement of the StableTTS flow-matching decoder, in any float dtype (float64 is what the GPU tests compare
against): CFM.forward -> solve_euler -> Decoder of training/stabletts/matcha/models/components/{flow_matching, decoder,
diffusion_transformer}.py, written from their formulas for ONE utterance (every mask is then all ones, and the convs are zero
padded at the utterance's own ends).  sd: a MatchaTTS state dict (synthetic.make_random_stabletts_cfm); cfg:
config.stabletts_cfm_config."""
import math

import numpy as np
import torch
import torch.nn.functional as F


def _w(sd, name, dtype):
    return sd[name].detach().to(dtype)


def t_schedule(n):
    """(t, dt) of the n Euler steps in the reference's fp32 arithmetic (flow_matching.py:54-55,87-98): t_span = 1 - cos(linspace
    pi / 2), t accumulates and dt is the distance from it to the next knot.  float32 arrays."""
    span = torch.linspace(0, 1, n + 1)
    span = (1 - torch.cos(span * 0.5 * torch.pi)).numpy()
    ts, dts = np.zeros(n, np.float32), np.zeros(n, np.float32)
    t, dt = span[0], span[1] - span[0]
    for k in range(n):
        ts[k], dts[k] = t, dt
        t = np.float32(t + dt)
        if k + 1 < n:
            dt = np.float32(span[k + 2] - t)
    return ts, dts


def time_embedding(sd, cfg, t, dtype):
    """SinusoidalPosEmb(scale 1000) -> time_mlp (decoder.py:35-62,120): [hidden]."""
    H = cfg["hidden_channels"]
    half = H // 2
    freq = torch.exp(torch.arange(half, dtype=dtype) * -(math.log(10000) / (half - 1)))
    a = 1000 * torch.as_tensor(t, dtype=dtype) * freq
    emb = torch.cat([a.sin(), a.cos()])
    e = "decoder.estimator.time_mlp.layer."
    h = F.silu(_w(sd, e + "0.weight", dtype) @ emb + _w(sd, e + "0.bias", dtype))
    return _w(sd, e + "2.weight", dtype) @ h + _w(sd, e + "2.bias", dtype)


def film_rows(sd, cfg, temb, l, dtype):
    """(gamma, beta) [hidden] each of block l (decoder.py:31-33)."""
    b = "decoder.estimator.blocks.%d.time_fusion.film." % l
    gb = _w(sd, b + "weight", dtype)[:, :, 0] @ temb + _w(sd, b + "bias", dtype)
    return gb.chunk(2)


def ada_rows(sd, cfg, c, l, dtype):
    """The six adaLN chunks [6, hidden] of block l for the speaker vector c (diffusion_transformer.py:107-111)."""
    b = "decoder.estimator.blocks.%d.block.adaLN_modulation." % l
    h = F.silu(_w(sd, b + "0.weight", dtype) @ c + _w(sd, b + "0.bias", dtype))
    return (_w(sd, b + "2.weight", dtype) @ h + _w(sd, b + "2.bias", dtype)).reshape(6, -1)


def rope_table(T, d, dtype):
    """cos / sin [T, d/2] of the rotary embedding (diffusion_transformer.py:151-166): theta and the angle are fp32 in the
    reference whatever the model's dtype, so they are here; cos / sin are then taken in `dtype`."""
    theta = 1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))
    ang = (torch.arange(T).float()[:, None] * theta[None, :]).to(dtype)
    return ang.cos(), ang.sin()


def rope(x, cos, sin):
    """x [heads, T, dk]: the first d = 2 * cos.shape[1] features rotated (diffusion_transformer.py:179-197)."""
    hd = cos.shape[1]
    a, b, rest = x[..., :hd], x[..., hd:2 * hd], x[..., 2 * hd:]
    return torch.cat([a * cos - b * sin, b * cos + a * sin, rest], -1)


def _conv(sd, name, x, dtype):
    w = _w(sd, name + ".weight", dtype)
    return F.conv1d(x[None], w, _w(sd, name + ".bias", dtype), padding=w.shape[2] // 2)[0]


def cond_proj(sd, cfg, mu, dtype):
    e = "decoder.estimator.cond_proj."
    return _conv(sd, e + "4", F.silu(_conv(sd, e + "2", F.silu(_conv(sd, e + "0", mu, dtype)), dtype)), dtype)


def modulated_norm(x, shift, scale):
    """LayerNorm over channels without affine, then x (1 + scale) + shift; x [C, T]."""
    n = F.layer_norm(x.T, (x.shape[0],), eps=1e-5).T
    return n * (1 + scale[:, None]) + shift[:, None]


def block(sd, cfg, l, x, temb, ada, cs, dtype, taps=None):
    """DitWrapper l (decoder.py:15-18; diffusion_transformer.py:98-116) on x [hidden, T]."""
    heads = cfg["n_heads"]
    H, T = x.shape
    dk = H // heads
    gamma, beta = film_rows(sd, cfg, temb, l, dtype)
    x = gamma[:, None] * x + beta[:, None]
    b = "decoder.estimator.blocks.%d.block." % l
    n1 = modulated_norm(x, ada[0], ada[1])
    q, k, v = (_conv(sd, b + "attn.conv_" + n, n1, dtype).reshape(heads, dk, T).transpose(1, 2) for n in "qkv")
    q, k = rope(q, *cs), rope(k, *cs)
    if taps is not None:
        taps["norm1"], taps["q"], taps["k"], taps["v"] = n1, q, k, v
    p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(dk), -1)
    o = (p @ v).transpose(1, 2).reshape(H, T)
    x = x + ada[2][:, None] * _conv(sd, b + "attn.conv_o", o, dtype)
    n2 = modulated_norm(x, ada[3], ada[4])
    y = _conv(sd, b + "mlp.conv_2", F.silu(_conv(sd, b + "mlp.conv_1", n2, dtype)), dtype)
    return x + ada[5][:, None] * y


def estimator(sd, cfg, x, cond, t, adas, cs, dtype, taps=None):
    """Decoder.forward (decoder.py:103-138) with cond = cond_proj(mu) given; x [noise, T] -> [noise, T]."""
    e = "decoder.estimator."
    NL = cfg["n_layers"]
    temb = time_embedding(sd, cfg, t, dtype)
    h = _conv(sd, e + "in_proj", torch.cat([x, cond]), dtype)
    skips = []
    for l in range(NL):
        if l < NL // 2:
            skips.append(h)
        else:
            h = _conv(sd, e + "lsc_layers.%d" % (l - NL // 2), torch.cat([h, skips.pop()]), dtype)
        h = block(sd, cfg, l, h, temb, adas[l], cs, dtype, taps if l == 0 else None)
    return _conv(sd, e + "final_proj", h, dtype)


def decode(sd, cfg, mu, spk, noise, n_timesteps=10, temperature=1.0, guidance_scale=0.5, dtype=torch.float64, taps=None):
    """mu [cond, T], spk: a speaker id or an embedding [spk_emb_dim], noise [noise, T] -> the normalised mel [noise, T] after
    the last Euler step (numpy, `dtype`).  taps: a dict that receives the conditioning rows and block 0's tensors of the
    first estimator evaluation."""
    with torch.no_grad():
        mu = torch.as_tensor(np.asarray(mu), dtype=dtype)
        T = mu.shape[1]
        c = _w(sd, "spk_emb.weight", dtype)[int(spk)] if np.ndim(spk) == 0 else torch.as_tensor(np.asarray(spk), dtype=dtype)
        NL, dk = cfg["n_layers"], cfg["hidden_channels"] // cfg["n_heads"]
        cs = rope_table(T, dk // 2, dtype)
        cond_c = cond_proj(sd, cfg, mu, dtype)
        ada_c = [ada_rows(sd, cfg, c, l, dtype) for l in range(NL)]
        if guidance_scale > 0:
            cond_u = cond_proj(sd, cfg, _w(sd, "fake_content", dtype)[0].repeat(1, T), dtype)
            ada_u = [ada_rows(sd, cfg, _w(sd, "fake_speaker", dtype)[0], l, dtype) for l in range(NL)]
        x = torch.as_tensor(np.asarray(noise), dtype=dtype) * temperature
        ts, dts = t_schedule(n_timesteps)
        if taps is not None:
            taps["ada"], taps["cond"], taps["rope"] = torch.stack(ada_c), cond_c, cs
            taps["film"] = torch.stack([torch.cat(film_rows(sd, cfg, time_embedding(sd, cfg, float(t), dtype), l, dtype))
                                        for t in ts for l in range(NL)]).reshape(n_timesteps, NL, -1)
        for k in range(n_timesteps):
            d = estimator(sd, cfg, x, cond_c, float(ts[k]), ada_c, cs, dtype, taps if k == 0 else None)
            if guidance_scale > 0:
                d = d + guidance_scale * (d - estimator(sd, cfg, x, cond_u, float(ts[k]), ada_u, cs, dtype))
            x = x + float(dts[k]) * d
        return x.numpy()


def denormalise(mel, sd):
    return mel * float(sd["mel_std"]) + float(sd["mel_mean"])
