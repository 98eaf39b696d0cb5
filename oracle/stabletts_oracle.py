"""CPU restatement of StableTTS text-to-mel, in any float dtype (float64 is what the GPU tests compare against):
MatchaTTS.synthesise (training/stabletts/matcha/models/matcha_tts.py:93-211) with TextEncoder.forward
(components/text_encoder.py:109-139), written from their formulas for ONE utterance.  The blocks, the conditioning rows and the
time schedule are those of stabletts_cfm_oracle; the estimator is restated here with the padded extent synthesise gives it:
the frame axis is padded to a multiple of 4 and only what the blocks write is masked, so the noise, cond_proj and in_proj live
on T_pad columns and reach the last valid frames through the convs' taps.  sd: a MatchaTTS state dict
(synthetic.make_random_stabletts); cfg: config.stabletts_config."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import stabletts_cfm_oracle as so

_w, _conv = so._w, so._conv


def ceil4(n):
    return (int(n) + 3) // 4 * 4


def token_rows(sd, cfg, ids, bert, dtype):
    """x [cond, T] (text_encoder.py:111-131): ids [streams, T], bert [bert_dim, T]."""
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long)
    E, P = int(cfg["emb_dim"]), int(cfg["punc_dim"])
    parts = [_w(sd, "encoder.emb.weight", dtype)[ids[0]] * torch.tensor(math.sqrt(E), dtype=torch.float32).to(dtype)]
    pe = _w(sd, "encoder.punc_emb.weight", dtype)
    parts += [pe[ids[s]] * torch.tensor(math.sqrt(P), dtype=torch.float32).to(dtype) for s in range(1, ids.shape[0])]
    b = torch.as_tensor(np.asarray(bert), dtype=dtype).T
    parts.append(b @ _w(sd, "encoder.bert_proj.1.weight", dtype).T + _w(sd, "encoder.bert_proj.1.bias", dtype))
    return torch.cat(parts, 1).T


def enc_block(sd, cfg, prefix, x, c, cs, dtype):
    """One DiTConVBlock of an encoder stack (diffusion_transformer.py:98-116) on x [hidden, T], all frames valid."""
    heads = int(cfg["enc_n_heads"])
    H, T = x.shape
    dk = H // heads
    a = prefix + "adaLN_modulation."
    h = F.silu(_w(sd, a + "0.weight", dtype) @ c + _w(sd, a + "0.bias", dtype))
    ada = (_w(sd, a + "2.weight", dtype) @ h + _w(sd, a + "2.bias", dtype)).reshape(6, -1)
    n1 = so.modulated_norm(x, ada[0], ada[1])
    q, k, v = (_conv(sd, prefix + "attn.conv_" + n, n1, dtype).reshape(heads, dk, T).transpose(1, 2) for n in "qkv")
    q, k = so.rope(q, *cs), so.rope(k, *cs)
    p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(dk), -1)
    o = (p @ v).transpose(1, 2).reshape(H, T)
    x = x + ada[2][:, None] * _conv(sd, prefix + "attn.conv_o", o, dtype)
    n2 = so.modulated_norm(x, ada[3], ada[4])
    y = _conv(sd, prefix + "mlp.conv_2", F.silu(_conv(sd, prefix + "mlp.conv_1", n2, dtype)), dtype)
    return x + ada[5][:, None] * y


def enc_stack(sd, cfg, stack, x, c, dtype):
    """Encoder.forward (text_encoder.py:40-46): the blocks, then proj.  stack: "encoder" or "dp_encoder"."""
    cs = so.rope_table(x.shape[1], int(cfg["enc_hidden_channels"]) // int(cfg["enc_n_heads"]) // 2, dtype)
    for l in range(int(cfg["enc_n_layers"])):
        x = enc_block(sd, cfg, "encoder.%s.encoder.%d." % (stack, l), x, c, cs, dtype)
    return _conv(sd, "encoder.%s.proj" % stack, x, dtype)


def duration_rule(logw, pause, length_scale):
    """w_round of matcha_tts.py:147-152 in fp32: the pause where it is not 0, times length_scale, rounded half to even, at
    least 1.  logw, pause: float32 arrays; returns (int64 durations, the fp32 value before rounding)."""
    v = np.asarray(logw, np.float32)
    if pause is not None:
        p = np.asarray(pause, np.float32)
        v = np.where(p == 0, v, p)
    v = (v * np.float32(length_scale)).astype(np.float32)
    return np.maximum(np.rint(v), 1).astype(np.int64), v


def estimator(sd, cfg, x, cond, T, t, adas, cs, dtype):
    """Decoder.forward (decoder.py:103-138) as synthesise calls it: x [noise, T_pad] and cond [hidden, T_pad] over the padded
    extent, the mask over the first T columns.  in_proj is not masked, and its output is the skip of the LAST long-skip
    conv, whose taps read it past T; every block's output is masked.  Returns [noise, T]."""
    e = "decoder.estimator."
    NL = cfg["n_layers"]
    temb = so.time_embedding(sd, cfg, t, dtype)
    h0 = _conv(sd, e + "in_proj", torch.cat([x, cond]), dtype)
    h = h0[:, :T]
    skips = []
    for l in range(NL):
        if l < NL // 2:
            skips.append(h0 if l == 0 else h)
        else:
            s = skips.pop()
            h = _conv(sd, e + "lsc_layers.%d" % (l - NL // 2), torch.cat([F.pad(h, (0, s.shape[1] - T)), s]), dtype)[:, :T]
        h = so.block(sd, cfg, l, h, temb, adas[l], cs, dtype)
    return _conv(sd, e + "final_proj", h, dtype)


def decode(sd, cfg, mu, spk, noise, extent=None, n_timesteps=10, temperature=1.0, guidance_scale=0.5, dtype=torch.float64):
    """CFM.forward (flow_matching.py:33-100,182-194) on mu [cond, T] padded with zero columns to `extent` (None: ceil4(T)),
    noise [noise, extent].  extent == T is stabletts_cfm_oracle.decode.  Returns the normalised mel [noise, T] (numpy)."""
    with torch.no_grad():
        mu = torch.as_tensor(np.asarray(mu), dtype=dtype)
        T = mu.shape[1]
        Tp = ceil4(T) if extent is None else int(extent)
        mu = F.pad(mu, (0, Tp - T))
        c = _w(sd, "spk_emb.weight", dtype)[int(spk)]
        NL, dk = cfg["n_layers"], cfg["hidden_channels"] // cfg["n_heads"]
        cs = so.rope_table(T, dk // 2, dtype)
        cond_c = so.cond_proj(sd, cfg, mu, dtype)
        ada_c = [so.ada_rows(sd, cfg, c, l, dtype) for l in range(NL)]
        if guidance_scale > 0:
            cond_u = so.cond_proj(sd, cfg, _w(sd, "fake_content", dtype)[0].repeat(1, Tp), dtype)
            ada_u = [so.ada_rows(sd, cfg, _w(sd, "fake_speaker", dtype)[0], l, dtype) for l in range(NL)]
        x = torch.as_tensor(np.asarray(noise), dtype=dtype)[:, :Tp] * temperature
        ts, dts = so.t_schedule(n_timesteps)
        for k in range(n_timesteps):
            d = estimator(sd, cfg, x, cond_c, T, float(ts[k]), ada_c, cs, dtype)
            if guidance_scale > 0:
                d = d + guidance_scale * (d - estimator(sd, cfg, x, cond_u, T, float(ts[k]), ada_u, cs, dtype))
            x = torch.cat([x[:, :T] + float(dts[k]) * d, x[:, T:]], 1)
        return x[:, :T].numpy()


def synthesise(sd, cfg, ids, bert, sid, noise, pause=None, n_timesteps=10, temperature=1.0, length_scale=1.0, guidance_scale=0.5,
               dtype=torch.float64, durations=None, extent=None):
    """One utterance: ids [streams, T], bert [bert_dim, T], pause [T] or None; noise [noise, >= ceil4(frames)].  durations:
    given durations replace the rule's (a float64 evaluation may round a token on a boundary the other way than fp32 does).
    Returns x, mu_dp, logw (before rounding, fp32 rule on the dtype's sums), durations, mu_y, decoder_outputs (pause frames
    filled), mel, encoder_outputs, mel_enc."""
    with torch.no_grad():
        x = token_rows(sd, cfg, ids, bert, dtype)
        mu_dp = enc_stack(sd, cfg, "dp_encoder", x, _w(sd, "dur_spk_emb.weight", dtype)[int(sid)], dtype)
        mu_mel = enc_stack(sd, cfg, "encoder", x, _w(sd, "spk_emb.weight", dtype)[int(sid)], dtype)
        logw = torch.sigmoid(mu_dp).sum(0).numpy()
        w, pre = duration_rule(logw.astype(np.float32), pause, length_scale)
        if durations is not None:
            w = np.asarray(durations, np.int64)
        tok = np.repeat(np.arange(len(w)), w)
        mu_y = x[:, tok]
        dec = decode(sd, cfg, mu_y, sid, noise, extent, n_timesteps, temperature, guidance_scale, dtype)
        if pause is not None:
            pau = np.asarray(pause, np.float32)[tok] > 0
            dec = np.where(pau[None, :], dec[:, :1], dec)
        enc = mu_mel[:, tok].numpy()
        return {"x": x.numpy(), "mu_dp": mu_dp.numpy(), "logw": logw, "pre_round": pre, "durations": w, "mu_y": mu_y.numpy(),
                "decoder_outputs": dec, "mel": so.denormalise(dec, sd), "encoder_outputs": enc, "mel_enc": so.denormalise(enc, sd)}
