"""Seeded synthetic checkpoints in the reference's ``G_*.pth['model']`` layout.

No checkpoint (``vosk-model-tts-ru-0.9-multi`` / ``G_*.pth``) exists on the build or GPU
boxes, so benchmarks and parity tests run on random weights of the reference
architecture (BASELINE.md section 3).  The tensor names and shapes follow
``SynthesizerTrn.state_dict()`` before weight-norm removal (SURVEY.md appendix B;
/root/reference/training/vits2/models.py:1508-1630): weight-normed convs appear as
``weight_g`` / ``weight_v`` pairs exactly as in a training checkpoint, so the loader's
folding path (``weights.fold_weight_norm``) is exercised.

Unlike the reference's own initialisation, the tensors that the reference zero-inits
(``flow.*.post`` models.py:371-372, ``ConvFlow.proj`` modules.py:361-362, LayerNorm beta)
are given non-zero values here, otherwise the coupling flow and the spline would be
identity maps and the parity tests would not exercise them.

The generator draws every tensor from its own ``torch.Generator`` (seeded from the
tensor name), so the values do not depend on enumeration order or torch's global RNG.
"""
import math
import zlib

import numpy as np
import torch


def _conv(out, name, co, ci, ks, wn=False, bias=True, gain=1.0, transposed=False):
    """Appends the spec of one Conv1d / ConvTranspose1d (weight-normed: weight_g + weight_v) to `out`."""
    shape = (ci, co, ks) if transposed else (co, ci, ks)
    fan_in = ci * ks if not transposed else ci * ks / 4.0
    std = gain / math.sqrt(fan_in)
    if wn:
        out.append((name + ".weight_g", (shape[0], 1, 1), "wn_g", name + ".weight_v"))
        out.append((name + ".weight_v", shape, "normal", std))
    else:
        out.append((name + ".weight", shape, "normal", std))
    if bias:
        out.append((name + ".bias", (co,), "normal", 0.05))


def _spec(cfg, posterior=False):
    """Ordered list of (name, shape, kind, scale) for every tensor ``infer`` touches (posterior=True: and the posterior
    encoder ``enc_q`` that ``voice_conversion`` uses, models.py:1616, 813-842)."""
    H = cfg["hidden_channels"]
    I = cfg["inter_channels"]
    Fc = cfg["filter_channels"]
    G = cfg["gin_channels"]
    nh = cfg["n_heads"]
    W = cfg["window_size"]
    k = cfg["kernel_size"]
    out = []

    def conv(*a, **kw):
        _conv(out, *a, **kw)

    def ln(name, c):
        out.append((name + ".gamma", (c,), "gamma", 0.1))
        out.append((name + ".beta", (c,), "normal", 0.1))

    def encoder(prefix, hidden, filt, n_layers, ks, heads):
        for i in range(n_layers):
            a = "%s.attn_layers.%d" % (prefix, i)
            dk = hidden // heads
            out.append((a + ".emb_rel_k", (1, 2 * W + 1, dk), "normal", dk ** -0.5))
            out.append((a + ".emb_rel_v", (1, 2 * W + 1, dk), "normal", dk ** -0.5))
            for nm in ("conv_q", "conv_k", "conv_v", "conv_o"):
                conv(a + "." + nm, hidden, hidden, 1, gain=1.0)
            ln("%s.norm_layers_1.%d" % (prefix, i), hidden)
            conv("%s.ffn_layers.%d.conv_1" % (prefix, i), filt, hidden, ks, gain=1.2)
            conv("%s.ffn_layers.%d.conv_2" % (prefix, i), hidden, filt, ks, gain=1.2)
            ln("%s.norm_layers_2.%d" % (prefix, i), hidden)

    def dds(prefix, c, ks, n_layers):
        for i in range(n_layers):
            out.append(("%s.convs_sep.%d.weight" % (prefix, i), (c, 1, ks), "normal", 0.4))
            out.append(("%s.convs_sep.%d.bias" % (prefix, i), (c,), "normal", 0.2))
            conv("%s.convs_1x1.%d" % (prefix, i), c, c, 1, gain=1.0)
            ln("%s.norms_1.%d" % (prefix, i), c)
            ln("%s.norms_2.%d" % (prefix, i), c)

    # --- speaker table, text encoder (models.py:283-326, attentions.py:13-65)
    if cfg["n_speakers"] > 1:
        out.append(("emb_g.weight", (cfg["n_speakers"], G), "normal", 1.0))
    out.append(("enc_p.emb.weight", (cfg["n_vocab"], H), "normal", H ** -0.5))
    encoder("enc_p.encoder", H, Fc, cfg["n_layers"], k, nh)
    if cfg["use_spk_conditioned_encoder"] and G > 0:
        out.append(("enc_p.encoder.spk_emb_linear.weight", (H, G), "normal", 0.5 / math.sqrt(G)))
        out.append(("enc_p.encoder.spk_emb_linear.bias", (H,), "normal", 0.05))
    conv("enc_p.proj", 2 * I, H, 1, gain=0.6)

    # --- stochastic duration predictor (models.py:23-63); flows.1 is unused in reverse (:94-95)
    D = cfg["dp_filter_channels"]
    conv("dp.pre", D, H, 1)
    conv("dp.proj", D, D, 1)
    dds("dp.convs", D, cfg["dp_kernel_size"], 3)
    if G > 0:
        conv("dp.cond", D, G, 1, gain=0.5)
    out.append(("dp.flows.0.m", (2, 1), "ea_m", 0.2))
    out.append(("dp.flows.0.logs", (2, 1), "normal", 0.2))
    nb = cfg["dp_num_bins"]
    for f in range(cfg["dp_n_flows"]):
        p = "dp.flows.%d" % (2 * f + 1)
        conv(p + ".pre", D, 1, 1, gain=0.6)
        dds(p + ".convs", D, cfg["dp_kernel_size"], 3)
        out.append((p + ".proj.weight", (3 * nb - 1, D, 1), "spline_proj", nb))
        out.append((p + ".proj.bias", (3 * nb - 1,), "normal", 0.3))

    # --- flow (models.py:329-396 / 765-810, modules.py:111-184)
    fk = cfg["flow_kernel_size"]
    for f in range(cfg["flow_n_flows"]):
        p = "flow.flows.%d" % (2 * f)
        conv(p + ".pre", H, I // 2, 1)
        if cfg["use_transformer_flows"]:
            encoder(p + ".pre_transformer", H, H, 1, fk, cfg.get("flow_n_heads", 2))   # (2 heads hard-coded, models.py:355)
        for i in range(cfg["flow_wn_layers"]):
            conv("%s.enc.in_layers.%d" % (p, i), 2 * H, H, fk, wn=True, gain=1.0)
            rs = 2 * H if i < cfg["flow_wn_layers"] - 1 else H
            conv("%s.enc.res_skip_layers.%d" % (p, i), rs, H, 1, wn=True, gain=0.7)
        if G > 0:
            conv(p + ".enc.cond_layer", 2 * H * cfg["flow_wn_layers"], G, 1, wn=True, gain=0.5)
        conv(p + ".post", I // 2, H, 1, gain=0.35)

    # --- decoder (models.py:974-1063 / 845-898, modules.py:187-258)
    C0 = cfg["upsample_initial_channel"]
    if cfg["decoder"] in ("mb_istft", "ms_istft", "istft"):
        conv("dec.conv_pre", C0, I, 7, wn=True, gain=1.0)
    else:      # plain Generator: conv_pre is not weight-normed and a speaker projection is added to its output (models.py:851,869-875)
        conv("dec.conv_pre", C0, I, 7, wn=False, gain=1.0)
        if G > 0:
            conv("dec.cond", C0, G, 1, gain=0.5)
    ch = C0
    for i, (u, ku) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        conv("dec.ups.%d" % i, ch // 2, ch, ku, wn=True, gain=1.0, transposed=True)
        ch //= 2
        for j, (rk, rd) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            rb = "dec.resblocks.%d" % (i * len(cfg["resblock_kernel_sizes"]) + j)
            if cfg["resblock"] == "1":
                for d in range(len(rd)):
                    conv("%s.convs1.%d" % (rb, d), ch, ch, rk, wn=True, gain=0.55)
                    conv("%s.convs2.%d" % (rb, d), ch, ch, rk, wn=True, gain=0.55)
            else:
                for d in range(len(rd)):
                    conv("%s.convs.%d" % (rb, d), ch, ch, rk, wn=True, gain=0.55)
    if cfg["decoder"] == "mb_istft":
        conv("dec.subband_conv_post", cfg["subbands"] * (cfg["gen_istft_n_fft"] + 2), ch, 7,
             wn=True, bias=False, gain=0.25)
    elif cfg["decoder"] == "ms_istft":      # models.py:1095 (bias!), :1107 learned 63-tap merge filter
        conv("dec.subband_conv_post", cfg["subbands"] * (cfg["gen_istft_n_fft"] + 2), ch, 7, wn=True, bias=True, gain=0.25)
        conv("dec.multistream_conv_post", 1, cfg["subbands"], 63, wn=True, bias=False, gain=1.0)
    elif cfg["decoder"] == "istft":         # models.py:928
        conv("dec.conv_post", cfg["gen_istft_n_fft"] + 2, ch, 7, wn=True, bias=False, gain=0.25)
    else:
        conv("dec.conv_post", 1, ch, 7, wn=False, bias=False, gain=0.5)     # plain Conv1d (models.py:868)

    # --- posterior encoder (models.py:813-842): pre 1x1, 16-layer WN (kernel 5, weight-normed), proj 1x1
    if posterior:
        nq = 16
        conv("enc_q.pre", H, cfg.get("spec_channels", 80), 1, gain=0.5)
        for i in range(nq):
            conv("enc_q.enc.in_layers.%d" % i, 2 * H, H, 5, wn=True, gain=1.0)
            conv("enc_q.enc.res_skip_layers.%d" % i, 2 * H if i < nq - 1 else H, H, 1, wn=True, gain=0.5)
        if G > 0:
            conv("enc_q.enc.cond_layer", 2 * H * nq, G, 1, wn=True, gain=0.5)
        conv("enc_q.proj", 2 * I, H, 1, gain=0.1)
    return out


def _gen(name, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


def make_random_checkpoint(cfg, seed=1234, posterior=False):
    """state_dict (CPU fp32) in checkpoint layout; deterministic for (cfg, seed).  posterior=True adds the ``enc_q.*``
    tensors (every tensor is seeded by its name, so the others come out the same either way)."""
    return _draw(_spec(cfg, posterior), seed)


def _draw(spec, seed):
    sd = {}
    for name, shape, kind, arg in spec:
        if kind == "wn_g":
            continue
        g = _gen(name, seed)
        if kind == "normal":
            t = torch.randn(shape, generator=g) * arg
        elif kind == "ea_m":
            # shift log-durations up so that synthetic utterances average ~2 frames per token
            t = torch.randn(shape, generator=g) * arg - 0.9
        elif kind == "gamma":
            t = 1.0 + torch.randn(shape, generator=g) * arg
        elif kind == "spline_proj":
            nb = arg
            t = torch.randn(shape, generator=g) / math.sqrt(shape[1])
            t[: 2 * nb] *= 6.0   # widths / heights logits (divided by sqrt(filter) downstream)
            t[2 * nb:] *= 0.8    # derivative logits
        else:
            raise ValueError(kind)
        sd[name] = t.float().contiguous()
    for name, shape, kind, arg in spec:
        if kind != "wn_g":
            continue
        v = sd[arg]
        nrm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(shape)
        g = _gen(name, seed)
        sd[name] = (nrm * (1.0 + 0.15 * torch.randn(shape, generator=g))).float().contiguous()
    return sd


def param_names(cfg, posterior=False):
    return [s[0] for s in _spec(cfg, posterior)]


def make_random_speaker_encoder(cfg, seed=1234):
    """The ``enc_spk.*`` tensors of a QuickVC checkpoint (SpeakerEncoder, vc/models.py:728-736: nn.LSTM(n_mel, G, 3) +
    nn.Linear(G, G)), CPU fp32, deterministic for (cfg, seed).  Drawn like PyTorch's own initialisation, uniform in
    +-1/sqrt(G), so that the gates operate in the range a trained encoder sees rather than saturating."""
    G, n_mel = cfg["gin_channels"], cfg["n_mel_channels"]
    a = 1.0 / math.sqrt(G)
    shapes = []
    for l in range(cfg.get("spk_layers", 3)):
        shapes += [("enc_spk.lstm.weight_ih_l%d" % l, (4 * G, n_mel if l == 0 else G)), ("enc_spk.lstm.weight_hh_l%d" % l, (4 * G, G)),
                   ("enc_spk.lstm.bias_ih_l%d" % l, (4 * G,)), ("enc_spk.lstm.bias_hh_l%d" % l, (4 * G,))]
    shapes += [("enc_spk.linear.weight", (G, G)), ("enc_spk.linear.bias", (G,))]
    return {name: ((torch.rand(shape, generator=_gen(name, seed)) * 2 - 1) * a).float().contiguous() for name, shape in shapes}


def _spec_quickvc(cfg):
    """(name, shape, kind, scale) of every tensor of the reference QuickVC SynthesizerTrn (vc/models.py:774-842) but the
    speaker encoder: enc_p (PosteriorEncoder(768, I, H, 5, 1, 16), no g), enc_q (the same over the linear spectrogram, with
    g), the flow (ResidualCouplingBlock(I, H, 5, 1, 4, gin): mean-only coupling layers at even indices, Flip between) and
    the Multistream_iSTFT_Generator decoder (:416-501) with its cond Conv1d(256, 512, 1) and the updown_filter buffer."""
    H, I, G = cfg["hidden_channels"], cfg["inter_channels"], cfg["gin_channels"]
    out = []
    conv = lambda *a, **kw: _conv(out, *a, **kw)
    for p, cin, gin in (("enc_p", cfg["unit_channels"], 0), ("enc_q", cfg["filter_length"] // 2 + 1, G)):
        conv(p + ".pre", H, cin, 1, gain=0.5 if p == "enc_q" else 1.0)
        for i in range(16):
            conv("%s.enc.in_layers.%d" % (p, i), 2 * H, H, 5, wn=True, gain=1.0)
            conv("%s.enc.res_skip_layers.%d" % (p, i), 2 * H if i < 15 else H, H, 1, wn=True, gain=0.5)
        if gin:
            conv(p + ".enc.cond_layer", 2 * H * 16, gin, 1, wn=True, gain=0.5)
        conv(p + ".proj", 2 * I, H, 1, gain=0.1)
    for f in range(cfg["flow_n_flows"]):
        p = "flow.flows.%d" % (2 * f)
        conv(p + ".pre", H, I // 2, 1)
        for i in range(cfg["flow_wn_layers"]):
            conv("%s.enc.in_layers.%d" % (p, i), 2 * H, H, cfg["flow_kernel_size"], wn=True, gain=1.0)
            conv("%s.enc.res_skip_layers.%d" % (p, i), 2 * H if i < cfg["flow_wn_layers"] - 1 else H, H, 1, wn=True, gain=0.7)
        conv(p + ".enc.cond_layer", 2 * H * cfg["flow_wn_layers"], G, 1, wn=True, gain=0.5)
        conv(p + ".post", I // 2, H, 1, gain=0.35)
    C0 = cfg["upsample_initial_channel"]
    conv("dec.conv_pre", C0, I, 7, wn=True, gain=1.0)
    ch = C0
    nk = len(cfg["resblock_kernel_sizes"])
    for i, ku in enumerate(cfg["upsample_kernel_sizes"]):
        conv("dec.ups.%d" % i, ch // 2, ch, ku, wn=True, gain=1.0, transposed=True)
        ch //= 2
        for j, rd in enumerate(cfg["resblock_dilation_sizes"]):
            for d in range(len(rd)):
                conv("dec.resblocks.%d.convs1.%d" % (i * nk + j, d), ch, ch, cfg["resblock_kernel_sizes"][j], wn=True, gain=0.55)
                conv("dec.resblocks.%d.convs2.%d" % (i * nk + j, d), ch, ch, cfg["resblock_kernel_sizes"][j], wn=True, gain=0.55)
    conv("dec.subband_conv_post", cfg["subbands"] * (cfg["gen_istft_n_fft"] + 2), ch, 7, wn=True, bias=True, gain=0.25)
    conv("dec.multistream_conv_post", 1, cfg["subbands"], 63, wn=True, bias=False, gain=1.0)
    conv("dec.cond", C0, G, 1, gain=0.5)
    return out


def make_random_quickvc(cfg, seed=1234):
    """A whole QuickVC checkpoint state dict (CPU fp32) in the reference's names and shapes, weight-normed convs as
    weight_g / weight_v: enc_p, enc_q (real checkpoints carry it; inference never reads it), the flow, the decoder with its
    updown_filter buffer, and enc_spk exactly as make_random_speaker_encoder(cfg, seed) draws it."""
    sd = _draw(_spec_quickvc(cfg), seed)
    sb = cfg["subbands"]
    updown = torch.zeros(sb, sb, sb)
    for k in range(sb):
        updown[k, k, 0] = 1.0
    sd["dec.updown_filter"] = updown
    sd.update(make_random_speaker_encoder(cfg, seed))
    return sd


def make_random_contentvec(seed=1234, cv=None):
    """A ContentVec state dict (HubertModelWithFinalProj of vc/contentvec.py, CPU fp32) in the reference's names and shapes for
    the shape cv (config.contentvec_config; default hubert-base).  The positional conv is weight-normed as the published
    checkpoint stores it (weight_g [1, 1, K] / weight_v, dim=2).  Biases and the LayerNorm / GroupNorm affines are non-trivial;
    final_proj and masked_spec_embed, which inference never reads, are there as in a real checkpoint."""
    from . import config as _config
    cv = cv or _config.contentvec_config()
    C, H, Fh, K, G = cv["cv_conv_dim"], cv["cv_hidden"], cv["cv_ffn"], cv["cv_pos_k"], cv["cv_pos_groups"]
    out = []
    ln = lambda name, c: out.extend([(name + ".weight", (c,), "gamma", 0.1), (name + ".bias", (c,), "normal", 0.1)])
    fe = "feature_extractor.conv_layers.%d."
    for i, k in enumerate(cv["cv_conv_kernel"]):
        ci = 1 if i == 0 else C
        out.append((fe % i + "conv.weight", (C, ci, k), "normal", (0.5 if i == 0 else 1.6) / math.sqrt(ci * k)))
    ln(fe % 0 + "layer_norm", C)
    ln("feature_projection.layer_norm", C)
    _conv(out, "feature_projection.projection", H, C, 1)
    ln("encoder.layer_norm", H)
    for l in range(cv["cv_layers"]):
        p = "encoder.layers.%d." % l
        for n in ("q", "k", "v", "out"):
            _conv(out, p + "attention.%s_proj" % n, H, H, 1, gain=1.5 if n in "qk" else 1.0)
        ln(p + "layer_norm", H)
        _conv(out, p + "feed_forward.intermediate_dense", Fh, H, 1)
        _conv(out, p + "feed_forward.output_dense", H, Fh, 1)
        ln(p + "final_layer_norm", H)
    _conv(out, "final_proj", 256, H, 1)
    out.append(("masked_spec_embed", (H,), "normal", 1.0))
    sd = _draw(out, seed)
    for name, shape in list(((n, s) for n, s, _, _ in out)):
        if len(shape) == 3 and shape[2] == 1:
            sd[name] = sd[name][:, :, 0].contiguous()          # the Linear layers: [out, in]
    pos = "encoder.pos_conv_embed.conv."
    v = torch.randn((H, H // G, K), generator=_gen(pos + "weight_v", seed)) / math.sqrt(H // G * K)
    sd[pos + "weight_v"] = v.float().contiguous()
    nrm = v.norm(dim=(0, 1), keepdim=True)
    sd[pos + "weight_g"] = (nrm * (1.0 + 0.15 * torch.randn(nrm.shape, generator=_gen(pos + "weight_g", seed)))).float().contiguous()
    sd[pos + "bias"] = (torch.randn((H,), generator=_gen(pos + "bias", seed)) * 0.05).float().contiguous()
    return sd


def make_random_stabletts_cfm(cfg, seed=1234):
    """The tensors weights.pack_stabletts_cfm reads of a MatchaTTS state dict (decoder.estimator.*, spk_emb.weight,
    fake_speaker, fake_content, mel_mean, mel_std), CPU fp32, deterministic for (cfg, seed); every tensor is seeded by its name.
    Weights are drawn at 1 / sqrt(fan-in) so that activations keep their scale through the blocks.  The last adaLN linear,
    which the reference initialises to zero (decoder.py:98-101), is random here: with zeros every gate is 0 and every block
    the identity, and a comparison would prove nothing."""
    NC, MC, H, F, NL, G = (int(cfg[k]) for k in ("noise_channels", "cond_channels", "hidden_channels", "filter_channels", "n_layers",
                                                 "spk_emb_dim"))
    k = int(cfg["kernel_size"])
    e = "decoder.estimator."
    shapes = [(e + "time_mlp.layer.0", (F, H)), (e + "time_mlp.layer.2", (H, F)), (e + "in_proj", (H, NC + H, 1)),
              (e + "final_proj", (NC, H, 1)), (e + "cond_proj.0", (F, MC, k)), (e + "cond_proj.2", (F, F, k)),
              (e + "cond_proj.4", (H, F, k))]
    for l in range(NL):
        b = e + "blocks.%d." % l
        shapes += [(b + "time_fusion.film", (2 * H, H, 1)), (b + "block.adaLN_modulation.0", (H, G)),
                   (b + "block.adaLN_modulation.2", (6 * H, H)), (b + "block.mlp.conv_1", (F, H, k)), (b + "block.mlp.conv_2", (H, F, k))]
        shapes += [(b + "block.attn.conv_%s" % n, (H, H, 1)) for n in "qkvo"]
    shapes += [(e + "lsc_layers.%d" % j, (H, 2 * H, k)) for j in range(NL // 2)]
    sd = {}
    for name, shape in shapes:
        fan = int(np.prod(shape[1:]))
        sd[name + ".weight"] = (torch.randn(shape, generator=_gen(name + ".weight", seed)) / math.sqrt(fan)).float().contiguous()
        sd[name + ".bias"] = (torch.randn(shape[0], generator=_gen(name + ".bias", seed)) * 0.1).float().contiguous()
    for l in range(NL):      # FiLM's gamma around 1 (gamma * x + beta)
        sd[e + "blocks.%d.time_fusion.film.bias" % l][:H] += 1.0
    for name, shape, scale in (("spk_emb.weight", (int(cfg["n_spks"]), G), 1.0), ("fake_speaker", (1, G), 0.5),
                               ("fake_content", (1, MC, 1), 0.5)):
        sd[name] = (torch.randn(shape, generator=_gen(name, seed)) * scale).float().contiguous()
    sd["mel_mean"] = torch.tensor(-5.5)
    sd["mel_std"] = torch.tensor(2.1)
    return sd


def make_random_stabletts(cfg, seed=1234):
    """make_random_stabletts_cfm plus the tensors weights.pack_stabletts reads of the text side (encoder.*, dur_spk_emb.weight),
    for cfg = config.stabletts_config.  The embeddings are drawn at the reference's 1 / sqrt(width) (text_encoder.py:99,103);
    the last adaLN linear of every encoder block, zero in the reference (text_encoder.py:35-38), is random for the reason given
    there.  dp_encoder's proj gets a bias of -2.8 so that the 50 sigmoids sum to a few frames per token, as a trained model's."""
    sd = make_random_stabletts_cfm(cfg, seed)
    V, E, PD, BD, R, H, F, NE, G, DC = (int(cfg[k]) for k in ("n_vocab", "emb_dim", "punc_dim", "bert_dim", "bert_proj_dim",
                                                             "enc_hidden_channels", "enc_filter_channels", "enc_n_layers", "spk_emb_dim",
                                                             "dur_channels"))
    k = int(cfg["enc_kernel_size"])
    shapes = [("encoder.bert_proj.1", (R, BD))]
    for stack, co in (("encoder.encoder.", int(cfg["noise_channels"])), ("encoder.dp_encoder.", DC)):
        shapes.append((stack + "proj", (co, H, 1)))
        for l in range(NE):
            b = stack + "encoder.%d." % l
            shapes += [(b + "adaLN_modulation.0", (H, G)), (b + "adaLN_modulation.2", (6 * H, H)), (b + "mlp.conv_1", (F, H, k)),
                       (b + "mlp.conv_2", (H, F, k))]
            shapes += [(b + "attn.conv_%s" % n, (H, H, 1)) for n in "qkvo"]
    for name, shape in shapes:
        fan = int(np.prod(shape[1:]))
        sd[name + ".weight"] = (torch.randn(shape, generator=_gen(name + ".weight", seed)) / math.sqrt(fan)).float().contiguous()
        sd[name + ".bias"] = (torch.randn(shape[0], generator=_gen(name + ".bias", seed)) * 0.1).float().contiguous()
    sd["encoder.dp_encoder.proj.bias"] -= 2.8
    for name, shape, scale in (("encoder.emb.weight", (V, E), E ** -0.5), ("encoder.punc_emb.weight", (V, PD), PD ** -0.5),
                               ("dur_spk_emb.weight", (int(cfg["n_spks"]), G), 1.0)):
        sd[name] = (torch.randn(shape, generator=_gen(name, seed)) * scale).float().contiguous()
    return sd


def make_random_hifigan(seed=1234, h=None, gain=None):
    """A HiFi-GAN Generator checkpoint's `generator` state dict (matcha/hifigan/models.py:148-206, weight-normed convs as
    weight_g / weight_v pairs, which weights.load_hifigan folds), CPU fp32, deterministic for (h, seed); h: config.hifigan_config
    (None: v1).  The reference's init_weights (N(0, 0.01)) leaves a random mel's waveform near |wav| 0.06; the weights here are
    drawn at GAIN / sqrt(fan-in) instead, so that a mel of the scale synthesise produces reaches |wav| of about 0.3-0.9 without
    saturating tanh, and an absolute tolerance on it means something."""
    from . import config as _config
    h = _config.hifigan_config(h)
    gain = dict(HIFIGAN_GAIN, **(gain or {}))
    spec = []
    c0, ch = int(h["upsample_initial_channel"]), int(h["upsample_initial_channel"])
    _conv(spec, "conv_pre", c0, int(h["num_mels"]), 7, wn=True, gain=gain["pre"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        _conv(spec, "ups.%d" % i, ch // 2, ch, k, wn=True, gain=gain["up"] * math.sqrt(u), transposed=True)
        ch //= 2
        for j, (ks, dils) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            n = i * len(h["resblock_kernel_sizes"]) + j
            for d in range(len(dils)):
                for m in ((1, 2) if h["resblock"] == "1" else ("",)):
                    _conv(spec, "resblocks.%d.convs%s.%d" % (n, m, d), ch, ch, ks, wn=True, gain=gain["rb"])
    _conv(spec, "conv_post", 1, ch, 7, wn=True, gain=gain["post"])
    return _draw(spec, seed)


HIFIGAN_GAIN = {"pre": 0.25, "up": 1.0, "rb": 0.5, "post": 0.05}   # v1 on a mel of -5.5 + 2.1 N(0, 1): max |wav| 0.67, mean 0.18


def make_random_bert(bt=None, seed=1234):
    """A BertModel state dict (CPU fp32) in transformers' names and shapes for the shape bt (config.bert_config; default
    rubert-base's), holding all num_hidden_layers = cv_layers + 2 layers as a checkpoint does, every tensor seeded by its name.
    Weights are drawn at 1 / sqrt(fan-in), embeddings at 0.5, LayerNorm affines around (1, 0)."""
    from . import config as _config
    bt = bt or _config.bert_config()
    H, F = bt["cv_hidden"], bt["cv_ffn"]
    out = []
    ln = lambda name, c: out.extend([(name + ".weight", (c,), "gamma", 0.1), (name + ".bias", (c,), "normal", 0.1)])
    e = "embeddings."
    for n, rows in (("word", bt["bt_vocab"]), ("position", bt["bt_max_pos"]), ("token_type", bt["bt_type_rows"])):
        out.append((e + n + "_embeddings.weight", (rows, H), "normal", 0.5))
    ln(e + "LayerNorm", H)
    for l in range(bt["cv_layers"] + _config.BERT_DROPPED_LAYERS):
        p = "encoder.layer.%d." % l
        for n in ("query", "key", "value"):
            _conv(out, p + "attention.self." + n, H, H, 1, gain=1.5 if n != "value" else 1.0)
        _conv(out, p + "attention.output.dense", H, H, 1)
        ln(p + "attention.output.LayerNorm", H)
        _conv(out, p + "intermediate.dense", F, H, 1)
        _conv(out, p + "output.dense", H, F, 1)
        ln(p + "output.LayerNorm", H)
    sd = _draw(out, seed)
    for name, shape, _, _ in out:
        if len(shape) == 3 and shape[2] == 1:
            sd[name] = sd[name][:, :, 0].contiguous()          # the Linear layers: [out, in]
    return sd


def make_random_t2s(cfg, seed=1234, eos_scale=1.0):
    """A Text2SemanticDecoder state dict (CPU fp32) in the reference's names for the shape cfg (config.t2s_config), every tensor
    seeded by its name.  Weights are drawn at 1 / sqrt(fan-in), embeddings at 0.5, LayerNorm affines around (1, 0), alphas
    around 1.  eos_scale multiplies the EOS row of ar_predict_layer: above 1 a seeded model stops sooner (its EOS logit
    spreads further), 0 never lets EOS win."""
    H, F, V, PV = cfg["cv_hidden"], cfg["cv_ffn"], cfg["t2s_vocab"], cfg["t2s_phone_vocab"]
    out = [("ar_text_embedding.word_embeddings.weight", (PV, H), "normal", 0.5),
           ("ar_audio_embedding.word_embeddings.weight", (V, H), "normal", 0.5),
           ("ar_text_position.alpha", (1,), "gamma", 0.1), ("ar_audio_position.alpha", (1,), "gamma", 0.1)]
    _conv(out, "bert_proj", H, 1024, 1)
    _conv(out, "ar_predict_layer", V, H, 1, bias=False, gain=2.0)
    ln = lambda name: out.extend([(name + ".weight", (H,), "gamma", 0.1), (name + ".bias", (H,), "normal", 0.1)])
    for l in range(cfg["cv_layers"]):
        p = "h.layers.%d." % l
        _conv(out, p + "self_attn.in_proj", 3 * H, H, 1, gain=1.5)
        _conv(out, p + "self_attn.out_proj", H, H, 1)
        _conv(out, p + "linear1", F, H, 1)
        _conv(out, p + "linear2", H, F, 1)
        ln(p + "norm1")
        ln(p + "norm2")
    sd = _draw(out, seed)
    for name, shape, _, _ in out:
        if len(shape) == 3 and shape[2] == 1:
            sd[name] = sd[name][:, :, 0].contiguous()
    for p in ("in_proj", ):
        for l in range(cfg["cv_layers"]):
            w = "h.layers.%d.self_attn.%s" % (l, p)
            sd[w + "_weight"], sd[w + "_bias"] = sd.pop(w + ".weight"), sd.pop(w + ".bias")
    sd["ar_predict_layer.weight"][V - 1] *= eos_scale
    return sd


def make_random_sovits(hubert, rows=None, seed=2525, codebook=1024, spacing=12):
    """The tensors of a GPT-SoVITS s2 checkpoint that the prompt's codes read (weights.load_sovits's state dict), seeded, for a
    HuBERT state dict `hubert` (make_random_contentvec): ssl_proj = Conv1d(768, 768, 2, stride 2) with PyTorch's default
    init scale and a bias on a 1/8 grid (a zero feature row then projects to exactly representable values), and a codebook
    drawn where projected speech lies, so that speech uses many codes (a codebook drawn without regard to it picks the few
    codewords of smallest norm).  rows [N, 768], HuBERT's rows of some recordings: codeword k < (N - 1) // spacing is ssl_proj
    of the rows (k spacing, k spacing + 1) plus noise of 1e-3 of the codewords' spread (rows `spacing` apart, so that
    neighbouring codewords are told apart by more than the rounding of an fp32 HuBERT).  The other codewords (all of them
    without rows) are ssl_proj of rows gamma * n + beta, n zero-mean unit-variance over the channels and gamma / beta the
    encoder's last LayerNorm affine.  inited = 1: the codebook is trained."""
    H = int(np.asarray(hubert["encoder.layer_norm.weight"]).shape[0])
    r = np.random.default_rng(seed)
    w = r.uniform(-1, 1, (H, H, 2)) / math.sqrt(2 * H)
    b = np.round(r.normal(0, 0.1, H) * 8) / 8
    last = "encoder.layers.%d.final_layer_norm." % (sum(1 for k in hubert if k.endswith(".final_layer_norm.weight")) - 1)
    gamma = np.asarray(hubert[last + "weight"], np.float64)
    beta = np.asarray(hubert[last + "bias"], np.float64)
    z = r.standard_normal((2, codebook, H))
    z = (z - z.mean(2, keepdims=True)) / z.std(2, keepdims=True)
    x0, x1 = gamma * z[0] + beta, gamma * z[1] + beta
    n = 0
    if rows is not None:
        rows = np.asarray(rows, np.float64)
        n = min(codebook, (rows.shape[0] - 1) // spacing)
        i = np.arange(n) * spacing
        x0[:n], x1[:n] = rows[i], rows[i + 1]
    E = x0 @ w[:, :, 0].T + x1 @ w[:, :, 1].T + b
    if n:
        E[:n] += 1e-3 * E[:n].std(0) * r.standard_normal((n, H))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))
    return {"ssl_proj.weight": t(w), "ssl_proj.bias": t(b), "quantizer.vq.layers.0._codebook.embed": t(E),
            "quantizer.vq.layers.0._codebook.inited": torch.ones(1)}
