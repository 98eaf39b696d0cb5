"""Engine configuration = the ``model`` block of the reference training JSON
(/root/reference/training/vits2/configs/mb_istft_vits2_multi.json:42-79) plus
``n_vocab`` (training/vits2/text/symbols.py: 62 symbols) and ``n_speakers`` (json :37).

Constants that the reference hard-codes in ``SynthesizerTrn.__init__``
(training/vits2/models.py:1613-1625) are spelled out here: flow kernel 5, dilation 1,
4 WN layers, 4 flows; SDP filter 256, kernel 3, 4 flows (3 used in reverse, :94-95).
"""
import copy
import json

DEFAULT_CONFIG = {
    "n_vocab": 62,
    "n_speakers": 200,
    "gin_channels": 256,
    "inter_channels": 192,
    "hidden_channels": 192,
    "filter_channels": 768,
    "n_heads": 2,
    "n_layers": 6,
    "kernel_size": 3,
    "window_size": 4,
    "use_spk_conditioned_encoder": True,
    "cond_layer_idx": 2,
    "use_transformer_flows": True,
    "transformer_flow_type": "pre_conv2",
    "flow_n_heads": 2,               # heads of the flow's pre_transformer: hard-coded in the reference (models.py:355), NOT n_heads
    "flow_kernel_size": 5,
    "flow_dilation_rate": 1,
    "flow_wn_layers": 4,
    "flow_n_flows": 4,
    "dp_filter_channels": 256,
    "dp_kernel_size": 3,
    "dp_n_flows": 4,
    "dp_num_bins": 10,
    "dp_tail_bound": 5.0,
    "decoder": "mb_istft",           # "mb_istft" (Multiband_iSTFT_Generator) | "ms_istft" (Multistream_iSTFT_Generator) |
                                     # "istft" (iSTFT_Generator) | "hifigan" (Generator)
    "resblock": "1",
    "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "upsample_rates": [4, 4],
    "upsample_initial_channel": 512,
    "upsample_kernel_sizes": [16, 16],
    "subbands": 4,
    "gen_istft_n_fft": 16,
    "gen_istft_hop_size": 4,
    "sampling_rate": 22050,
    # input features of the posterior encoder enc_q (voice conversion only; json "data" block :2-15, models.py:1616)
    "use_mel_posterior_encoder": True,
    "filter_length": 1024,
    "hop_length": 256,
    "win_length": 1024,
    "n_mel_channels": 80,
    "mel_fmin": 0.0,
    "mel_fmax": None,                # None: sampling_rate / 2 (librosa.filters.mel)
    "spec_channels": 80,             # n_mel_channels (mel) or filter_length // 2 + 1 (linear spectrogram)
}


ISTFT_DECODERS = ("mb_istft", "ms_istft", "istft")      # decoders that end in conv_post -> exp / pi*sin -> inverse STFT


def from_training_json(path_or_dict, n_vocab=62):
    """Map a reference training config (json :42-79, :37) onto the engine config."""
    cfg = path_or_dict
    if not isinstance(cfg, dict):
        with open(path_or_dict) as f:
            cfg = json.load(f)
    m = cfg["model"]
    out = copy.deepcopy(DEFAULT_CONFIG)
    out["n_vocab"] = n_vocab
    out["n_speakers"] = cfg["data"].get("n_speakers", 0)
    out["sampling_rate"] = cfg["data"].get("sampling_rate", 22050)
    for k in ("gin_channels", "inter_channels", "hidden_channels", "filter_channels", "n_heads",
              "n_layers", "kernel_size", "resblock", "resblock_kernel_sizes",
              "resblock_dilation_sizes", "upsample_rates", "upsample_initial_channel",
              "upsample_kernel_sizes", "subbands", "gen_istft_n_fft", "gen_istft_hop_size"):
        if k in m:
            out[k] = m[k]
    out["use_spk_conditioned_encoder"] = bool(m.get("use_spk_conditioned_encoder", False))
    out["use_transformer_flows"] = bool(m.get("use_transformer_flows", False))
    # reference defaults (models.py:1561-1564): note the flow type defaults to "mono_layer_post_residual"
    out["transformer_flow_type"] = m.get("transformer_flow_type", "mono_layer_post_residual")
    # Only what the engine implements is accepted, with the reason up front instead of a KeyError inside pack():
    #  * use_sdp=False builds the deterministic DurationPredictor (models.py:1625-1628): not implemented;
    #  * use_transformer_flows=True needs "pre_conv2" (ResidualCouplingTransformersLayer2, models.py:329-396);
    #  * use_transformer_flows=False is the plain ResidualCouplingLayer + Flip stack ONLY when the flow type is not
    #    "mono_layer_post_residual": with that (default!) type the reference appends a MonoTransformerFlowLayer to
    #    every flow (models.py:716-734), which the engine does not have.
    if not bool(m.get("use_sdp", True)):
        raise ValueError("use_sdp=false (deterministic DurationPredictor, models.py:1627) is not supported by this engine")
    if out["use_transformer_flows"]:
        if out["transformer_flow_type"] != "pre_conv2":
            raise ValueError("transformer_flow_type %r not supported (only 'pre_conv2')" % out["transformer_flow_type"])
    elif out["transformer_flow_type"] == "mono_layer_post_residual":
        raise ValueError("use_transformer_flows=false with transformer_flow_type 'mono_layer_post_residual' (the reference "
                         "default) adds MonoTransformerFlowLayers to the flow (models.py:716-734): not supported")
    # posterior encoder input (voice conversion): the model block decides, as in onnx_export.py:38-45 / train.py:77, which
    # overwrite the data block's flag with it
    d = cfg["data"]
    out["use_mel_posterior_encoder"] = m.get("use_mel_posterior_encoder", False) is True
    for k in ("filter_length", "hop_length", "win_length", "n_mel_channels", "mel_fmin", "mel_fmax"):
        if k in d:
            out[k] = d[k]
    out["spec_channels"] = out["n_mel_channels"] if out["use_mel_posterior_encoder"] else out["filter_length"] // 2 + 1
    # same precedence as SynthesizerTrn.__init__ (models.py:1585-1606)
    if m.get("mb_istft_vits", False):
        out["decoder"] = "mb_istft"
    elif m.get("ms_istft_vits", False):
        out["decoder"] = "ms_istft"
    elif m.get("istft_vits", False):
        out["decoder"] = "istft"
        out["subbands"] = 1                     # iSTFT_Generator has a single band and no synthesis filter bank
    else:
        out["decoder"] = "hifigan"
    return out


def from_quickvc_json(path_or_dict):
    """Map a QuickVC config (vc/configs/quickvc.json) onto the engine config, model_family "quickvc".

    What the engine serves of it is SynthesizerTrn.infer (vc/models.py:862-872): the speaker encoder SpeakerEncoder
    (:728-767) with the target's mel front end (mel_spectrogram_torch, vc/convert.py:60-69), the content encoder enc_p, the
    reverse flow and the Multistream_iSTFT_Generator decoder.  Hard-coded in the reference, not in the json: the LSTM has 3
    layers with hidden = gin_channels = 256 over n_mel_channels inputs (models.py:842, SpeakerEncoder defaults :729); the
    content units are 768 wide (models.py:825, while the json's ssl_dim says 1024); enc_p is PosteriorEncoder(768, I, H, 5, 1, 16)
    without g; the flow is ResidualCouplingBlock(I, H, 5, 1, 4, gin) with 4 mean-only coupling layers (:840).  Only the published
    ms_istft_vits decoder with two upsampling stages is accepted (convt_pad)."""
    cfg = path_or_dict
    if not isinstance(cfg, dict):
        with open(path_or_dict) as f:
            cfg = json.load(f)
    m, d = cfg["model"], cfg["data"]
    if m.get("mb_istft_vits", False) or m.get("istft_vits", False) or not m.get("ms_istft_vits", False):
        raise ValueError("only the published QuickVC decoder (ms_istft_vits=true, Multistream_iSTFT_Generator) is supported; "
                         "mb_istft_vits / istft_vits are not")
    if int(m.get("gin_channels", 0)) != 256:
        raise ValueError("gin_channels must be 256: the speaker encoder's LSTM hidden size and embedding (models.py:842)")
    out = copy.deepcopy(DEFAULT_CONFIG)
    out["model_family"] = "quickvc"
    out["n_speakers"] = 0
    out["decoder"] = "ms_istft"
    out["unit_channels"] = 768
    for k in ("gin_channels", "inter_channels", "hidden_channels", "filter_channels", "resblock", "resblock_kernel_sizes",
              "resblock_dilation_sizes", "upsample_rates", "upsample_initial_channel", "upsample_kernel_sizes", "subbands",
              "gen_istft_n_fft", "gen_istft_hop_size"):
        if k in m:
            out[k] = m[k]
    for k in ("sampling_rate", "filter_length", "hop_length", "win_length", "n_mel_channels", "mel_fmin", "mel_fmax"):
        if k in d:
            out[k] = d[k]
    out["use_mel_posterior_encoder"] = True
    out["spec_channels"] = out["n_mel_channels"]
    out["spk_layers"] = 3
    out["use_transformer_flows"] = False
    out.update(flow_kernel_size=5, flow_dilation_rate=1, flow_wn_layers=4, flow_n_flows=4)
    if len(out["upsample_rates"]) != 2 or len(out["upsample_kernel_sizes"]) != 2:
        raise ValueError("the QuickVC decoder needs exactly two upsampling stages: its ConvTranspose1d output_padding = 1 - i "
                         "(vc/models.py:428-430) is negative past the second")
    for i in range(2):
        convt_pad(out, i)
    return out


STABLETTS_CFM = {
    # CFM.__init__ hard-codes the estimator (flow_matching.py:301); n_spks / spk_emb_dim and the mel statistics come from the
    # experiment's yaml (MatchaTTS.__init__, matcha_tts.py:28-38,92)
    "model_family": "stabletts",
    "noise_channels": 80, "cond_channels": 256, "hidden_channels": 384, "filter_channels": 768,
    "n_layers": 6, "n_heads": 4, "kernel_size": 3, "use_lsc": True,
    "n_spks": 2, "spk_emb_dim": 128,
    "solver": "euler",
}


def stabletts_cfm_config(overrides=None):
    """Engine config of the StableTTS flow-matching decoder, model_family "stabletts": the estimator's constants
    (flow_matching.py:301) with `overrides` (e.g. n_spks / spk_emb_dim of a checkpoint).  What is not built is refused with
    the reason."""
    out = copy.deepcopy(STABLETTS_CFM)
    out.update(overrides or {})
    H, heads, L = int(out["hidden_channels"]), int(out["n_heads"]), int(out["n_layers"])
    if not out.get("use_lsc", True):
        raise ValueError("use_lsc=false is not supported: the engine builds the U-Net long skips the reference always enables "
                         "(flow_matching.py:301)")
    if L < 2 or L % 2 or L > 8:
        raise ValueError("n_layers must be even and in 2..8: the long skips pair block i with block n_layers - 1 - i "
                         "(decoder.py:93-95)")
    if H % heads or (H // heads) not in (32, 64, 96, 128):
        raise ValueError("head width hidden_channels / n_heads must be 32, 64, 96 or 128: the attention kernels take no other")
    if out["solver"] != "euler":
        raise ValueError("only the fixed-step Euler solver is built (the reference's heun / midpoint / dopri5 paths are "
                         "commented out or unreachable, flow_matching.py:57-69)")
    if int(out["kernel_size"]) % 2 != 1:
        raise ValueError("kernel_size must be odd (padding = kernel_size // 2 keeps the length)")
    if H % 16 or H > 512 or int(out["filter_channels"]) % 16 or int(out["filter_channels"]) > 1024 or int(out["cond_channels"]) % 16 \
            or (int(out["noise_channels"]) + H) % 16 or int(out["noise_channels"]) % 4:
        raise ValueError("channel widths must be multiples of 16 (noise_channels of 4, noise + hidden of 16), hidden up to 512, "
                         "filter up to 1024: the FFMA conv and LayerNorm kernels' tiles")
    if int(out["n_spks"]) < 1 or not 1 <= int(out["spk_emb_dim"]) <= 1024:
        raise ValueError("n_spks must be >= 1 and spk_emb_dim in 1..1024")
    return out


STABLETTS_TEXT = {
    # TextEncoder.__init__ hard-codes both stacks and the embedding widths (text_encoder.py:72-106); n_vocab comes from the
    # experiment's yaml
    "n_vocab": 178, "n_streams": 5, "emb_dim": 160, "punc_dim": 16, "bert_dim": 768, "bert_proj_dim": 32,
    "enc_hidden_channels": 256, "enc_filter_channels": 1024, "enc_n_layers": 4, "enc_n_heads": 4, "enc_kernel_size": 3,
    "dur_channels": 50,
}


def stabletts_config(overrides=None):
    """Engine config of StableTTS text-to-mel: stabletts_cfm_config plus the text encoder's constants (STABLETTS_TEXT) with
    `overrides` (n_vocab, n_spks, ... of a checkpoint)."""
    out = stabletts_cfm_config(dict(STABLETTS_TEXT, **(overrides or {})))
    H, heads = int(out["enc_hidden_channels"]), int(out["enc_n_heads"])
    if int(out["emb_dim"]) + (int(out["n_streams"]) - 1) * int(out["punc_dim"]) + int(out["bert_proj_dim"]) != int(out["cond_channels"]) \
            or H != int(out["cond_channels"]):
        raise ValueError("emb_dim + (n_streams - 1) punc_dim + bert_proj_dim must equal cond_channels and enc_hidden_channels: the "
                         "concatenated embedding is both stacks' input and the decoder's mu (text_encoder.py:131, matcha_tts.py:170)")
    if H % heads or (H // heads) not in (32, 64, 96, 128):
        raise ValueError("head width enc_hidden_channels / enc_n_heads must be 32, 64, 96 or 128: the attention kernels take no other")
    if not 1 <= int(out["enc_n_layers"]) <= 8 or int(out["enc_kernel_size"]) % 2 != 1:
        raise ValueError("enc_n_layers must be in 1..8 and enc_kernel_size odd")
    if H % 16 or H > 512 or int(out["enc_filter_channels"]) % 16 or int(out["enc_filter_channels"]) > 1024:
        raise ValueError("encoder widths must be multiples of 16, hidden up to 512, filter up to 1024: the FFMA conv and LayerNorm "
                         "kernels' tiles")
    if not 1 <= int(out["bert_dim"]) <= 1024 or not 1 <= int(out["dur_channels"]) <= 1024 or int(out["n_vocab"]) < 1 \
            or not 1 <= int(out["n_streams"]) <= 8:
        raise ValueError("bert_dim and dur_channels must be in 1..1024, n_streams in 1..8, n_vocab >= 1")
    return out


# The HiFi-GAN vocoder StableTTS's cli.py:65-71 loads (hifigan_T2_v1 / hifigan_univ_v1): always config v1 of
# matcha/hifigan/config.py, its Generator reading 80 mel channels (models.py:154).
HIFIGAN_V1 = {
    "resblock": "1", "upsample_rates": [8, 8, 2, 2], "upsample_kernel_sizes": [16, 16, 4, 4], "upsample_initial_channel": 512,
    "resblock_kernel_sizes": [3, 7, 11], "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]], "num_mels": 80,
}


def hifigan_config(h=None):
    """The vocoder's shape from the reference's config-dict keys (HIFIGAN_V1 where `h` is None or leaves a key out).  Refuses,
    with the reason, what the engine does not build."""
    out = copy.deepcopy(HIFIGAN_V1)
    out.update({k: copy.deepcopy(v) for k, v in (h or {}).items() if k in HIFIGAN_V1})
    ur, uk, rk, rd = out["upsample_rates"], out["upsample_kernel_sizes"], out["resblock_kernel_sizes"], out["resblock_dilation_sizes"]
    if str(out["resblock"]) not in ("1", "2"):
        raise ValueError("resblock must be '1' or '2'")
    out["resblock"] = str(out["resblock"])
    if not 1 <= len(ur) <= 8 or len(uk) != len(ur) or any(k < u or (k - u) % 2 for u, k in zip(ur, uk)):
        raise ValueError("1..8 upsampling stages, each kernel >= its rate with kernel - rate even (padding (k - u) / 2 emits u T samples)")
    c0 = int(out["upsample_initial_channel"])
    if c0 % (1 << len(ur)) or (c0 >> len(ur)) % 16:
        raise ValueError("upsample_initial_channel must halve to a multiple of 16 at every stage (the FFMA conv's channel chunk)")
    if not 1 <= len(rk) <= 3 or len(rd) != len(rk) or len({len(d) for d in rd}) != 1 or not 1 <= len(rd[0]) <= 8:
        raise ValueError("1..3 resblock kernels per stage, each with the same number (1..8) of dilations")
    if any(k % 2 == 0 for k in rk):
        raise ValueError("resblock kernels must be odd")
    if int(out["num_mels"]) % 16:
        raise ValueError("num_mels must be a multiple of 16 (the FFMA conv's channel chunk)")
    return out


def hop_samples(h):
    """Samples per mel frame of a vocoder config: the product of its upsampling rates (256 for v1)."""
    n = 1
    for u in h["upsample_rates"]:
        n *= int(u)
    return n


def convt_pad(cfg, i):
    """(padding, output_padding) of the decoder's upsampling ConvTranspose1d of stage i: (K-u)//2 and 0 in VITS2
    (training/vits2/models.py, every generator), (K-u+1-i)//2 and 1-i in QuickVC (vc/models.py:428-430).  The engine lays out
    u*T output rows per stage, so the stage must emit exactly that many: K - u + output_padding == 2 * padding."""
    u, K = cfg["upsample_rates"][i], cfg["upsample_kernel_sizes"][i]
    if cfg.get("model_family", "vits2") == "quickvc":
        p, op = (K - u + 1 - i) // 2, 1 - i
        if K - u + op != 2 * p:
            raise ValueError("upsampling stage %d (rate %d, kernel %d) would emit %d frames per input frame plus %d, not exactly %d"
                             % (i, u, K, u, K - u + op - 2 * p, u))
        return p, op
    return (K - u) // 2, 0


def hop_total(cfg):
    """Output samples per latent frame (256 for the reference config)."""
    up = 1
    for u in cfg["upsample_rates"]:
        up *= u
    if cfg["decoder"] in ISTFT_DECODERS:
        up *= cfg["gen_istft_hop_size"] * cfg["subbands"]
    return up


# ContentVec (vc/contentvec.py: HubertModelWithFinalProj(HubertConfig(conv_bias=False, classifier_proj_size=256))): the defaults
# of transformers' HubertConfig, which are hubert-base's.
CONTENTVEC_DEFAULTS = {
    "hidden_size": 768, "num_hidden_layers": 12, "num_attention_heads": 12, "intermediate_size": 3072, "hidden_act": "gelu",
    "feat_extract_norm": "group", "feat_extract_activation": "gelu", "conv_dim": [512] * 7,
    "conv_stride": [5, 2, 2, 2, 2, 2, 2], "conv_kernel": [10, 3, 3, 3, 3, 2, 2], "conv_bias": False,
    "num_conv_pos_embeddings": 128, "num_conv_pos_embedding_groups": 16, "do_stable_layer_norm": False,
    "feat_proj_layer_norm": True, "layer_norm_eps": 1e-5,
}
CV_GN_EPS = 1e-5          # HubertGroupNormConvLayer's nn.GroupNorm default


def contentvec_config(path_or_dict=None):
    """The engine's ContentVec shape (cv_* keys) from a Hugging Face HubertConfig config.json (None: the defaults).  Refuses, with
    the reason, what the engine does not compute."""
    cfg = dict(CONTENTVEC_DEFAULTS)
    if path_or_dict is not None:
        src = path_or_dict
        if not isinstance(src, dict):
            with open(path_or_dict) as f:
                src = json.load(f)
        cfg.update({k: src[k] for k in CONTENTVEC_DEFAULTS if k in src})
    if cfg["feat_extract_norm"] != "group":
        raise ValueError("feat_extract_norm %r: only 'group' (GroupNorm after the first conv) is supported" % cfg["feat_extract_norm"])
    if cfg["do_stable_layer_norm"]:
        raise ValueError("do_stable_layer_norm=true (pre-LN transformer) is not supported: ContentVec is post-LN")
    if cfg["conv_bias"]:
        raise ValueError("conv_bias=true is not supported: ContentVec's feature encoder has no conv bias")
    if not cfg["feat_proj_layer_norm"]:
        raise ValueError("feat_proj_layer_norm=false is not supported")
    for k in ("hidden_act", "feat_extract_activation"):
        if cfg[k] != "gelu":
            raise ValueError("%s %r: only 'gelu' is supported" % (k, cfg[k]))
    dims, ks, ss = list(cfg["conv_dim"]), list(cfg["conv_kernel"]), list(cfg["conv_stride"])
    if not (2 <= len(dims) <= 8 and len(ks) == len(dims) == len(ss)) or len(set(dims)) != 1 or dims[0] % 16 or dims[0] > 1024:
        raise ValueError("the feature encoder needs 2..8 convs of one width, a multiple of 16 up to 1024")
    if any(s != 2 for s in ss[1:]):
        raise ValueError("conv strides after the first must be 2 (got %s)" % ss[1:])
    if not 1 <= ks[0] <= 16:
        raise ValueError("the first conv's kernel must be 1..16")
    H, nh = cfg["hidden_size"], cfg["num_attention_heads"]
    if H % nh or (H // nh) % 32 or H // nh > 128 or H > 1024:
        raise ValueError("head dim %s is not one the attention kernels take (a multiple of 32 up to 128)" % (H / nh))
    pk, pg = cfg["num_conv_pos_embeddings"], cfg["num_conv_pos_embedding_groups"]
    if pk % 2:
        raise ValueError("num_conv_pos_embeddings must be even (got %d)" % pk)
    if pk > 130 or H % pg or (H // pg) % 16:
        raise ValueError("positional conv of %d taps in %d groups is not supported (up to 130 taps, groups a multiple of 16 wide)" % (pk, pg))
    return {"cv_layers": cfg["num_hidden_layers"], "cv_hidden": H, "cv_heads": nh, "cv_ffn": cfg["intermediate_size"],
            "cv_conv_dim": dims[0], "cv_conv_kernel": ks, "cv_conv_stride": ss, "cv_pos_k": pk, "cv_pos_groups": pg,
            "cv_ln_eps": float(cfg["layer_norm_eps"]), "cv_gn_eps": CV_GN_EPS}


def contentvec_frames(n_samples, cv=None):
    """Frames ContentVec gives a clip of n_samples (0: too short): L0 = (n - k0) // s0 + 1, then L_i = (L_{i-1} - k_i) // s_i + 1."""
    cv = cv or contentvec_config()
    L = None
    for k, s in zip(cv["cv_conv_kernel"], cv["cv_conv_stride"]):
        n = n_samples if L is None else L
        L = (n - k) // s + 1 if n >= k else 0
    return max(L, 0)


# BERT as training/stabletts/matcha/onnx/bert-export.py exports it (transformers' BertModel returning hidden_states[-3]): the
# defaults of BertConfig, which are rubert-base's shape.
BERT_DEFAULTS = {
    "hidden_size": 768, "num_hidden_layers": 12, "num_attention_heads": 12, "intermediate_size": 3072, "hidden_act": "gelu",
    "layer_norm_eps": 1e-12, "vocab_size": 30522, "max_position_embeddings": 512, "type_vocab_size": 2,
    "position_embedding_type": "absolute",
}
BERT_DROPPED_LAYERS = 2   # hidden_states[-3] is the output of layer n_layers - 2: the last two layers never run


def bert_config(path_or_dict=None, layers=None):
    """The engine's BERT shape (cv_* keys for the transformer, bt_* for the embeddings) from a Hugging Face BertConfig
    config.json (None: the defaults).  cv_layers is the number of layers that run: `layers` when given (what an exported graph
    holds), else num_hidden_layers - 2.  Refuses, with the reason, what the engine does not compute."""
    cfg = dict(BERT_DEFAULTS)
    if path_or_dict is not None:
        src = path_or_dict
        if not isinstance(src, dict):
            with open(path_or_dict) as f:
                src = json.load(f)
        cfg.update({k: src[k] for k in BERT_DEFAULTS if k in src and src[k] is not None})
    if cfg["hidden_act"] != "gelu":
        raise ValueError("hidden_act %r: only 'gelu' (erf) is supported" % cfg["hidden_act"])
    if cfg["position_embedding_type"] != "absolute":
        raise ValueError("position_embedding_type %r: only 'absolute' is supported" % cfg["position_embedding_type"])
    H, nh, F = int(cfg["hidden_size"]), int(cfg["num_attention_heads"]), int(cfg["intermediate_size"])
    if H % nh or (H // nh) % 32 or H // nh > 128 or H % 16 or H > 1024:
        raise ValueError("hidden_size %d / %d heads: the attention kernels take head widths that are multiples of 32 up to 128, "
                         "and the LayerNorm kernel widths up to 1024" % (H, nh))
    if F % 16 or F < 16:
        raise ValueError("intermediate_size must be a positive multiple of 16")
    n = int(cfg["num_hidden_layers"]) - BERT_DROPPED_LAYERS if layers is None else int(layers)
    if n < 1:
        raise ValueError("no BERT layer would run (num_hidden_layers must be at least 3: hidden_states[-3] is layer n - 2)")
    if int(cfg["vocab_size"]) < 1 or int(cfg["max_position_embeddings"]) < 1 or int(cfg["type_vocab_size"]) < 1:
        raise ValueError("vocab_size, max_position_embeddings and type_vocab_size must be positive")
    return {"cv_layers": n, "cv_hidden": H, "cv_heads": nh, "cv_ffn": F, "cv_ln_eps": float(cfg["layer_norm_eps"]),
            "bt_vocab": int(cfg["vocab_size"]), "bt_max_pos": int(cfg["max_position_embeddings"]),
            "bt_type_rows": int(cfg["type_vocab_size"])}


T2S_MAX_POSITIONS = 4000     # rows of the sine table SinePositionalEmbedding builds at construction (embedding.py:48)


def t2s_config(model, sd=None):
    """The engine's GPT-SoVITS text-to-semantic shape (cv_* keys for the layers, t2s_* for the tables) from the `model` block
    of a checkpoint's config (Text2SemanticDecoder.__init__, ar/models/t2s_model.py:39-80), checked against the state dict's
    tensors when given.  Refuses, with the reason, what the engine does not compute."""
    H, E, nh, L = (int(model[k]) for k in ("hidden_dim", "embedding_dim", "head", "n_layer"))
    V, PV, EOS = int(model["vocab_size"]), int(model["phoneme_vocab_size"]), int(model["EOS"])
    if E != H:
        raise ValueError("embedding_dim %d != hidden_dim %d: the layers read the embeddings directly" % (E, H))
    if EOS != V - 1:
        raise ValueError("EOS %d != vocab_size - 1 (%d): the sampler takes EOS as the last logit" % (EOS, V - 1))
    if L < 1 or nh < 1 or H % nh or (H // nh) % 32 or H // nh > 128 or H % 16 or H > 1024:
        raise ValueError("hidden_dim %d / %d heads: the attention kernels take head widths that are multiples of 32 up to 128, "
                         "and the LayerNorm kernels widths up to 1024" % (H, nh))
    if 4 * H > 4096:
        raise ValueError("the FFN width 4 hidden_dim must be at most 4096")
    if V < 2 or V > 4096:
        raise ValueError("vocab_size %d: the sampler's block sort takes 2 to 4096 entries" % V)
    if PV < 1:
        raise ValueError("phoneme_vocab_size must be positive")
    if sd is not None:
        shapes = {"ar_text_embedding.word_embeddings.weight": (PV, H), "ar_audio_embedding.word_embeddings.weight": (V, H),
                  "ar_predict_layer.weight": (V, H), "bert_proj.weight": (H, 1024)}
        for k, shp in shapes.items():
            if k not in sd or tuple(sd[k].shape) != shp:
                raise ValueError("%s: expected shape %s, found %s" % (k, shp, None if k not in sd else tuple(sd[k].shape)))
        n = 0
        while "h.layers.%d.self_attn.in_proj_weight" % n in sd:
            n += 1
        if n != L:
            raise ValueError("the state dict holds %d layers, the config n_layer %d" % (n, L))
        if tuple(sd["h.layers.0.linear1.weight"].shape) != (4 * H, H):
            raise ValueError("linear1 must be [4 hidden_dim, hidden_dim] (dim_feedforward = 4 hidden_dim)")
    return {"model_family": "t2s", "cv_layers": L, "cv_hidden": H, "cv_heads": nh, "cv_ffn": 4 * H, "cv_ln_eps": 1e-5,
            "t2s_vocab": V, "t2s_phone_vocab": PV, "t2s_positions": T2S_MAX_POSITIONS}


# GPT-SoVITS SoVITS (SynthesizerTrn of training/gpt-sovits/module/models.py): what inference_cli.py:164-200 runs on a reference
# recording before text-to-semantic decoding.  The prompt's length limits are at 16 kHz (inference_cli.py:182).
SOVITS_PROMPT_MIN, SOVITS_PROMPT_MAX = 48000, 320000
SOVITS_PROMPT_MESSAGE = "Prompt audio length must be longer than 3 seconds and shorter than 20 seconds!"


def sovits_pad(sampling_rate):
    """Zeros appended to a 16 kHz prompt: int(hps.data.sampling_rate * 0.3) (inference_cli.py:176-192), counted at the s2
    model's rate although the samples they follow are at 16 kHz."""
    return int(sampling_rate * 0.3)


def sovits_config(s2_config, hubert_config=None, codebook=1024):
    """The engine's GPT-SoVITS SoVITS shape, model_family "sovits": the cv_* fields of the HuBERT (contentvec_config of its
    config.json, with its refusals; None: chinese-hubert-base's shape, HubertConfig's defaults), the quantizer's codebook
    entries (sv_codebook), and from the s2 config.json (path or dict) its data.sampling_rate and the prompt pad it implies."""
    src = s2_config
    if not isinstance(src, dict):
        with open(s2_config) as f:
            src = json.load(f)
    data = src.get("data") if isinstance(src, dict) else None
    if not isinstance(data, dict) or "sampling_rate" not in data:
        raise ValueError("the s2 config has no data.sampling_rate")
    sr = int(data["sampling_rate"])
    if sr <= 0:
        raise ValueError("data.sampling_rate must be positive (got %d)" % sr)
    if int(codebook) < 1 or int(codebook) > 65536:
        raise ValueError("the codebook must hold 1 to 65536 entries (got %d)" % int(codebook))
    out = {"model_family": "sovits", "sampling_rate": sr, "sovits_pad": sovits_pad(sr), "sv_codebook": int(codebook)}
    out.update(contentvec_config(hubert_config))
    return out
