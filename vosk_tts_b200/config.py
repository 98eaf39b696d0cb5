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
