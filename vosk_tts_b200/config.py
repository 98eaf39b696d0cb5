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
