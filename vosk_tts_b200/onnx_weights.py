"""Weights straight from a vosk-tts ``model.onnx`` (SURVEY.md section 8f rank 2(i)).

The deployed model directory ships only the ONNX graph (vosk_tts/model.py:46); the graph was traced from
``SynthesizerTrn.infer`` by training/vits2/onnx_export.py:47-104 after weight norm was removed, so its initializers ARE
the folded state dict: parameters consumed by Conv/Gather/Mul/Add keep their module names (``enc_p.emb.weight``,
``dec.ups.0.weight`` ...); the weight of an ``nn.Linear`` is exported as the transposed right operand of a MatMul
under an anonymous name (``onnx::MatMul_<n>``) and is recovered through the graph: the MatMul whose output feeds the
Add that consumes ``<module>.bias``.

The ``onnx`` package is not a dependency: ModelProto / GraphProto / TensorProto are read with the ~60-line protobuf
wire-format reader below (only the fields needed: graph=7; node=1, initializer=5; TensorProto dims=1, data_type=2,
float_data=4, int64_data=7, name=8, raw_data=9; NodeProto input=1, output=2, op_type=4, attribute=5 with
AttributeProto name=1, i=3, t=5, ints=8).

``stabletts_from_onnx`` reads a multistream (StableTTS) voice's model.onnx, the MatchaWithVocoder graph of
matcha/onnx/export.py, the same way (DESIGN.md section 4.q).
"""
import re
import struct

import numpy as np

_DTYPES = {1: np.float32, 6: np.int32, 7: np.int64, 10: np.float16, 11: np.float64, 9: np.bool_}


def _varint(buf, pos):
    out, shift = 0, 0
    while True:
        if pos >= len(buf):
            raise ValueError("truncated protobuf varint")
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7


def _fields(buf):
    """Yields (field_number, wire_type, value) of one message; length-delimited values are memoryviews."""
    pos, n = 0, len(buf)
    while pos < n:
        key, pos = _varint(buf, pos)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = bytes(buf[pos:pos + 8]); pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            v = buf[pos:pos + ln]; pos += ln
        elif wt == 5:
            v = bytes(buf[pos:pos + 4]); pos += 4
        else:
            raise ValueError("unsupported protobuf wire type %d" % wt)
        if pos > n:
            raise ValueError("truncated protobuf message")
        yield fno, wt, v


def _packed_varints(v):
    out, pos = [], 0
    while pos < len(v):
        x, pos = _varint(v, pos)
        out.append(x)
    return out


def _tensor(buf):
    dims, dtype, name, raw, floats, int64s = [], 1, "", None, None, []
    for fno, wt, v in _fields(buf):
        if fno == 1:
            dims += _packed_varints(v) if wt == 2 else [v]
        elif fno == 2:
            dtype = v
        elif fno == 8:
            name = bytes(v).decode()
        elif fno == 9:
            raw = v
        elif fno == 4:
            floats = np.frombuffer(v, np.float32) if wt == 2 else np.array([struct.unpack("<f", v)[0]], np.float32)
        elif fno == 7:
            int64s += _packed_varints(v) if wt == 2 else [v]
        elif fno == 14 and v == 1:
            raise ValueError("initializer %r uses external data; only self-contained model.onnx files are supported" % name)
    if dtype not in _DTYPES:
        return name, None
    dt = _DTYPES[dtype]
    if raw is not None:
        arr = np.frombuffer(raw, dt)
    elif floats is not None:
        arr = floats.astype(dt)
    elif int64s:
        arr = np.array(int64s, np.int64).astype(dt)
    else:
        arr = np.zeros(0, dt)
    return name, arr.reshape(dims) if dims else arr.reshape(())


def _attributes(buf):
    """(name, int or [ints] or ndarray) of one NodeProto.attribute entry: the integer attributes (strides, dilations) and the
    tensor-valued ones (a Constant node's value)."""
    name, ints, i, t = "", [], None, None
    for fno, wt, v in _fields(buf):
        if fno == 1:
            name = bytes(v).decode()
        elif fno == 8:
            ints += _packed_varints(v) if wt == 2 else [v]
        elif fno == 3 and wt == 0:
            i = v
        elif fno == 5 and wt == 2:
            t = _tensor(v)[1]
    return name, (t if t is not None else ints if ints else i)


def read_graph(path, with_attributes=False):
    """Returns (initializers {name: ndarray}, nodes [(op_type, inputs, outputs[, attrs])]) of a self-contained ONNX file."""
    with open(path, "rb") as f:
        data = memoryview(f.read())
    graph = None
    for fno, wt, v in _fields(data):
        if fno == 7 and wt == 2:
            graph = v
    if graph is None:
        raise ValueError("%s: no GraphProto (not an ONNX ModelProto?)" % path)
    inits, nodes = {}, []
    for fno, wt, v in _fields(graph):
        if fno == 5 and wt == 2:
            name, arr = _tensor(v)
            if arr is not None:
                inits[name] = arr
        elif fno == 1 and wt == 2:
            op, ins, outs, attrs = "", [], [], {}
            for f2, w2, v2 in _fields(v):
                if f2 == 1:
                    ins.append(bytes(v2).decode())
                elif f2 == 2:
                    outs.append(bytes(v2).decode())
                elif f2 == 4:
                    op = bytes(v2).decode()
                elif f2 == 5 and with_attributes:
                    k, val = _attributes(v2)
                    attrs[k] = val
            nodes.append((op, ins, outs, attrs) if with_attributes else (op, ins, outs))
    return inits, nodes


def state_dict_from_onnx(path):
    """Folded (weight-norm-free) state dict of the VITS graph in ``path``: {module-style name: float32 ndarray}.

    Named initializers are taken as they are; every ``<module>.bias`` that an Add combines with the output of a MatMul
    whose right operand is an anonymous 2-D initializer yields ``<module>.weight`` = that operand transposed (nn.Linear)."""
    inits, nodes = read_graph(path) if isinstance(path, (str, bytes)) or hasattr(path, "__fspath__") else path
    nodes = [n[:3] for n in nodes]
    sd = {k: np.ascontiguousarray(v) for k, v in inits.items() if not k.startswith("onnx::") and v.dtype == np.float32 and v.ndim >= 1}
    producer = {}
    for op, ins, outs in nodes:
        for o in outs:
            producer[o] = (op, ins)
    for op, ins, outs in nodes:
        if op != "Add" or len(ins) != 2:
            continue
        for bias_name, other in ((ins[0], ins[1]), (ins[1], ins[0])):
            if bias_name.endswith(".bias") and bias_name in inits and other in producer and producer[other][0] == "MatMul":
                w_name = producer[other][1][1]
                if w_name in inits and inits[w_name].ndim == 2 and inits[w_name].shape[1] == inits[bias_name].shape[0]:
                    sd[bias_name[:-len("bias")] + "weight"] = np.ascontiguousarray(inits[w_name].T)
    # ElementwiseAffine (modules.py:296): the reverse pass computes exp(-logs) and the exporter folds the negation into an
    # anonymous constant, so ``<flow>.logs`` = -(the Exp operand) for every ``<flow>.m`` that lost its sibling
    lost = [k[:-1] + "logs" for k in sd if k.endswith(".m") and (k[:-1] + "logs") not in sd]
    exps = [inits[ins[0]] for op, ins, outs in nodes if op == "Exp" and ins and ins[0].startswith("onnx::") and ins[0] in inits]
    for name in lost:
        cands = [e for e in exps if e.shape == sd[name[:-4] + "m"].shape]
        if len(cands) == 1:
            sd[name] = np.ascontiguousarray(-cands[0])
    return sd


def _count(sd, pattern):
    rx = re.compile(pattern)
    return len({m.group(1) for k in sd for m in [rx.match(k)] if m})


def _hifigan_shape(sd, attr_of, p):
    """The HiFi-GAN Generator's shape (config keys upsample_* and resblock*) of the weights under prefix p: widths and kernels
    from the tensors, upsampling rates and dilations from the strides / dilations of the (Conv)Transpose nodes."""
    q = re.escape(p)
    n_ups = _count(sd, q + r"ups\.(\d+)\.weight")
    one = p + "resblocks.0.convs1.0.weight" in sd
    stem = "convs1" if one else "convs"
    nk = _count(sd, q + r"resblocks\.(\d+)\.convs1?\.0\.weight") // max(n_ups, 1)
    dil = []
    for j in range(nk):
        n_conv = _count(sd, q + r"resblocks\.%d\.%s\.(\d+)\.weight" % (j, stem))
        dil.append([int((attr_of[p + "resblocks.%d.%s.%d.weight" % (j, stem, m)][1].get("dilations") or [1])[0]) for m in range(n_conv)])
    return {"upsample_initial_channel": int(sd[p + "conv_pre.weight"].shape[0]),
            "upsample_kernel_sizes": [int(sd[p + "ups.%d.weight" % i].shape[2]) for i in range(n_ups)],
            "upsample_rates": [int(attr_of[p + "ups.%d.weight" % i][1]["strides"][0]) for i in range(n_ups)],
            "resblock": "1" if one else "2",
            "resblock_kernel_sizes": [int(sd[p + "resblocks.%d.%s.0.weight" % (j, stem)].shape[2]) for j in range(nk)],
            "resblock_dilation_sizes": dil}


def config_from_onnx(path, sampling_rate=22050):
    """Engine configuration (vosk_tts_b200.config.DEFAULT_CONFIG keys) recovered from the tensor shapes of the graph's
    initializers plus the strides / dilations of its Conv / ConvTranspose nodes -- a deployed model directory carries no
    training json.  ``cond_layer_idx`` (attentions.py:41) and the spline tail bound (models.py:1625) are not encoded in
    any shape and keep the reference's constants."""
    from . import config as _config
    inits, nodes = read_graph(path, with_attributes=True)
    sd = state_dict_from_onnx((inits, nodes))
    attr_of = {}                         # weight initializer name -> attributes of the conv node that consumes it
    for op, ins, outs, attrs in nodes:
        if op in ("Conv", "ConvTranspose") and len(ins) >= 2:
            attr_of[ins[1]] = (op, attrs)
    cfg = dict(_config.DEFAULT_CONFIG)
    cfg["sampling_rate"] = sampling_rate
    cfg["n_vocab"], cfg["hidden_channels"] = (int(x) for x in sd["enc_p.emb.weight"].shape)
    if "emb_g.weight" in sd:
        cfg["n_speakers"], cfg["gin_channels"] = (int(x) for x in sd["emb_g.weight"].shape)
    else:
        cfg["n_speakers"], cfg["gin_channels"] = 0, 0
    cfg["n_layers"] = _count(sd, r"enc_p\.encoder\.attn_layers\.(\d+)\.conv_q\.weight")
    rel = sd["enc_p.encoder.attn_layers.0.emb_rel_k"]
    cfg["window_size"] = (int(rel.shape[1]) - 1) // 2
    cfg["n_heads"] = cfg["hidden_channels"] // int(rel.shape[2])
    f1 = sd["enc_p.encoder.ffn_layers.0.conv_1.weight"]
    cfg["filter_channels"], cfg["kernel_size"] = int(f1.shape[0]), int(f1.shape[2])
    cfg["inter_channels"] = int(sd["enc_p.proj.weight"].shape[0]) // 2
    cfg["use_spk_conditioned_encoder"] = "enc_p.encoder.spk_emb_linear.weight" in sd
    # stochastic duration predictor: flows = [EA, (ConvFlow, Flip) x n]; the reverse graph keeps ConvFlows 3, 5, ...
    cfg["dp_filter_channels"] = int(sd["dp.pre.weight"].shape[0])
    cf = sorted(int(k.split(".")[2]) for k in sd if k.startswith("dp.flows.") and k.endswith(".proj.weight"))
    cfg["dp_n_flows"] = (cf[-1] + 1) // 2
    cfg["dp_kernel_size"] = int(sd["dp.flows.%d.convs.convs_sep.0.weight" % cf[-1]].shape[2])
    cfg["dp_num_bins"] = (int(sd["dp.flows.%d.proj.weight" % cf[-1]].shape[0]) + 1) // 3
    # coupling flows: flows = [(coupling, Flip) x n]
    cfg["flow_n_flows"] = _count(sd, r"flow\.flows\.(\d+)\.enc\.in_layers\.0\.weight")
    cfg["flow_wn_layers"] = _count(sd, r"flow\.flows\.0\.enc\.in_layers\.(\d+)\.weight")
    w_in = "flow.flows.0.enc.in_layers.0.weight"
    cfg["flow_kernel_size"] = int(sd[w_in].shape[2])
    cfg["flow_dilation_rate"] = 1
    if cfg["flow_wn_layers"] > 1:
        d = attr_of.get("flow.flows.0.enc.in_layers.1.weight", ("", {}))[1].get("dilations")
        cfg["flow_dilation_rate"] = int(d[0]) if d else 1
    cfg["use_transformer_flows"] = any(k.startswith("flow.flows.0.pre_transformer.") for k in sd)
    cfg["transformer_flow_type"] = "pre_conv2"
    # decoder
    # OnnxSTFT's inverse basis [n_fft+2, 1, n_fft] (stft.py:191-214): an anonymous constant or the buffer ``dec.stft.inverse_basis``
    basis = [(k, v) for k, v in inits.items() if (k.startswith("onnx::ConvTranspose") or k.endswith("inverse_basis"))
             and v.ndim == 3 and v.shape[1] == 1 and v.shape[0] == v.shape[2] + 2 and k in attr_of]
    if "dec.multistream_conv_post.weight" in sd:
        cfg["decoder"] = "ms_istft"
    elif "dec.subband_conv_post.weight" in sd:
        cfg["decoder"] = "mb_istft"
    elif basis and "dec.conv_post.weight" in sd:
        cfg["decoder"] = "istft"
    else:
        cfg["decoder"] = "hifigan"
    cfg.update(_hifigan_shape(sd, attr_of, "dec."))
    if cfg["decoder"] != "hifigan":
        if len(basis) != 1:
            raise ValueError("cannot locate the inverse-STFT basis of the decoder in the graph")
        n_fft = int(basis[0][1].shape[2])
        cfg["gen_istft_n_fft"] = n_fft
        cfg["gen_istft_hop_size"] = int(attr_of[basis[0][0]][1]["strides"][0])
        post = "dec.conv_post.weight" if cfg["decoder"] == "istft" else "dec.subband_conv_post.weight"
        cfg["subbands"] = int(sd[post].shape[0]) // (n_fft + 2)
    if not cfg["use_transformer_flows"]:
        raise ValueError("plain coupling flows are unreachable through the reference exporter; unexpected graph")
    return cfg


NOT_EXPORT = "the exported graph is not built as matcha/onnx/export.py builds it"


def stabletts_from_onnx(path):
    """A multistream voice's model.onnx -- matcha/onnx/export.py's MatchaWithVocoder: MatchaTTS.synthesise with n_timesteps
    unrolled, then the HiFi-GAN -- read back into what StableTTS takes.  Returns a dict:
      state_dict     MatchaTTS's tensors in the checkpoint's names (the "matcha." prefix dropped), weight_norm-free;
      vocoder        the Generator's tensors (the "vocoder." prefix dropped), as remove_weight_norm left them;
      config         config.stabletts_config of the graph's shapes (widths, layer and head counts, streams, speakers);
      vocoder_config config.hifigan_config of the Generator's shapes and its (Conv)Transpose nodes' strides and dilations;
      n_timesteps    the Euler steps the graph unrolls.
    The exporter keeps every parameter under its module name, and that includes the time conditioning (time_mlp, each
    block's film), fake_speaker and fake_content: it folds nothing that needs them.  nn.Linear layers on 3-D input
    (encoder.bert_proj.1) become a MatMul with the transposed weight as an anonymous initializer, recovered through the Add
    of its bias.  mel_mean and mel_std become anonymous scalars: the Mul and Add that denormalise the mel the vocoder reads.
    The graph has no mel encoder (encoder.encoder.*): it feeds only encoder_outputs, which the graph does not return.
    Anything else is refused with a ValueError that names the reason."""
    def refuse(reason):
        raise ValueError("%s: %s: %s" % (path, NOT_EXPORT, reason))
    try:
        inits, nodes = read_graph(path, with_attributes=True)
    except (ValueError, UnicodeDecodeError, struct.error) as e:
        refuse("not a readable self-contained ONNX model (%s)" % e)
    sd = state_dict_from_onnx((inits, nodes))
    if any(k.startswith(("enc_p.", "dec.")) for k in sd):
        refuse("it holds a VITS model (enc_p.*, dec.*), not MatchaWithVocoder")
    if "encoder.emb.weight" in sd:
        refuse("it is a mel-only export without the vocoder (MatchaTTS at the top level); the engine needs the graph with the "
               "HiFi-GAN embedded")
    mt = {k[len("matcha."):]: v for k, v in sd.items() if k.startswith("matcha.")}
    voc = {k[len("vocoder."):]: v for k, v in sd.items() if k.startswith("vocoder.")}
    if "encoder.emb.weight" not in mt or "conv_pre.weight" not in voc:
        refuse("it has no matcha.encoder.emb.weight or no vocoder.conv_pre.weight")
    if "spk_emb.weight" not in mt:
        refuse("a single-speaker model (no spk_emb): the engine's StableTTS is conditioned on a speaker embedding")
    e = "decoder.estimator."
    for k in (e + "time_mlp.layer.0.weight", e + "blocks.0.time_fusion.film.weight", "fake_speaker", "fake_content",
              "encoder.bert_proj.1.weight", "encoder.dp_encoder.proj.weight"):
        if k not in mt:
            refuse("matcha.%s is missing (folded into constants or not exported)" % k)
    producer, consumers, const = {}, {}, {}
    for i, (op, ins, outs, attrs) in enumerate(nodes):
        for o in outs:
            producer[o] = i
        for x in ins:
            consumers.setdefault(x, []).append(i)
        if op == "Constant" and isinstance(attrs.get("value"), np.ndarray):
            const[outs[0]] = attrs["value"]
    const.update(inits)
    attr_of = {ins[1]: (op, attrs) for op, ins, outs, attrs in nodes if op in ("Conv", "ConvTranspose") and len(ins) >= 2}

    def uses(name, op):
        return [i for i in consumers.get(name, []) if nodes[i][0] == op]

    def heads(w_name, width):
        # MultiHeadAttention views conv_q's output as [b, n_heads, k_channels, t]: a Reshape whose shape is a Concat of
        # the dynamic b, the constants n_heads and k_channels, and the dynamic t
        convs = uses(w_name, "Conv")
        for r in (uses(nodes[convs[0]][2][0], "Reshape") if convs else []):
            cat = nodes[producer[nodes[r][1][1]]] if nodes[r][1][1] in producer else None
            if cat and cat[0] == "Concat" and len(cat[1]) == 4 and all(x in const for x in cat[1][1:3]):
                h, dk = (int(np.asarray(const[x]).reshape(-1)[0]) for x in cat[1][1:3])
                if h * dk == width:
                    return h
        refuse("cannot read the head count of %s from its Reshape" % w_name)

    # mel = decoder_outputs * mel_std + mel_mean (matcha/utils/model.py denormalize) is what the vocoder's conv_pre reads
    add = nodes[producer.get(nodes[uses("vocoder.conv_pre.weight", "Conv")[0]][1][0], 0)]
    scal = lambda x: x in inits and inits[x].size == 1 and inits[x].dtype == np.float32
    mul = nodes[producer[add[1][0]]] if add[0] == "Add" and add[1][0] in producer else None
    if not (mul and mul[0] == "Mul" and scal(add[1][1]) and scal(mul[1][1])):
        refuse("the vocoder's input is not the denormalised mel (x * mel_std + mel_mean)")
    mt["mel_std"], mt["mel_mean"] = inits[mul[1][1]].reshape(()), inits[add[1][1]].reshape(())
    # the estimator runs twice per Euler step (the conditional and the guidance branch, flow_matching.py:179-194)
    passes = len(uses("matcha." + e + "in_proj.weight", "Conv"))
    if passes < 2 or passes % 2:
        refuse("%d estimator passes, not two per Euler step" % passes)
    dp, f1 = "encoder.dp_encoder.encoder.", mt[e + "blocks.0.block.mlp.conv_1.weight"]
    ef1 = mt[dp + "0.mlp.conv_1.weight"]
    n_blocks = _count(mt, re.escape(e) + r"blocks\.(\d+)\.block\.attn\.conv_q\.weight")
    n_enc = _count(mt, re.escape(dp) + r"(\d+)\.attn\.conv_q\.weight")
    cfg = {"noise_channels": int(mt[e + "final_proj.weight"].shape[0]), "cond_channels": int(mt[e + "cond_proj.0.weight"].shape[1]),
           "hidden_channels": int(mt[e + "in_proj.weight"].shape[0]), "filter_channels": int(f1.shape[0]),
           "kernel_size": int(f1.shape[2]), "n_layers": n_blocks,
           "n_heads": heads("matcha." + e + "blocks.0.block.attn.conv_q.weight", int(mt[e + "in_proj.weight"].shape[0])),
           "n_spks": int(mt["spk_emb.weight"].shape[0]), "spk_emb_dim": int(mt["spk_emb.weight"].shape[1]),
           "n_vocab": int(mt["encoder.emb.weight"].shape[0]), "emb_dim": int(mt["encoder.emb.weight"].shape[1]),
           "punc_dim": int(mt["encoder.punc_emb.weight"].shape[1]),
           "n_streams": 1 + len(uses("matcha.encoder.punc_emb.weight", "Gather")),
           "bert_dim": int(mt["encoder.bert_proj.1.weight"].shape[1]), "bert_proj_dim": int(mt["encoder.bert_proj.1.weight"].shape[0]),
           "enc_hidden_channels": int(mt[dp + "0.attn.conv_q.weight"].shape[0]), "enc_filter_channels": int(ef1.shape[0]),
           "enc_kernel_size": int(ef1.shape[2]), "enc_n_layers": n_enc,
           "enc_n_heads": heads("matcha." + dp + "0.attn.conv_q.weight", int(mt[dp + "0.attn.conv_q.weight"].shape[0])),
           "dur_channels": int(mt["encoder.dp_encoder.proj.weight"].shape[0])}
    h = _hifigan_shape({"vocoder." + k: v for k, v in voc.items()}, attr_of, "vocoder.")
    h["num_mels"] = int(voc["conv_pre.weight"].shape[1])
    from . import config as _config
    return {"state_dict": mt, "vocoder": voc, "config": _config.stabletts_config(cfg), "vocoder_config": _config.hifigan_config(h),
            "n_timesteps": passes // 2}
