"""Plain-function restatement of ContentVec's forward (transformers' HubertModel as vc/contentvec.py builds it, one clip, no
attention mask), in PyTorch CPU ops, in float32 or float64.  `sd` is a state dict in the reference's names with the positional
conv folded (weights.fold_contentvec_pos_conv); `cv` the shape (config.contentvec_config)."""
import math

import torch
import torch.nn.functional as F


def contentvec_units(sd, cv, wav, dtype=torch.float64, stages=None):
    """wav: 1-D samples.  Returns last_hidden_state [T, hidden].  stages: a dict that receives "feat" (the feature encoder's
    output [T, conv_dim]) and "enc_in" (the transformer's input after the positional conv and its LayerNorm [T, hidden])."""
    w = lambda k: torch.as_tensor(sd[k]).to(dtype)
    x = torch.as_tensor(wav).to(dtype).reshape(1, 1, -1)
    fe = "feature_extractor.conv_layers.%d."
    for i, (k, s) in enumerate(zip(cv["cv_conv_kernel"], cv["cv_conv_stride"])):
        x = F.conv1d(x, w(fe % i + "conv.weight"), stride=s)
        if i == 0:
            x = F.group_norm(x, x.shape[1], w(fe % 0 + "layer_norm.weight"), w(fe % 0 + "layer_norm.bias"), eps=cv["cv_gn_eps"])
        x = F.gelu(x)
    x = x[0].T                                                              # [T, C]
    if stages is not None:
        stages["feat"] = x
    eps = cv["cv_ln_eps"]
    ln = lambda t, p: F.layer_norm(t, t.shape[-1:], w(p + ".weight"), w(p + ".bias"), eps=eps)
    x = ln(x, "feature_projection.layer_norm")
    x = x @ w("feature_projection.projection.weight").T + w("feature_projection.projection.bias")
    pos = "encoder.pos_conv_embed.conv."
    K = cv["cv_pos_k"]
    p = F.conv1d(x.T[None], w(pos + "weight"), w(pos + "bias"), padding=K // 2, groups=cv["cv_pos_groups"])
    p = F.gelu(p[0, :, :-1] if K % 2 == 0 else p[0]).T
    x = ln(x + p, "encoder.layer_norm")
    if stages is not None:
        stages["enc_in"] = x
    T, H, nh = x.shape[0], cv["cv_hidden"], cv["cv_heads"]
    dk = H // nh
    for l in range(cv["cv_layers"]):
        pre = "encoder.layers.%d." % l
        lin = lambda t, n: t @ w(pre + n + ".weight").T + w(pre + n + ".bias")
        q = lin(x, "attention.q_proj").reshape(T, nh, dk).transpose(0, 1) * dk ** -0.5
        k = lin(x, "attention.k_proj").reshape(T, nh, dk).transpose(0, 1)
        v = lin(x, "attention.v_proj").reshape(T, nh, dk).transpose(0, 1)
        a = torch.softmax(q @ k.transpose(1, 2), dim=-1) @ v
        x = ln(x + lin(a.transpose(0, 1).reshape(T, H), "attention.out_proj"), pre + "layer_norm")
        h = F.gelu(lin(x, "feed_forward.intermediate_dense"))
        x = ln(x + lin(h, "feed_forward.output_dense"), pre + "final_layer_norm")
    return x


def flops_per_frame(cv, frames):
    """Multiply-adds x 2 of one clip of `frames` frames, per frame (the transformer's attention grows with the clip)."""
    C, H, Fh = cv["cv_conv_dim"], cv["cv_hidden"], cv["cv_ffn"]
    ks, ss = cv["cv_conv_kernel"], cv["cv_conv_stride"]
    per = 2.0 * C * ks[0] * math.prod(ss[1:])                           # layer 0 at its rate
    rate = math.prod(ss[1:])
    for k, s in zip(ks[1:], ss[1:]):
        rate //= s
        per += 2.0 * C * C * k * rate
    per += 2.0 * C * H
    per += 2.0 * H * (H // cv["cv_pos_groups"]) * cv["cv_pos_k"]
    per += cv["cv_layers"] * (2.0 * (4 * H * H + 2 * H * Fh) + 4.0 * frames * H)
    return per
