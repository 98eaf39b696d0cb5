"""Restatement of GPT-SoVITS text-to-semantic decoding (Text2SemanticDecoder.infer_panel, training/gpt-sovits/
ar/models/t2s_model.py:324-448, and the sampler of ar/models/utils.py:110-161) in torch, in any float dtype, for the tests.

Without a KV cache: the logits of every sampling step come from one pass of the layer stack over [text; y] under the prefix
mask of infer_panel (key k is visible to query q iff k < T or k <= q), which is what the cached steps compute."""
import math

import numpy as np
import torch


def sine_table(n, dim, dtype):
    position = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe = torch.zeros(n, dim)
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.to(dtype)


def embed(w, cfg, phones, y, bert=None, dtype=torch.float64):
    """The rows [text; y] infer_panel feeds its layers (w: the state dict in dtype)."""
    x = torch.as_tensor(np.asarray(phones, np.int64))
    T = x.numel()
    y = torch.as_tensor(np.asarray(y, np.int64)).reshape(-1)
    pe = sine_table(max(T, y.numel()) + 1, cfg["cv_hidden"], dtype)
    xt = w["ar_text_embedding.word_embeddings.weight"][x]
    bp = torch.zeros(T, 1024, dtype=dtype) if bert is None else torch.as_tensor(np.asarray(bert)).to(dtype)
    xt = xt + (bp @ w["bert_proj.weight"].T + w["bert_proj.bias"])
    xt = xt + w["ar_text_position.alpha"] * pe[:T]
    ya = w["ar_audio_embedding.word_embeddings.weight"][y] + w["ar_audio_position.alpha"] * pe[:y.numel()]
    return torch.cat([xt, ya], 0)


def prefix_attention(qkv, T, nh):
    """The attention core of one layer on its qkv rows [n, 3H]: softmax(q k^T sqrt(1 / dk)) v per head under infer_panel's
    prefix mask (key k is visible to query q iff k < T or k <= q), [n, H]."""
    n, H = qkv.shape[0], qkv.shape[1] // 3
    dk = H // nh
    qi = torch.arange(n)[:, None]
    ki = torch.arange(n)[None, :]
    visible = (ki < T) | (ki <= qi)
    q, k, v = (qkv[:, i * H:(i + 1) * H].reshape(n, nh, dk).transpose(0, 1) for i in range(3))
    a = (q * math.sqrt(1.0 / dk)) @ k.transpose(1, 2)
    a = torch.softmax(a.masked_fill(~visible, float("-inf")), -1) @ v
    return a.transpose(0, 1).reshape(n, H)


def step_logits(sd, cfg, phones, y, bert=None, dtype=torch.float64, P=0):
    """Logits [len(y) - P + 1, V] of every sampling step along the token sequence y (its first P tokens the prompt, then the
    sampled tokens): step i reads row T + P + i - 1 of [text; y]."""
    w = {k: v.to(dtype) for k, v in sd.items()}
    H, nh, L = cfg["cv_hidden"], cfg["cv_heads"], cfg["cv_layers"]
    T = len(phones)
    h = embed(w, cfg, phones, y, bert, dtype)
    for l in range(L):
        p = "h.layers.%d." % l
        qkv = h @ w[p + "self_attn.in_proj_weight"].T + w[p + "self_attn.in_proj_bias"]
        a = prefix_attention(qkv, T, nh) @ w[p + "self_attn.out_proj.weight"].T + w[p + "self_attn.out_proj.bias"]
        h = torch.nn.functional.layer_norm(h + a, (H,), w[p + "norm1.weight"], w[p + "norm1.bias"], 1e-5)
        f = torch.relu(h @ w[p + "linear1.weight"].T + w[p + "linear1.bias"]) @ w[p + "linear2.weight"].T + w[p + "linear2.bias"]
        h = torch.nn.functional.layer_norm(h + f, (H,), w[p + "norm2.weight"], w[p + "norm2.bias"], 1e-5)
    return h[T + P - 1:] @ w["ar_predict_layer.weight"].T


def sample(logits, previous, top_k, top_p, temperature, penalty, q, eos=None):
    """ar.models.utils.sample restated on one step's logits (1-d, the EOS column already dropped at step 0) with the Exp(1)
    draws q.  Returns (token, argmax of the penalised logits, margins): margins = (logit gap at the top-k pivot, |cum - top_p|
    nearest the top-p cut, winner vs runner-up of probs / q in logit units (times the temperature), the gap between the EOS
    entry (index eos, when given and present) and the largest other penalised logit)."""
    l = logits.clone()
    prev = torch.as_tensor(np.asarray(previous, np.int64)).reshape(-1)
    if prev.numel():
        s = l[prev]
        l[prev] = torch.where(s < 0, s * penalty, s / penalty)
    pen = l.clone()
    big = float("inf")
    cut_margin = big
    if top_p < 1.0:
        sl, si = torch.sort(l, descending=True, stable=True)
        cum = torch.cumsum(torch.softmax(sl, -1), -1)
        rm = cum > top_p
        rm[0] = False
        cut_margin = float((cum[1:] - top_p).abs().min()) if cum.numel() > 1 else big
        l = l.masked_fill(rm.scatter(0, si, rm), float("-inf"))
    l = l / max(temperature, 1e-5)
    kk = min(top_k, l.numel())
    v = torch.topk(l, kk).values
    pivot = v[-1]
    srt = torch.sort(l[torch.isfinite(l)], descending=True).values
    piv_gap = float((srt[kk - 1] - srt[kk]) * max(temperature, 1e-5)) if srt.numel() > kk else big
    l = torch.where(l < pivot, float("-inf"), l)
    probs = torch.softmax(l, -1)
    sc = probs / torch.as_tensor(np.asarray(q)).to(probs.dtype)
    tok = int(torch.argmax(sc))
    top2 = torch.topk(sc, 2).values if sc.numel() > 1 else torch.stack([sc.max(), torch.zeros((), dtype=sc.dtype)])
    win = float(torch.log(top2[0] / top2[1]) * max(temperature, 1e-5)) if top2[1] > 0 else big
    pa = int(torch.argmax(pen))
    eos_gap = float((pen[eos] - pen[:eos].max()).abs()) if eos is not None and eos < pen.numel() else big
    return tok, pa, (piv_gap, cut_margin, win, eos_gap)


def decode(sd, cfg, phones, prompt=None, bert=None, q=None, top_k=20, top_p=0.6, temperature=0.6, penalty=1.35, early_stop=-1,
           step_cap=1500, dtype=torch.float64):
    """infer_panel at batch 1 with the Exp(1) draws q [steps, V] (step 0 reads the first V - 1).  Returns (y[:-1] with the
    prompt, idx, per-step margins, per-step logits)."""
    V = cfg["t2s_vocab"]
    P = 0 if prompt is None else len(prompt)
    y = [] if prompt is None else [int(t) for t in prompt]
    margins, lgs = [], []
    for i in range(step_cap):
        lg = step_logits(sd, cfg, phones, y, bert, dtype)[-1]
        lgs.append(lg.clone())
        if i == 0:
            lg = lg[:-1]
        tok, pa, m = sample(lg, y, top_k, top_p, temperature, penalty, q[i][:lg.numel()], eos=V - 1)
        margins.append(m)
        y.append(tok)
        if (early_stop != -1 and len(y) - P > early_stop) or pa == V - 1 or tok == V - 1:
            break
    return np.array(y[:-1], np.int64), (0 if P == 0 else i - 1), margins, lgs
