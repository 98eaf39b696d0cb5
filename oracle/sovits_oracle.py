"""Float64 restatement of GPT-SoVITS's SynthesizerTrn.extract_latent (training/gpt-sovits/module/models.py:990-993) at the
25 Hz frame rate: ssl_proj = Conv1d(768, 768, 2, stride=2) over the HuBERT rows (an odd last row is dropped), then one
EuclideanCodebook.quantize (module/core_vq.py:175-183), the argmax over the codebook of -|x - E_k|^2.  Also the margin of every
row, best minus second-best score, which says how large an error in the scores may become before it changes the code."""
import numpy as np


def project(feats, w, b):
    """feats [T, H] (frame-major HuBERT rows) -> ssl_proj's rows [T // 2, H] in float64."""
    x = np.asarray(feats, np.float64)
    w = np.asarray(w, np.float64)
    T2 = x.shape[0] // 2
    pairs = x[:2 * T2].reshape(T2, 2, -1)
    return pairs[:, 0] @ w[:, :, 0].T + pairs[:, 1] @ w[:, :, 1].T + np.asarray(b, np.float64)


def scores(proj, E):
    """-|x - E_k|^2 of every projected row x and codeword E_k, [T', K], in float64 (core_vq's dist)."""
    p = np.asarray(proj, np.float64)
    E = np.asarray(E, np.float64)
    return -((p * p).sum(1, keepdims=True) - 2 * p @ E.T + (E * E).sum(1)[None, :])


def extract_latent(feats, sd):
    """feats [T, H] and the s2 tensors (weights.load_sovits's state dict) -> (codes int64 [T // 2], lowest index on ties;
    margin float64 [T // 2], best minus second-best score; best float64 [T // 2], the best score)."""
    g = lambda k: sd[k].detach().cpu().double().numpy() if hasattr(sd[k], "detach") else np.asarray(sd[k], np.float64)
    s = scores(project(feats, g("ssl_proj.weight"), g("ssl_proj.bias")), g("quantizer.vq.layers.0._codebook.embed"))
    codes = s.argmax(1)
    top2 = -np.sort(-s, axis=1)[:, :2] if s.shape[1] > 1 else np.concatenate([s, s - np.inf], 1)
    return codes.astype(np.int64), top2[:, 0] - top2[:, 1], top2[:, 0]
