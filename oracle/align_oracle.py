"""CPU restatement of the text-to-frame alignment at the head of SynthesizerTrn.forward (training/vits2/models.py:1632-1660):
enc_p on the ids, enc_q + forward flow on the recording's features, the Gaussian log-likelihood ``neg_cent`` of every frame
under every token's prior, and Monotonic Alignment Search.  Built from the restatements of ``vits_oracle`` / ``vc_oracle`` /
``mas_oracle``; pinned to the unmodified reference by tests/test_align_host.py through tests/golden/ref_alignment.npz
(oracle/make_golden_align.py).  TEST INFRASTRUCTURE: the product path is vosk_tts_b200/csrc (neg_cent_kernel, mas_kernel).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import mas_oracle
from oracle.vc_oracle import flow_forward, posterior_encoder
from oracle.vits_oracle import text_encoder


def neg_cent(z_p, m_p, logs_p):
    """float64 direct form of models.py:1645-1651 for one utterance: z_p [I, t_y], m_p / logs_p [I, t_x] -> [t_y, t_x],
    sum_d (-0.5 log 2pi - logs_p[d, i] - 0.5 (z_p[d, j] - m_p[d, i])^2 exp(-2 logs_p[d, i]))."""
    z, m, lg = (np.asarray(a, np.float64) for a in (z_p, m_p, logs_p))
    out = np.sum(-0.5 * math.log(2 * math.pi) - lg, axis=0)[None, :].repeat(z.shape[1], 0)
    s = np.exp(-2.0 * lg)
    for d in range(z.shape[0]):
        q = z[d][:, None] - m[d][None, :]
        out -= 0.5 * q * q * s[d][None, :]
    return out


def path_of(value_path):
    """int path [t_y, t_x] (one 1 per frame) -> token of every frame int32 [t_y] and frames per token int32 [t_x]."""
    tof = np.argmax(value_path, axis=1).astype(np.int32)
    return tof, value_path.sum(0).astype(np.int32)


def path_score(nc, tof):
    """float64 sum of nc [t_y, t_x] along the path given as the token of every frame (summed in frame order)."""
    s = 0.0
    for y, x in enumerate(tof):
        s += float(nc[y, x])
    return s


def two_best(nc, t_y, t_x):
    """The best two path scores over all monotonic paths (every frame on one token, tokens in order, each token at least
    one frame, from (0, 0) to (t_y - 1, t_x - 1)) by the MAS recurrence in float64, keeping the two best DISTINCT paths'
    scores per cell (equal scores of two different paths both count).  Returns (best, second); second = -inf when only one
    path exists.  The margin best - second bounds how much score error the MAS argmax tolerates."""
    nc = np.asarray(nc, np.float64)
    NEG = -np.inf
    prev = None
    for y in range(t_y):
        cur = np.full((t_x, 2), NEG)
        for x in range(max(0, t_x + y - t_y), min(t_x, y + 1)):
            if y == 0:
                cand = [0.0]
            else:
                cand = list(prev[x]) + (list(prev[x - 1]) if x > 0 else [])
            cand = sorted((c for c in cand if c != NEG), reverse=True)[:2]
            for k, c in enumerate(cand):
                cur[x, k] = c + nc[y, x]
        prev = cur
    return float(prev[t_x - 1, 0]), float(prev[t_x - 1, 1])


def align(w, cfg, ids, spec, sid, eps):
    """One utterance: ids int64 [t_x], spec float32 [spec_channels, t_y] (the reference's `y`), sid (ignored without
    speakers), eps [1, inter, >= t_y] for enc_q's randn_like (models.py:841).  Returns z_p, m_p, logs_p (float32 [I, t]),
    neg_cent (float64 [t_y, t_x]), the MAS path on its float32 rounding (token_of_frame, durations), its score and the
    2-best margin."""
    tok = torch.as_tensor(np.asarray(ids, np.int64))[None]
    y = torch.as_tensor(np.asarray(spec, np.float32))[None]
    t_x, t_y = tok.shape[1], y.shape[2]
    g = None
    if cfg["n_speakers"] > 0 and cfg["gin_channels"] > 0:          # models.py:1633-1637
        g = F.embedding(torch.tensor([int(sid)]), w["emb_g.weight"]).unsqueeze(-1)
    with torch.no_grad():
        _, m_p, logs_p, _ = text_encoder(tok, torch.tensor([t_x]), g, w, cfg)
        z, _, _, y_mask = posterior_encoder(y, torch.tensor([t_y]), g, w, torch.as_tensor(eps))
        z_p = flow_forward(z, y_mask, g, w, cfg)
    z_p, m_p, logs_p = (a[0].numpy().astype(np.float32) for a in (z_p, m_p, logs_p))
    nc = neg_cent(z_p, m_p, logs_p)
    path = mas_oracle.maximum_path_vectorised(nc.astype(np.float32)[None], [t_y], [t_x])[0]
    tof, dur = path_of(path)
    best, second = two_best(nc, t_y, t_x)
    return dict(z_p=z_p, m_p=m_p, logs_p=logs_p, neg_cent=nc, token_of_frame=tof, durations=dur, score=path_score(nc, tof),
                margin=best - second)
