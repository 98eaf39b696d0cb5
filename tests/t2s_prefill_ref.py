"""Restatements of the GPT-SoVITS text prefill's exact kernels (csrc/t2s.cu: t2s_prefill_embed_kernel, t2s_relu_kernel,
t2s_kv_store_kernel, t2s_init_kernel) in numpy float32, each rounded operation in the kernel's order, so that a correct
kernel matches them bit for bit.  The prefix attention's reference and bound are attn_ref.reference(..., T=...).

Layout (as vtts_t2s_decode packs a batch): utterance b's T[b] text rows, then its P[b] prompt rows, start at offsets(T, P)[b],
each utterance's T + P rows rounded up to a multiple of 8, with no gap between utterances.  init [B][4] = T, P, the first
cache row and the first token slot.  Planes are conv_ref.split_bf16 of the fp32 value written."""
import numpy as np

from conv_ref import split_bf16  # noqa: F401  (the planes)

ST_T, ST_P, ST_KV, ST_NY, ST_GEN, ST_STOP, ST_YOFF = range(7)


def offsets(T, P):
    """First row of each utterance, and the packed row total."""
    n = (np.asarray(T, np.int64) + np.asarray(P, np.int64) + 7) // 8 * 8
    off = np.concatenate([[0], np.cumsum(n)])
    return off[:-1].astype(np.int64), int(off[-1])


def embed(ids, T, P, temb, aemb, pe, alpha_t, alpha_a, x, bp=None, bp_bias=None, corrupt=()):
    """t2s_prefill_embed_kernel into a copy of x [rows, H]: text row t = (temb[id] + (bp row or bp_bias)) + alpha_t * pe[t],
    prompt row t = aemb[id] + alpha_a * pe[t - T], every op rounded to float32 on its own.  corrupt: "swap_alpha" (alpha_a
    on text rows and alpha_t on prompt rows), "prompt_pe_t" (prompt rows read pe[t])."""
    f = np.float32
    x = np.array(x, np.float32)
    at, aa = (f(alpha_a), f(alpha_t)) if "swap_alpha" in corrupt else (f(alpha_t), f(alpha_a))
    offs, _ = offsets(T, P)
    for b, (Tb, Pb) in enumerate(zip(T, P)):
        r0 = offs[b]
        rt = np.arange(r0, r0 + Tb)
        add = bp[rt] if bp is not None else np.broadcast_to(np.asarray(bp_bias, f), (Tb, x.shape[1]))
        x[rt] = (temb[ids[rt]] + add).astype(f) + (at * pe[:Tb]).astype(f)
        if Pb:
            rp = np.arange(r0 + Tb, r0 + Tb + Pb)
            pos = np.arange(Tb, Tb + Pb) if "prompt_pe_t" in corrupt else np.arange(Pb)
            x[rp] = aemb[ids[rp]] + (aa * pe[pos]).astype(f)
    return x


def rows_of(T, P):
    """Every packed row index that belongs to an utterance."""
    offs, _ = offsets(T, P)
    return np.concatenate([np.arange(o, o + t + p) for o, t, p in zip(offs, T, P)])


def relu(y, lens_rows):
    """t2s_relu_kernel's value on the rows lens_rows of y: fmaxf(y, 0) (NaN gives 0)."""
    out = np.array(y, np.float32)
    out[lens_rows] = np.fmax(out[lens_rows], np.float32(0))
    return out


def kv_store(qkv, T, P, kv_off, kc, vc):
    """t2s_kv_store_kernel into copies of the caches kc, vc [kv_rows, H]: row t of utterance b's k and v to cache row
    kv_off[b] + t."""
    H = kc.shape[1]
    kc, vc = np.array(kc, np.float32), np.array(vc, np.float32)
    offs, _ = offsets(T, P)
    for b, (Tb, Pb) in enumerate(zip(T, P)):
        src = np.arange(offs[b], offs[b] + Tb + Pb)
        dst = np.arange(kv_off[b], kv_off[b] + Tb + Pb)
        kc[dst] = qkv[src, H:2 * H]
        vc[dst] = qkv[src, 2 * H:]
    return kc, vc


def init(T, P, kv_off, y_off, prompts, pre, V, y, hx, corrupt=()):
    """t2s_init_kernel: (state [B, 8], y, seen [B, (V + 31) // 32] uint32, hx [B, H]); prompts back to back.  corrupt:
    "hx_text" (hx from row T - 1)."""
    B = len(T)
    nw = (V + 31) // 32
    st = np.zeros((B, 8), np.int32)
    y = np.array(y, np.int32)
    hx = np.array(hx, np.float32)
    seen = np.zeros((B, nw), np.uint32)
    offs, _ = offsets(T, P)
    p0 = 0
    for b in range(B):
        st[b, ST_T], st[b, ST_P], st[b, ST_KV], st[b, ST_NY], st[b, ST_YOFF] = T[b], P[b], kv_off[b], P[b], y_off[b]
        pr = np.asarray(prompts[p0:p0 + P[b]], np.int64)
        p0 += P[b]
        y[y_off[b]:y_off[b] + P[b]] = pr
        for tok in pr:
            seen[b, tok >> 5] |= np.uint32(1) << np.uint32(tok & 31)
        last = T[b] - 1 if "hx_text" in corrupt else T[b] + P[b] - 1
        hx[b] = pre[offs[b] + last]
    return st, y, seen, hx


# ------------------------------------------------------------------------------------------------ attention test inputs
EDGE_PAIRS = [(1, 0), (1, 1), (1, 31), (31, 1), (32, 0), (33, 0), (5, 27), (30, 3), (32, 32)]   # 32-key chunk edges
REAL_PAIRS = [(120, 450), (600, 40)]                                                        # prompts of 3-10 s at 50 Hz
LONG_PAIR = (200, 3700)                                                                     # near the 4000-row table


def ragged_pairs(B, seed, extra=()):
    """A ragged batch of B (T, P): the chunk-edge and real pairs, `extra`, then seeded pairs whose T + P is a multiple of 8
    (adjacent utterances touch) or not."""
    r = np.random.default_rng(seed)
    pairs = list(EDGE_PAIRS) + list(REAL_PAIRS) + list(extra)
    while len(pairs) < B:
        T, P = int(r.integers(1, 70)), int(r.integers(0, 90))
        if len(pairs) % 2:
            P += (-(T + P)) % 8
        pairs.append((T, P))
    order = r.permutation(B)
    return [pairs[i] for i in order]


def attn_qkv(pairs, heads, dk, pattern, seed, probe=None, extra_rows=16):
    """qkv float32 [rows, 3H] of the packed utterances, NaN on every other row (the rounding rows and extra_rows behind the
    last utterance).  pattern: "random" (scores ~ N(0, 1.5^2)), "rising" (each key's score above the previous one's, 30 over
    the utterance, so that every 32-key chunk raises the running max), "large" (|s| around 80: most weights underflow),
    "equal" (every score 0: the output is the mean of the visible v).  probe: a key index (or "first_prompt" / "last") of
    each utterance whose score is +30 for every query and whose v is the one-hot marker 1e4 e_0 of every head; returns
    (qkv, probe keys) then."""
    T = [p[0] for p in pairs]
    P = [p[1] for p in pairs]
    H = heads * dk
    offs, tot = offsets(T, P)
    r = np.random.default_rng(seed)
    qkv = np.full((tot + extra_rows, 3 * H), np.nan, np.float32)
    scale = np.float32(np.sqrt(1.0 / dk))
    keys = []
    for b, (Tb, Pb) in enumerate(pairs):
        n = Tb + Pb
        q = r.standard_normal((n, heads, dk))
        k = r.standard_normal((n, heads, dk))
        v = r.standard_normal((n, heads, dk))
        if pattern == "random":
            k *= 1.5
        elif pattern == "rising":
            u = np.abs(r.standard_normal((heads, dk))) + 0.5
            q = np.broadcast_to(u, (n, heads, dk)).copy()
            uu = (u * u).sum(1) * float(scale)
            k = (30.0 * np.arange(n) / max(n - 1, 1))[:, None, None] * u[None] / uu[None, :, None]
        elif pattern == "large":
            q *= 80 ** 0.5
            k *= 80 ** 0.5
        elif pattern == "equal":
            k[:] = 0
        if probe is not None:
            kp = {"first_prompt": Tb, "last": n - 1}.get(probe, probe) if not isinstance(probe, int) else min(probe, n - 1)
            kp = min(kp, n - 1)
            keys.append(kp)
            q[:, :, 0] = 1.0
            k[:, :, 0] = 0.0
            k[kp] = 0.0
            k[kp, :, 0] = 30.0 / float(scale)
            v[kp] = 0.0
            v[kp, :, 0] = 1e4
        rows = slice(offs[b], offs[b] + n)
        qkv[rows, :H] = q.reshape(n, H)
        qkv[rows, H:2 * H] = k.reshape(n, H)
        qkv[rows, 2 * H:] = v.reshape(n, H)
    return (qkv, keys) if probe is not None else qkv
