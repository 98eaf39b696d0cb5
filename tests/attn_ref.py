"""Plain float64 restatement of one launch of the relative-position attention (attentions.py:165-196; csrc/attn_tc.cuh
attn_tc_kernel, csrc/kernels.cuh attn_kernel / attn_split_kernel) on a packed ragged batch, and the error bound a correct
kernel must meet against it.

Layout (as the engine packs utterances): utterance b occupies rows offs[b] .. offs[b] + lens[b] of qkv [rows, 3H]
(conv_ref.offsets: SEQ_GAP = 8 rows between utterances); head h reads q, k, v from channels h*dk, H + h*dk, 2H + h*dk.
For query i and key j < len of the same utterance
  s_ij = (q_i . k_j + [|j-i| <= W] q_i . Ek[j-i+W]) / sqrt(dk),   p = softmax_j(s),   o_i = sum_j p_ij (v_j + [|j-i| <= W] Ev[j-i+W]).

Operands.  The FFMA kernels pre-scale q in fp32 (q / sqrtf(dk), one rounding) and multiply fp32 q, k, v and the fp32 tables:
`reference(kind="ffma")` is the exact attention of exactly those operands.  The tensor-core kernel multiplies split-bf16
planes: q, k, v split on the device (conv_ref.split_bf16: round half away from zero), the relative tables split by the
packer (round to nearest even; taken from the blob as the engine binds them).  Its scores are the products it issues,
qh.kh + qh.kl + ql.kh (ql.kl dropped), scaled by the fp32 1/sqrtf(dk); its values are vh + vl and Evh + Evl.
`reference(kind="tc")` forms exactly these sums in float64 ("operand-exact emulation") and the exact softmax of them.

Bound.  What the emulation cannot restate exactly is bounded per output element:
  score error      |ds_ij| <= D_ij = (n_s + 4) u A_ij + 4 u (|s_ij| + M_i) + (n_t + 2) 2^-21
                   A_ij the sum of the magnitudes of the score products (band included, scaled), n_s = 3 dk (tensor cores)
                   or dk (FFMA) accumulated terms, u = 2^-23 (tensor-core accumulation may truncate: one ulp, not half;
                   Higham eq. 4.4 holds for any order of the additions, conv_ref.py); the 4 u (|s| + M) term covers the
                   roundings of the scale, of the band add and of s*log2(e) - m*log2(e) inside exp2f (M_i = max_j |s_ij|);
                   exp2f / expf are within 2 ulp (2^-22 relative on each p and on each rescale factor of the running max,
                   at most one per key tile: n_t tiles), which is a score error of 2^-22 in natural-log units.
  softmax          p~_ij = p_ij e^(ds_ij) / sum_k p_ik e^(ds_ik), so to first order dp_ij = p_ij (ds_ij - sum_k p_ik ds_ik) and
                   |do_i| <= sum_j p_ij |ds_ij - sum_k p_ik ds_ik| |v~_j| <= sum_j p_ij (D_ij + Dbar_i) |v~_j|,
                   Dbar_i = sum_k p_ik D_ik, |v~_j| = |v_j| + [band] |Ev[j-i+W]|; 5 % added for the second order (D < 0.05).
  P split          (tensor cores) P is split into bf16 hi + lo in registers (2^-16 relative) and the pl*vl product is
                   dropped (below 2^-16 |p v|): 3 * 2^-16 sum_j p_ij |v~_j|.
  P.V accumulation fp32 over n_v = 3 (n_keys rounded up to the 64-key tile + 16 band slots on each of up to 3 tiles) + n_t
                   terms (tensor cores) or n_keys + 2W + 5 + n_t (FFMA), with the running-max rescales as terms:
                   n_v u sum_j p_ij |v~_j|.
  l and 1/l        the row sum of n_keys positive terms in fp32, the reciprocal and the product: (n_keys + 8) u |o_i|.
Lazy running max.  The tensor-core kernel refreshes its running max only when a tile exceeds it by more than ATC_LAZY = 6
(p up to e^6 before the division): the products and sums scale with l, so every relative bound above holds unchanged.

Prefix mask (T given; csrc/t2s.cu t2s_prefix_attn_kernel, GPT-SoVITS's text prefill).  No band (W = 0, no tables); row i of
an utterance whose first T rows are its text sees key j iff j < T or j <= i, so each row has its own key count n_i (T for a
text row, i + 1 for a prompt row), and every term above that counts keys (n_t tiles of 32, n_v, the n_keys + 8 of l) takes
n_i.  The kernel is an FFMA kernel (fp32 fmaf dot products, n_s = dk) with an online softmax that rescales once per 32-key
tile, and it scales q by the fp32 sqrtf(1 / dk) (the reference's q * sqrt(1 / dk)) instead of dividing by sqrtf(dk): the
operands here are those.  `/` is correctly rounded (the build has no fast-math flags), covered by the l term."""
import numpy as np

from conv_ref import SEQ_GAP, U23, U24, bf16_value, offsets, split_bf16  # noqa: F401  (SEQ_GAP: the packing)

LAZY = 6.0
SPLIT_ERR = 3 * 2.0 ** -16
TC_KT, FFMA_KT = 64, 32          # key tiles of attn_tc_kernel and of the FFMA kernels
QBLK = 512                       # query rows per block of the float64 reference (memory)


def blob_tensor(blob, manifest, name):
    """A tensor of a packed blob (weights.pack) by its manifest name, as float32."""
    for line in manifest.splitlines():
        nm, off, n = line.split()
        if nm == name:
            return np.asarray(blob[int(off):int(off) + int(n)], np.float32)
    raise KeyError(name)


def layer_tables(blob, manifest, layer, dk):
    """The relative-position tables of `layer` ("enc.<i>" / "flow.<f>.tr") as the engine binds them:
    relk / relv float32 [nrel, dk] (FFMA kernels) and, when packed, rk / rv float64 [2][nrel, dk] (the packer's hi / lo bf16
    split tiles of the tensor-core kernel)."""
    relk = blob_tensor(blob, manifest, layer + ".relk").reshape(-1, dk)
    relv = blob_tensor(blob, manifest, layer + ".relv").reshape(-1, dk)
    nrel = relk.shape[0]
    t = dict(relk=relk, relv=relv)
    try:
        for nm in ("rk", "rv"):
            pl = [blob_tensor(blob, manifest, layer + "." + nm + s).view(np.uint16).reshape(16, 128) for s in "hl"]
            t[nm] = np.stack([bf16_value(p)[:nrel, :dk] for p in pl])
    except KeyError:
        pass
    return t


def _split_values(x):
    hi, lo = split_bf16(x)
    return bf16_value(hi), bf16_value(lo)


def _head(qkv, r0, n, h, dk, H, col_shift=0):
    q = qkv[r0:r0 + n, h * dk + col_shift:h * dk + col_shift + dk]
    k = qkv[r0:r0 + n, H + h * dk:H + (h + 1) * dk]
    v = qkv[r0:r0 + n, 2 * H + h * dk:2 * H + (h + 1) * dk]
    return np.asarray(q, np.float32), np.asarray(k, np.float32), np.asarray(v, np.float32)


def _prefix_keys(n, T):
    """Keys row i of a T-text-row utterance of n rows sees: T for a text row, i + 1 for a prompt row ([n, 1])."""
    i = np.arange(n)
    return np.where(i < T, T, i + 1)[:, None]


def reference(qkv, lens, heads, W, tables, kind, corrupt=None, T=None, offs=None):
    """Float64 reference of every utterance.  Returns a list of (rows [n], out [n, H], bound [n, H]): the qkv / output rows
    of the utterance and the value a correct kernel is within `bound` of.
      kind      "tc" (operand-exact emulation of attn_tc_kernel) or "ffma" (exact attention of the FFMA kernels' operands)
      corrupt   deliberate errors for the rejection studies: drop_slot (band term dropped at that relative slot), shift
                (band slots shifted by that many keys), no_ev, mask_last (last valid key masked), unmask_next (the first
                row beyond the utterance read as a key), rel_scale2 (1/sqrt(dk) twice on the relative logits), head_shift
                (head 0 reads q 32 channels further), drop_qlkh (tensor cores: no ql.kh product)
      T         the prefix mask (see above) with utterance b's first T[b] rows its text; W = 0, tables None, kind "ffma"
      offs      the utterances' first rows (default: offsets(lens))"""
    corrupt = corrupt or {}
    qkv = np.asarray(qkv, np.float32)
    H = qkv.shape[1] // 3
    dk = H // heads
    nrel = 2 * W + 1
    offs = offsets(lens) if offs is None else offs
    prefix = T is not None
    if prefix:
        assert W == 0 and tables is None and kind == "ffma"
        tables = dict(relk=np.zeros((1, dk), np.float32), relv=np.zeros((1, dk), np.float32))
    tc = kind == "tc"
    if tc:
        ekh, ekl = tables["rk"]
        evt = tables["rv"][0] + tables["rv"][1]
        scale = float(np.float32(1.0) / np.sqrt(np.float32(dk)))
        n_s = 3 * dk
    else:
        ek = tables["relk"].astype(np.float64)
        evt = tables["relv"].astype(np.float64)
        sq = np.sqrt(np.float32(dk))
        n_s = dk
    res = []
    for b, n in enumerate(lens):
        r0 = offs[b]
        nk = n + (1 if "unmask_next" in corrupt else 0) - (1 if "mask_last" in corrupt else 0)
        nq = n
        out = np.zeros((nq, H))
        bnd = np.zeros((nq, H))
        for h in range(heads):
            q, k, v = _head(qkv, r0, max(nq, nk), h, dk, H, 32 if (h == 0 and "head_shift" in corrupt) else 0)
            q, k, v = q[:nq], k[:nk], v[:nk]
            if tc:
                qh, ql = _split_values(q)
                kh, kl = _split_values(k)
                vh, vl = _split_values(v)
                S = qh @ kh.T + qh @ kl.T + (0.0 if "drop_qlkh" in corrupt else ql @ kh.T)
                Sa = np.abs(qh) @ np.abs(kh).T + np.abs(qh) @ np.abs(kl).T + np.abs(ql) @ np.abs(kh).T
                Sr = qh @ ekh.T + qh @ ekl.T + ql @ ekh.T
                Sra = np.abs(qh) @ np.abs(ekh).T + np.abs(qh) @ np.abs(ekl).T + np.abs(ql) @ np.abs(ekh).T
                S, Sa, Sr, Sra = S * scale, Sa * scale, Sr * scale, Sra * scale
                if "rel_scale2" in corrupt:
                    Sr = Sr * scale
                vt = vh + vl
                n_t = -(-nk // TC_KT)
                n_v = 3 * (n_t * TC_KT + 3 * 16) + n_t
            else:
                if prefix:                                   # t2s_prefix_attn_kernel: q * (float)sqrt(1.0 / dk)
                    qs = (q * np.float32(np.sqrt(1.0 / dk))).astype(np.float64)
                else:
                    qs = (q / sq).astype(np.float64)        # the kernels' fp32 pre-scaled q
                S, Sa = qs @ k.T.astype(np.float64), np.abs(qs) @ np.abs(k.T.astype(np.float64))
                Sr, Sra = qs @ ek.T, np.abs(qs) @ np.abs(ek.T)
                if "rel_scale2" in corrupt:
                    Sr = Sr / float(sq)
                vt = v.astype(np.float64)
                nkr = _prefix_keys(nq, T[b]) if prefix else nk
                n_t = -(-nkr // FFMA_KT)
                n_v = nkr + nrel + 4 + n_t
            for i0 in range(0, nq, QBLK):
                i1 = min(nq, i0 + QBLK)
                i = np.arange(i0, i1)[:, None]
                j = np.arange(nk)[None, :]
                d = j - i + corrupt.get("shift", 0)
                inband = np.abs(d) <= W
                slot = np.clip(d + W, 0, 2 * W)
                if "drop_slot" in corrupt:
                    inband = inband & (slot != corrupt["drop_slot"])
                s = S[i0:i1] + np.where(inband, np.take_along_axis(Sr[i0:i1], slot, 1), 0.0)
                A = Sa[i0:i1] + np.where(inband, np.take_along_axis(Sra[i0:i1], slot, 1), 0.0)
                vis = (j < T[b]) | (j <= i) if prefix else np.ones(s.shape, bool)
                s = np.where(vis, s, 0.0)
                m = np.where(vis, s, -np.inf).max(1, keepdims=True)
                p = np.where(vis, np.exp(s - m), 0.0)
                p /= p.sum(1, keepdims=True)
                M = np.abs(s).max(1, keepdims=True)
                rt = n_t[i0:i1] if prefix else n_t
                D = (n_s + 4) * U23 * A + 4 * U23 * (np.abs(s) + M) + (rt + 2) * 2.0 ** -21

                def band_scatter(w):               # [nq, nk] -> [nq, nrel]: weight of each relative slot
                    r = np.zeros((i1 - i0, nrel))
                    np.add.at(r, (np.broadcast_to(i - i0, w.shape)[inband], slot[inband]), w[inband])
                    return r

                pb = band_scatter(p)
                o = p @ vt + (0.0 if "no_ev" in corrupt else pb @ evt)
                pv_abs = p @ np.abs(vt) + pb @ np.abs(evt)
                Dbar = (p * D).sum(1, keepdims=True)
                soft = 1.05 * ((p * D) @ np.abs(vt) + band_scatter(p * D) @ np.abs(evt) + Dbar * pv_abs)
                rv, rk = (n_v[i0:i1], nkr[i0:i1]) if prefix else (n_v, nk)
                acc = rv * U23 * pv_abs * (1.0 + 2.0 ** -7 if tc else 1.0)
                e = soft + acc + (SPLIT_ERR * pv_abs if tc else 0.0) + (rk + 8) * U23 * np.abs(o)
                out[i0:i1, h * dk:(h + 1) * dk] = o
                bnd[i0:i1, h * dk:(h + 1) * dk] = e
        res.append((r0 + np.arange(nq), out, bnd))
    return res


def within(out, ref, bound):
    """True when every |out - ref| <= bound (NaN fails)."""
    return bool(np.all(np.abs(np.asarray(out, np.float64) - ref) <= bound))


def worst(out, results):
    """Largest |out - ref| / bound over all utterances of one launch (out: [rows, H]); inf when any output is not finite."""
    w = 0.0
    for rows, ref, bnd in results:
        o = np.asarray(out, np.float64)[rows]
        if not np.all(np.isfinite(o)):
            return float("inf")
        w = max(w, float(np.max(np.abs(o - ref) / bnd)))
    return w


# ------------------------------------------------------------------------------------------------ float32 restatements
def f32_attention(qkv, lens, heads, W, relk, relv, lazy=None, no_rescale=False, tile=TC_KT, T=None, offs=None, corrupt=()):
    """The attention in float32 arithmetic on the FFMA kernels' operands.  lazy=None: one softmax over all keys, products
    and sums taken in reverse key order; lazy=threshold: online softmax over key tiles with the running max refreshed only
    when a tile exceeds it by more than `threshold` (as attn_tc_kernel), no_rescale: such a refresh leaves O and l as they
    are (a corruption).  Returns (out [rows, H] float32, number of refreshes).
    T: the prefix mask as t2s_prefix_attn_kernel computes it (W = 0, relk / relv unused): key order, 32-key chunks, the
    running max raised by every chunk that exceeds it, l and the accumulators rescaled each chunk, then acc / l; rows at
    offs.  corrupt (deliberate errors): "self" (a prompt row does not see itself), "text_sees_prompt" (text rows see every
    row), "no_rescale" (acc is not rescaled; l is), "no_max" (no running max: p = expf(s), nothing rescaled)."""
    if T is not None:
        return _f32_prefix(qkv, lens, heads, T, offs, corrupt), 0
    qkv = np.asarray(qkv, np.float32)
    H = qkv.shape[1] // 3
    dk = H // heads
    offs = offsets(lens)
    out = np.zeros((qkv.shape[0], H), np.float32)
    relk, relv = np.asarray(relk, np.float32), np.asarray(relv, np.float32)
    sq = np.sqrt(np.float32(dk))
    refreshes = 0
    for b, n in enumerate(lens):
        r0 = offs[b]
        for h in range(heads):
            q, k, v = _head(qkv, r0, n, h, dk, H)
            qs = (q / sq).astype(np.float32)
            i = np.arange(n)[:, None]
            j = np.arange(n)[None, :]
            inband = np.abs(j - i) <= W
            slot = np.clip(j - i + W, 0, 2 * W)
            s = (qs @ k.T).astype(np.float32) + np.where(inband, np.take_along_axis(qs @ relk.T, slot, 1), 0).astype(np.float32)
            if lazy is None:
                p = np.exp(s - s.max(1, keepdims=True)).astype(np.float32)
                l = np.zeros((n, 1), np.float32)
                o = np.zeros((n, dk), np.float32)
                for jj in range(n - 1, -1, -1):
                    pj = p[:, jj:jj + 1]
                    l = (l + pj).astype(np.float32)
                    vj = v[jj][None, :] + np.where(inband[:, jj:jj + 1], relv[slot[:, jj]], 0).astype(np.float32)
                    o = (o + pj * vj).astype(np.float32)
            else:
                m = np.full((n, 1), -np.inf, np.float32)
                l = np.zeros((n, 1), np.float32)
                o = np.zeros((n, dk), np.float32)
                for t0 in range(0, n, tile):
                    st = s[:, t0:t0 + tile]
                    mx = st.max(1, keepdims=True)
                    if t0 == 0:
                        m = mx
                    else:
                        up = mx > m + np.float32(lazy)
                        refreshes += int(up.sum())
                        alpha = np.where(up, np.exp(m - mx), np.float32(1)).astype(np.float32)
                        m = np.where(up, mx, m)
                        if not no_rescale:
                            l = (l * alpha).astype(np.float32)
                            o = (o * alpha).astype(np.float32)
                    p = np.exp(st - m).astype(np.float32)
                    l = (l + p.sum(1, keepdims=True, dtype=np.float32)).astype(np.float32)
                    for jj in range(p.shape[1]):
                        key = t0 + jj
                        vj = v[key][None, :] + np.where(inband[:, key:key + 1], relv[slot[:, key]], 0).astype(np.float32)
                        o = (o + p[:, jj:jj + 1] * vj).astype(np.float32)
            out[r0:r0 + n, h * dk:(h + 1) * dk] = (o / l).astype(np.float32)
    return out, refreshes


def _f32_prefix(qkv, lens, heads, T, offs, corrupt):
    qkv = np.asarray(qkv, np.float32)
    H = qkv.shape[1] // 3
    dk = H // heads
    out = np.zeros((qkv.shape[0], H), np.float32)
    scale = np.float32(np.sqrt(1.0 / dk))
    f32 = np.float32
    for b, n in enumerate(lens):
        r0, Tb = offs[b], T[b]
        i = np.arange(n)
        nk = _prefix_keys(n, Tb)[:, 0]
        if "self" in corrupt:
            nk = np.where(i < Tb, Tb, i)                  # n = t < T ? T : t
        if "text_sees_prompt" in corrupt:
            nk = np.where(i < Tb, n, i + 1)
        for h in range(heads):
            q, k, v = _head(qkv, r0, n, h, dk, H)
            S = ((q * scale).astype(f32) @ k.T).astype(f32)
            m = np.full(n, -np.inf, f32)
            l = np.zeros(n, f32)
            acc = np.zeros((n, dk), f32)
            for k0 in range(0, int(nk.max()), FFMA_KT):
                cols = np.arange(k0, min(k0 + FFMA_KT, n))
                vis = cols[None, :] < nk[:, None]
                sc = np.where(vis, S[:, cols], -np.inf).astype(f32)
                mn = np.maximum(m, sc.max(1)) if "no_max" not in corrupt else np.zeros(n, f32)
                with np.errstate(invalid="ignore"):
                    corr = np.where(vis.any(1), np.exp(m - mn), f32(1)).astype(f32)
                with np.errstate(over="ignore", invalid="ignore"):
                    p = np.where(vis, np.exp(sc - mn[:, None]), 0).astype(f32)
                with np.errstate(over="ignore", invalid="ignore"):
                    l = (l * corr + p.sum(1, dtype=f32)).astype(f32)
                    if "no_rescale" not in corrupt:
                        acc = (acc * corr[:, None]).astype(f32)
                    acc = (acc + p @ v[cols]).astype(f32)
                m = mn
            with np.errstate(over="ignore", invalid="ignore"):
                out[r0:r0 + n, h * dk:(h + 1) * dk] = (acc / l[:, None]).astype(f32)
    return out
