"""Checkpoint -> engine weights: weight-norm folding and the packed device blob.

Contract (SURVEY.md section 5 "Checkpoint / resume"; /root/reference/training/vits2/utils.py:18-50,
onnx_export.py:55,78-79): a ``G_*.pth`` holds ``{'model': state_dict, ...}`` with weight-normed convs
stored as ``weight_g`` / ``weight_v``; the exporter loads it and removes weight norm on ``dec`` and
``flow`` before tracing.  ``fold_weight_norm`` performs the same fold; ``pack`` (below) lays every
tensor out the way the CUDA kernels consume it.
"""
import json
import math

import numpy as np
import torch

from . import config as _config


def fold_weight_norm(sd):
    """w = g * v / ||v||, the norm taken over all dims but 0 (torch.nn.utils.weight_norm dim=0;
    for ConvTranspose1d dim 0 is the *input* channel, e.g. dec.ups.0.weight_g is [512,1,1])."""
    out = {}
    sd = {k: (torch.from_numpy(np.array(v)) if isinstance(v, np.ndarray) else v) for k, v in sd.items()}   # numpy (model.onnx) or torch
    for k, v in sd.items():
        if k.endswith(".weight_v"):
            base = k[: -len("_v")]
            g = sd[base + "_g"]
            t = v.float()
            nrm = t.reshape(t.shape[0], -1).norm(dim=1).reshape([-1] + [1] * (t.dim() - 1))
            out[base] = (t * (g.float() / nrm)).contiguous()
        elif k.endswith(".weight_g"):
            continue
        else:
            out[k] = v.float().contiguous() if torch.is_floating_point(v) else v
    return out


def load_checkpoint(path, allow_pickle=False):
    """Reads a reference ``G_*.pth`` (utils.py:18-21) and returns the folded state dict.

    The ``{'model': state_dict, 'iteration': int, 'optimizer': ..., 'learning_rate': float}`` layout is plain tensors
    and numbers, so the file is read with ``weights_only=True``: a crafted checkpoint in a model directory cannot run
    code at load time (the reference's inference package only ever opens ``model.onnx``).  ``allow_pickle=True`` is an
    explicit opt-in for legacy files that need full unpickling."""
    ck = torch.load(path, map_location="cpu", weights_only=not allow_pickle)
    sd = ck["model"] if isinstance(ck, dict) and "model" in ck else ck
    sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
    return fold_weight_norm(sd)


# ----------------------------------------------------------------------------------------------
# Packing: folded state dict -> one fp32 blob + manifest, laid out the way csrc/ consumes it.
#   generic conv  <name>.w : [k][Cin][ldw]  (ldw = Cout rounded up to 4, zero padded), <name>.b : [ldw]
#   every tensor starts on a 256-byte boundary.
# ----------------------------------------------------------------------------------------------
def _kaiser(M, beta):
    n = np.arange(M)
    alpha = (M - 1) / 2.0
    return np.i0(beta * np.sqrt(np.clip(1 - ((n - alpha) / alpha) ** 2, 0, 1))) / np.i0(beta)


def istft_inverse_basis(n_fft, hop):
    """OnnxSTFT.__init__ (training/vits2/stft.py:191-214): pinv(scale*[Re;Im]FFT(I)[:n/2+1]).T * hann."""
    scale = n_fft / hop
    fb = np.fft.fft(np.eye(n_fft))
    cutoff = n_fft // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff]), np.imag(fb[:cutoff])])
    inv = np.linalg.pinv(scale * fb).T.astype(np.float32)          # FloatTensor(...) cast (:199-200)
    n = np.arange(n_fft)
    hann = (0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)).astype(np.float32)   # get_window('hann', fftbins=True).float()
    return (inv * hann[None, :]).astype(np.float32)                # [2*cutoff, n_fft]


def _hz_to_mel_slaney(f):
    f = np.asarray(f, np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz_slaney(m):
    m = np.asarray(m, np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr, n_fft, n_mels, fmin=0.0, fmax=None):
    """librosa.filters.mel(sr=, n_fft=, n_mels=, fmin=, fmax=) with its defaults (Slaney mel scale, Slaney area
    normalisation), as mel_processing.py:85-86 calls it: float32 [n_mels, n_fft // 2 + 1], computed in float64."""
    fmax = sr / 2.0 if fmax is None else float(fmax)
    fftfreqs = np.fft.rfftfreq(n_fft, 1.0 / sr)
    mel_f = _mel_to_hz_slaney(np.linspace(_hz_to_mel_slaney(fmin), _hz_to_mel_slaney(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    lower = -ramps[:n_mels] / fdiff[:n_mels, None]
    upper = ramps[2:] / fdiff[1:, None]
    weights = np.maximum(0.0, np.minimum(lower, upper))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


def stft_basis(n_fft):
    """Windowed DFT basis of the spectrogram front end (csrc/vc.cuh stft_mag_kernel): float32 [n_fft samples][n_fft columns],
    columns (2k, 2k+1) = hann[n] * (cos, -sin)(2 pi k n / n_fft) of bin k < n_fft/2, except that column 1 (the sine of bin 0,
    identically zero) holds the cosine of the Nyquist bin.  Periodic Hann window of n_fft (torch.hann_window)."""
    n = np.arange(n_fft)
    hann = 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)
    k = np.arange(n_fft // 2)
    ang = 2.0 * np.pi * ((np.outer(n, k) % n_fft) / n_fft)
    basis = np.zeros((n_fft, n_fft), np.float64)
    basis[:, 0::2] = np.cos(ang)
    basis[:, 1::2] = -np.sin(ang)
    basis[:, 1] = np.where(n % 2 == 0, 1.0, -1.0)
    return (basis * hann[:, None]).astype(np.float32)


def pqmf_synthesis_filter(subbands=4, taps=62, cutoff_ratio=0.15, beta=9.0):
    """PQMF.__init__ (training/vits2/pqmf.py:15-43,63-89): fp32 [subbands, taps+1]."""
    n = np.arange(taps + 1)
    omega_c = np.pi * cutoff_ratio
    with np.errstate(invalid="ignore", divide="ignore"):
        h_i = np.sin(omega_c * (n - 0.5 * taps)) / (np.pi * (n - 0.5 * taps))
    h_i[taps // 2] = np.cos(0) * cutoff_ratio
    h = h_i * _kaiser(taps + 1, beta)
    hs = np.zeros((subbands, taps + 1))
    for k in range(subbands):
        hs[k] = 2 * h * np.cos((2 * k + 1) * (np.pi / (2 * subbands)) * (n - ((taps - 1) / 2))
                               - (-1) ** k * np.pi / 4)
    return hs.astype(np.float32)


def to_bf16_bits(a):
    """float32 -> bf16 bit patterns (uint16), round-to-nearest-even like __float2bfloat16_rn."""
    x = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = (x + 0x7FFF + ((x >> 16) & 1)) >> 16
    return r.astype(np.uint16)


def from_bf16_bits(b):
    return (b.astype(np.uint32) << 16).view(np.float32)


def conv_ffma_layout(w, b=None):
    """Conv1d weight [Co, Ci, k] (+ bias [Co]) in the FFMA conv's layout: w [k][Ci][ldw], bias [ldw], ldw = Co rounded up to 4."""
    w = np.asarray(w, np.float32)
    co, ci, k = w.shape
    ldw = (co + 3) // 4 * 4
    wp = np.zeros((k, ci, ldw), np.float32)
    wp[:, :, :co] = np.transpose(w, (2, 1, 0))
    bp = np.zeros(ldw, np.float32)
    if b is not None:
        bp[:co] = np.asarray(b, np.float32)
    return wp, bp


def conv_tc_planes(w):
    """Conv1d weight [Co, Ci, k] -> split-bf16 bit planes (hi, lo), each uint16 [k][Co][Ci] (K-major rows for TMA):
    hi = rne_bf16(w), lo = rne_bf16(w - hi)."""
    wt = np.ascontiguousarray(np.transpose(np.asarray(w, np.float32), (2, 0, 1)))
    hi = to_bf16_bits(wt)
    return hi, to_bf16_bits(wt - from_bf16_bits(hi))


def conv_tc3_planes(w):
    """Exact 3-way split (hi, mid, lo) of a conv weight [Co, Ci, k], each uint16 [k][Co][Ci]: hi + mid + lo == w to the last
    fp32 bit."""
    wt = np.ascontiguousarray(np.transpose(np.asarray(w, np.float32), (2, 0, 1)))
    hi = to_bf16_bits(wt)
    r1 = wt - from_bf16_bits(hi)
    mid = to_bf16_bits(r1)
    return hi, mid, to_bf16_bits(r1 - from_bf16_bits(mid))


class _Packer:
    ALIGN = 64  # floats

    def __init__(self):
        self.chunks = []
        self.entries = []
        self.pos = 0

    def add(self, name, arr):
        a = np.ascontiguousarray(np.asarray(arr, dtype=np.float32)).reshape(-1)
        pad = (-self.pos) % self.ALIGN
        if pad:
            self.chunks.append(np.zeros(pad, np.float32))
            self.pos += pad
        self.entries.append((name, self.pos, a.size))
        self.chunks.append(a)
        self.pos += a.size

    def conv(self, name, w, b=None, co_perm=None, ci_perm=None, need_w=True):
        """w: [Co, Ci, k] (Conv1d layout).  need_w=False: only the bias is packed (the conv runs on tensor-core from its .th/.tl copy)."""
        w = np.asarray(w, np.float32)
        if co_perm is not None:
            w = w[co_perm]
            b = None if b is None else np.asarray(b, np.float32)[co_perm]
        if ci_perm is not None:
            w = w[:, ci_perm]
        wp, bp = conv_ffma_layout(w, b)
        if need_w:
            self.add(name + ".w", wp)
        self.add(name + ".b", bp)

    def conv_tc(self, name, w, co_perm=None, ci_perm=None):
        """Split-bf16 copy of a conv weight for the tensor-core path: <name>.th / <name>.tl = [k][Cout][Cin] bf16
        (K-major rows for TMA), hi = rne_bf16(w), lo = rne_bf16(w - hi); two bf16 per fp32 blob slot."""
        w = np.asarray(w, np.float32)
        if co_perm is not None:
            w = w[co_perm]
        if ci_perm is not None:
            w = w[:, ci_perm]
        hi, lo = conv_tc_planes(w)
        assert hi.size % 2 == 0
        self.add(name + ".th", hi.reshape(-1).view(np.float32))
        self.add(name + ".tl", lo.reshape(-1).view(np.float32))

    def conv_tc3(self, name, w, co_perm=None, ci_perm=None):
        """Exact 3-way split copy (precision mode 3): <name>.t3h / .t3m / .t3l with hi + mid + lo == w to the last fp32 bit."""
        w = np.asarray(w, np.float32)
        if co_perm is not None:
            w = w[co_perm]
        if ci_perm is not None:
            w = w[:, ci_perm]
        hi, mid, lo = conv_tc3_planes(w)
        self.add(name + ".t3h", hi.reshape(-1).view(np.float32))
        self.add(name + ".t3m", mid.reshape(-1).view(np.float32))
        self.add(name + ".t3l", lo.reshape(-1).view(np.float32))

    def finish(self):
        blob = np.concatenate(self.chunks) if self.chunks else np.zeros(0, np.float32)
        manifest = "".join("%s %d %d\n" % e for e in self.entries)
        return blob, manifest


def convt_phases(u, K, p=None):
    """Polyphase split of ConvTranspose1d(k=K, stride=u, padding=p) (default p = (K-u)//2; config.convt_pad gives each
    stage's): for phase r the taps (in increasing input position) are kernel columns j_m, and `pad` inputs lie left of t.
    out[u*t + r] = sum_m x[t - pad + m] * W[:, :, j_m]."""
    if p is None:
        p = (K - u) // 2
    phases = []
    for r in range(u):
        d_min = -((r + p) // u)            # ceil(-(r+p)/u)
        d_max = (K - 1 - r - p) // u
        js = [r + p + u * (d_max - m) for m in range(d_max - d_min + 1)]
        assert all(0 <= j < K for j in js)
        phases.append((d_max, js))
    return phases


def tc_supported(cfg):
    """The tensor-core conv path packs 64-channel K chunks: every conv it takes over must have Cin % 64 == 0."""
    n_ups = len(cfg["upsample_rates"])
    return (cfg["decoder"] in ("mb_istft", "ms_istft", "istft") and str(cfg["resblock"]) == "1" and cfg["hidden_channels"] % 64 == 0 and
            cfg["filter_channels"] % 64 == 0 and cfg["inter_channels"] % 64 == 0 and
            (cfg["upsample_initial_channel"] >> n_ups) % 64 == 0)


def _pack_wn_encoder(P, g, dst, src, H, tc, fw):
    """The 16-layer WN stack (kernel 5, no cond here) and proj of a PosteriorEncoder (models.py:813-842; QuickVC's enc_p and
    enc_q, vc/models.py:242-271) under <dst>.in<i> / .rsx<i> / .rss<i> / .proj, gate channels interleaved; <dst>.pre and the
    cond rows are packed by the caller."""
    il = np.arange(2 * H).reshape(2, H).T.reshape(-1)
    nq = 16
    for i in range(nq):
        lay = "%s.enc.in_layers.%d" % (src, i)
        P.conv("%s.in%d" % (dst, i), g(lay + ".weight"), g(lay + ".bias"), co_perm=il, need_w=fw)
        if tc:
            P.conv_tc("%s.in%d" % (dst, i), g(lay + ".weight"), co_perm=il)
        rw, rb = g("%s.enc.res_skip_layers.%d.weight" % (src, i)), g("%s.enc.res_skip_layers.%d.bias" % (src, i))
        if i < nq - 1:
            P.conv("%s.rsx%d" % (dst, i), rw[:H], rb[:H], need_w=fw)
            P.conv("%s.rss%d" % (dst, i), rw[H:], rb[H:], need_w=fw)
            if tc:
                P.conv_tc("%s.rsx%d" % (dst, i), rw[:H])
                P.conv_tc("%s.rss%d" % (dst, i), rw[H:])
        else:
            P.conv("%s.rss%d" % (dst, i), rw, rb, need_w=fw)
            if tc:
                P.conv_tc("%s.rss%d" % (dst, i), rw)
    P.conv(dst + ".proj", g(src + ".proj.weight"), g(src + ".proj.bias"), need_w=fw)
    if tc:
        P.conv_tc(dst + ".proj", g(src + ".proj.weight"))


def _flow_cond_rows(g, cfg, rows_w, rows_b):
    """Appends the WN cond_layer rows of every coupling layer (flow.flows.<2f>.enc.cond_layer), layer by layer, with the
    gate channels interleaved as the packed in_layers are: one block of the stacked conditioning matrix cond.w / cond.b."""
    H, nl = cfg["hidden_channels"], cfg["flow_wn_layers"]
    il = np.arange(2 * H).reshape(2, H).T.reshape(-1)     # gate interleave: [t0,s0,t1,s1,...]
    for f in range(cfg["flow_n_flows"]):
        cw = g("flow.flows.%d.enc.cond_layer.weight" % (2 * f))[:, :, 0]
        cb = g("flow.flows.%d.enc.cond_layer.bias" % (2 * f))
        for i in range(nl):
            rows_w.append(cw[i * 2 * H:(i + 1) * 2 * H][il])
            rows_b.append(cb[i * 2 * H:(i + 1) * 2 * H][il])


def _pack_flow_decoder(P, g, w, cfg, tc, fw, enc_layer=None):
    """The reverse flow (flow.*) and the decoder (dec.*) of a VITS2 or QuickVC state dict; enc_layer packs the flow's
    pre_transformer (use_transformer_flows only)."""
    H, I = cfg["hidden_channels"], cfg["inter_channels"]
    # ---- flow (reverse); channel flips are folded into the pre/post weights (see csrc/engine.cu)
    nf = cfg["flow_n_flows"]
    half = I // 2
    rev = np.arange(half)[::-1].copy()
    for f in range(nf):
        src = "flow.flows.%d" % (2 * f)
        dst = "flow.%d" % f
        flipped = ((nf - f) % 2) == 1
        P.conv(dst + ".pre", g(src + ".pre.weight"), g(src + ".pre.bias"), ci_perm=rev if flipped else None)
        if cfg["use_transformer_flows"]:
            enc_layer(dst + ".tr", src + ".pre_transformer", 0, with_tc=tc, need_w=fw)
        nl = cfg["flow_wn_layers"]
        il = np.arange(2 * H).reshape(2, H).T.reshape(-1)
        for i in range(nl):
            P.conv("%s.in%d" % (dst, i), g("%s.enc.in_layers.%d.weight" % (src, i)),
                   g("%s.enc.in_layers.%d.bias" % (src, i)), co_perm=il, need_w=fw)
            rw, rb = g("%s.enc.res_skip_layers.%d.weight" % (src, i)), g("%s.enc.res_skip_layers.%d.bias" % (src, i))
            if tc:
                P.conv_tc("%s.in%d" % (dst, i), g("%s.enc.in_layers.%d.weight" % (src, i)), co_perm=il)
            if i < nl - 1:
                P.conv("%s.rsx%d" % (dst, i), rw[:H], rb[:H], need_w=fw)
                P.conv("%s.rss%d" % (dst, i), rw[H:], rb[H:], need_w=fw)
                if tc:
                    P.conv_tc("%s.rsx%d" % (dst, i), rw[:H])
                    P.conv_tc("%s.rss%d" % (dst, i), rw[H:])
            else:
                P.conv("%s.rss%d" % (dst, i), rw, rb, need_w=fw)
                if tc:
                    P.conv_tc("%s.rss%d" % (dst, i), rw)
        P.conv(dst + ".post", g(src + ".post.weight"), g(src + ".post.bias"), co_perm=rev if flipped else None, need_w=fw)
        if tc:
            P.conv_tc(dst + ".post", g(src + ".post.weight"), co_perm=rev if flipped else None)

    # ---- decoder
    pre_w = g("dec.conv_pre.weight")
    if nf % 2 == 1:   # odd number of flips leaves the latent channel-reversed: fold into conv_pre
        pre_w = pre_w[:, ::-1].copy()
    P.conv("dec.pre", pre_w, g("dec.conv_pre.bias"), need_w=fw)
    if tc:
        P.conv_tc("dec.pre", pre_w)
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, ku) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        wt = g("dec.ups.%d.weight" % i)                      # [Cin, Cout, K]
        bt = g("dec.ups.%d.bias" % i)
        for r, (pad, js) in enumerate(convt_phases(u, ku, _config.convt_pad(cfg, i)[0])):
            wr = np.stack([wt[:, :, j] for j in js], axis=-1)   # [Cin, Cout, ntaps]
            P.conv("dec.up%d.p%d" % (i, r), np.transpose(wr, (1, 0, 2)), bt, need_w=fw)
            if tc:
                P.conv_tc("dec.up%d.p%d" % (i, r), np.transpose(wr, (1, 0, 2)))
        for j in range(nk):
            n = i * nk + j
            nd = len(cfg["resblock_dilation_sizes"][j])
            for d in range(nd):
                if cfg["resblock"] == "1":
                    P.conv("dec.rb%d.c1.%d" % (n, d), g("dec.resblocks.%d.convs1.%d.weight" % (n, d)), g("dec.resblocks.%d.convs1.%d.bias" % (n, d)), need_w=fw)
                    P.conv("dec.rb%d.c2.%d" % (n, d), g("dec.resblocks.%d.convs2.%d.weight" % (n, d)), g("dec.resblocks.%d.convs2.%d.bias" % (n, d)), need_w=fw)
                    if tc:
                        P.conv_tc("dec.rb%d.c1.%d" % (n, d), g("dec.resblocks.%d.convs1.%d.weight" % (n, d)))
                        P.conv_tc("dec.rb%d.c2.%d" % (n, d), g("dec.resblocks.%d.convs2.%d.weight" % (n, d)))
                else:
                    P.conv("dec.rb%d.c.%d" % (n, d), g("dec.resblocks.%d.convs.%d.weight" % (n, d)), g("dec.resblocks.%d.convs.%d.bias" % (n, d)))
    if cfg["decoder"] in ("mb_istft", "ms_istft", "istft"):
        # All three end in conv_post -> exp / pi*sin -> inverse STFT -> zero-stuffing by `subbands` -> a 63-tap filter per band
        # (zero padding 31).  Only the filter differs: the fixed PQMF synthesis bank (pqmf.py:63-89), the learned
        # multistream_conv_post (models.py:1107), or -- one band, nothing after the iSTFT (models.py:962-965) -- a unit impulse.
        post = "dec.conv_post" if cfg["decoder"] == "istft" else "dec.subband_conv_post"
        post_b = g(post + ".bias") if (post + ".bias") in w else None          # only the multistream decoder has one (:1095)
        P.conv("dec.post", g(post + ".weight"), post_b, need_w=fw)
        if tc:
            P.conv_tc("dec.post", g(post + ".weight"))
        P.add("dec.istft", istft_inverse_basis(cfg["gen_istft_n_fft"], cfg["gen_istft_hop_size"]))
        if cfg["decoder"] == "mb_istft":
            bank = pqmf_synthesis_filter(cfg["subbands"])
        elif cfg["decoder"] == "ms_istft":
            bank = g("dec.multistream_conv_post.weight")[0]
            assert bank.shape == (cfg["subbands"], 63), bank.shape
        else:
            bank = np.zeros((1, 63), np.float32)
            bank[0, 31] = 1.0
        P.add("dec.pqmf", bank)
    else:
        P.conv("dec.post", g("dec.conv_post.weight"), None)



def pack(w, cfg, tc=True, precision=None, posterior=False):
    """w: folded state dict (reference names); returns (blob float32[n], manifest str).
    posterior=True also packs the posterior encoder enc_q and the spectrogram front end (voice conversion, vtts_convert),
    after every other tensor: the rest of the blob and its manifest stay what they are without it.
    tc=True also packs split-bf16 copies of the convs for the tensor-core path (precision modes 1 / 2).
    precision: None packs everything (a blob any engine mode can be created from); 0 / 1 / 2 leave out the tensors that
    mode never reads (mode 0: no split-bf16 copies at all; mode 1: none for the text encoder) -- what travels in the
    one-time NCCL weight broadcast of a multi-GPU job."""
    tc = tc and tc_supported(cfg) and precision != 0
    enc_tc = tc and precision in (None, 2)
    enc_tc3 = tc and precision in (None, 3)    # exact 3-way split copies of the text encoder's convs (mode 3)
    fw = not (tc and precision in (1, 2, 3))   # fp32 copies of the flow / decoder convs (the tensor-core modes read only .th/.tl + bias)
    ew = not (tc and precision in (2, 3))      # ... of the text encoder's convs
    g = lambda k: w[k].detach().cpu().numpy() if hasattr(w[k], "detach") else np.asarray(w[k])
    H, I, G = cfg["hidden_channels"], cfg["inter_channels"], cfg["gin_channels"]
    D = cfg["dp_filter_channels"]
    P = _Packer()

    def ln(dst, src):
        P.add(dst + ".g", g(src + ".gamma"))
        P.add(dst + ".b", g(src + ".beta"))

    def enc_layer(dst, src, i, with_tc=False, need_w=True, with_tc3=False):
        a = "%s.attn_layers.%d" % (src, i)
        wq = np.concatenate([g(a + ".conv_q.weight"), g(a + ".conv_k.weight"), g(a + ".conv_v.weight")], 0)
        bq = np.concatenate([g(a + ".conv_q.bias"), g(a + ".conv_k.bias"), g(a + ".conv_v.bias")], 0)
        P.conv(dst + ".qkv", wq, bq, need_w=need_w)
        P.conv(dst + ".o", g(a + ".conv_o.weight"), g(a + ".conv_o.bias"), need_w=need_w)
        if with_tc:
            f_ = "%s.ffn_layers.%d" % (src, i)
            P.conv_tc(dst + ".qkv", wq)
            P.conv_tc(dst + ".o", g(a + ".conv_o.weight"))
            P.conv_tc(dst + ".ffn1", g(f_ + ".conv_1.weight"))
            P.conv_tc(dst + ".ffn2", g(f_ + ".conv_2.weight"))
        if with_tc3:
            f_ = "%s.ffn_layers.%d" % (src, i)
            P.conv_tc3(dst + ".qkv", wq)
            P.conv_tc3(dst + ".o", g(a + ".conv_o.weight"))
            P.conv_tc3(dst + ".ffn1", g(f_ + ".conv_1.weight"))
            P.conv_tc3(dst + ".ffn2", g(f_ + ".conv_2.weight"))
        P.add(dst + ".relk", g(a + ".emb_rel_k")[0])
        P.add(dst + ".relv", g(a + ".emb_rel_v")[0])
        if with_tc:
            # the same tables as split-bf16 [16 offsets][128 channels] tiles (zero padded) for the tensor-core attention:
            # Ek is a K-major B operand of Q Ek^T, Ev an MN-major B operand of P_band Ev (csrc/attn_tc.cuh)
            for nm, src_t in ((".rk", g(a + ".emb_rel_k")[0]), (".rv", g(a + ".emb_rel_v")[0])):
                nrel, dk = src_t.shape
                if nrel <= 16 and dk <= 128:
                    t = np.zeros((16, 128), np.float32)
                    t[:nrel, :dk] = src_t
                    hi = to_bf16_bits(t)
                    lo = to_bf16_bits(t - from_bf16_bits(hi))
                    P.add(dst + nm + "h", hi.reshape(-1).view(np.float32))
                    P.add(dst + nm + "l", lo.reshape(-1).view(np.float32))
        ln(dst + ".ln1", "%s.norm_layers_1.%d" % (src, i))
        f = "%s.ffn_layers.%d" % (src, i)
        P.conv(dst + ".ffn1", g(f + ".conv_1.weight"), g(f + ".conv_1.bias"), need_w=need_w)
        P.conv(dst + ".ffn2", g(f + ".conv_2.weight"), g(f + ".conv_2.bias"), need_w=need_w)
        ln(dst + ".ln2", "%s.norm_layers_2.%d" % (src, i))

    def dds(dst, src, n_layers=3):
        for i in range(n_layers):
            P.add("%s.%d.sep_w" % (dst, i), np.transpose(g("%s.convs_sep.%d.weight" % (src, i))[:, 0, :], (1, 0)))
            P.add("%s.%d.sep_b" % (dst, i), g("%s.convs_sep.%d.bias" % (src, i)))
            ln("%s.%d.ln1" % (dst, i), "%s.norms_1.%d" % (src, i))
            P.conv("%s.%d.pw" % (dst, i), g("%s.convs_1x1.%d.weight" % (src, i)), g("%s.convs_1x1.%d.bias" % (src, i)))
            ln("%s.%d.ln2" % (dst, i), "%s.norms_2.%d" % (src, i))

    # ---- speaker table + all per-utterance conditioning projections as one matrix
    has_g = cfg["n_speakers"] > 0 and G > 0
    if has_g:
        P.add("emb_g", g("emb_g.weight"))
        rows_w, rows_b = [], []
        if cfg["use_spk_conditioned_encoder"]:
            rows_w.append(g("enc_p.encoder.spk_emb_linear.weight"))
            rows_b.append(g("enc_p.encoder.spk_emb_linear.bias"))
        rows_w.append(g("dp.cond.weight")[:, :, 0])
        rows_b.append(g("dp.cond.bias"))
        _flow_cond_rows(g, cfg, rows_w, rows_b)
        if cfg["decoder"] == "hifigan" and "dec.cond.weight" in w:
            rows_w.append(g("dec.cond.weight")[:, :, 0])       # Generator's speaker projection (models.py:869-875)
            rows_b.append(g("dec.cond.bias"))
        P.add("cond.w", np.concatenate(rows_w, 0))
        P.add("cond.b", np.concatenate(rows_b, 0))

    # ---- text encoder
    P.add("enc.emb", g("enc_p.emb.weight"))
    for i in range(cfg["n_layers"]):
        enc_layer("enc.%d" % i, "enc_p.encoder", i, with_tc=enc_tc, need_w=ew, with_tc3=enc_tc3)
    P.conv("enc.proj", g("enc_p.proj.weight"), g("enc_p.proj.bias"), need_w=ew)
    if enc_tc:
        P.conv_tc("enc.proj", g("enc_p.proj.weight"))
    if enc_tc3:
        P.conv_tc3("enc.proj", g("enc_p.proj.weight"))

    # ---- stochastic duration predictor
    P.conv("dp.pre", g("dp.pre.weight"), g("dp.pre.bias"))
    P.conv("dp.proj", g("dp.proj.weight"), g("dp.proj.bias"))
    dds("dp.convs", "dp.convs")
    for n in range(2, cfg["dp_n_flows"] + 1):
        src = "dp.flows.%d" % (2 * n - 1)
        P.add("dp.cf%d.pre_w" % n, g(src + ".pre.weight")[:, 0, 0])
        P.add("dp.cf%d.pre_b" % n, g(src + ".pre.bias"))
        dds("dp.cf%d.convs" % n, src + ".convs")
        P.conv("dp.cf%d.proj" % n, g(src + ".proj.weight"), g(src + ".proj.bias"))
    P.add("dp.ea", np.concatenate([g("dp.flows.0.m").reshape(-1), g("dp.flows.0.logs").reshape(-1)]))

    _pack_flow_decoder(P, g, w, cfg, tc, fw, enc_layer)

    # ---- posterior encoder enc_q (models.py:813-842) + spectrogram front end, for voice conversion
    if posterior:
        if "enc_q.pre.weight" not in w:
            raise ValueError("the state dict has no enc_q (posterior encoder): voice conversion needs a training checkpoint "
                             "(G_*.pth); model.onnx holds only what SynthesizerTrn.infer uses")
        if cfg["flow_n_flows"] % 2:
            raise ValueError("voice conversion needs an even flow_n_flows (the Flip folding of the packed flow holds for both "
                             "directions only then)")
        sc = cfg.get("spec_channels", 80)
        pre = g("enc_q.pre.weight")
        if pre.shape[1] != sc:
            raise ValueError("enc_q.pre has %d input channels, the config says spec_channels=%d" % (pre.shape[1], sc))
        # enc_q.pre runs on the FFMA conv, which takes input channels in multiples of 16: zero-padded (513 -> 528 for a
        # linear spectrogram; the front end writes zeros into the pad columns)
        P.conv("encq.pre", np.pad(pre, ((0, 0), (0, (-sc) % 16), (0, 0))), g("enc_q.pre.bias"))
        _pack_wn_encoder(P, g, "encq", "enc_q", H, tc, fw)
        il = np.arange(2 * H).reshape(2, H).T.reshape(-1)
        nq = 16
        if has_g:
            cw, cb = g("enc_q.enc.cond_layer.weight")[:, :, 0], g("enc_q.enc.cond_layer.bias")
            P.add("encq.cond.w", np.concatenate([cw[i * 2 * H:(i + 1) * 2 * H][il] for i in range(nq)], 0))
            P.add("encq.cond.b", np.concatenate([cb[i * 2 * H:(i + 1) * 2 * H][il] for i in range(nq)], 0))
        n_fft = cfg.get("filter_length", 1024)
        P.add("vc.stft", stft_basis(n_fft))
        if cfg.get("use_mel_posterior_encoder", True):
            P.add("vc.mel", mel_basis(cfg.get("sampling_rate", 22050), n_fft, cfg.get("n_mel_channels", 80),
                                      cfg.get("mel_fmin", 0.0), cfg.get("mel_fmax")))
    return P.finish()


SPK_CTAS = 8      # CTAs of one cluster of the LSTM recurrence kernel (csrc/spk.cuh)


def spk_hh_layout(whh):
    """W_hh [4G][G] (PyTorch gate order i, f, g, o) in the layout of csrc/spk.cuh lstm_rec_kernel: [rank][k][gate * U + unit],
    U = G / SPK_CTAS, CTA `rank` owning hidden units [U rank, U rank + U) of every gate."""
    whh = np.asarray(whh, np.float32)
    G = whh.shape[1]
    U = G // SPK_CTAS
    w = whh.reshape(4, SPK_CTAS, U, G)                  # [gate][rank][unit][k]
    return np.ascontiguousarray(np.transpose(w, (1, 3, 0, 2)))   # [rank][k][gate][unit]


def hann_squared(n_fft):
    """Squared periodic Hann window of n_fft samples: the window envelope torch.istft divides by (vc/stft.py:197-202), summed
    by the tail kernel over the frames that cover each sample."""
    n = np.arange(n_fft)
    return ((0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)) ** 2).astype(np.float32)


CV_POS = "encoder.pos_conv_embed.conv."


def fold_contentvec_pos_conv(sd):
    """The positional conv's weight-norm fold, w = g * v / ||v||, with HubertPositionalConvEmbedding's dim=2: one norm per tap,
    taken over dims 0 and 1 (not fold_weight_norm's dim 0).  Takes weight_g / weight_v (the published checkpoint) or
    parametrizations.weight.original0 / original1 (what transformers 5.x writes); returns the state dict with a plain
    encoder.pos_conv_embed.conv.weight in their place."""
    out = dict(sd)
    for gk, vk in (("weight_g", "weight_v"), ("parametrizations.weight.original0", "parametrizations.weight.original1")):
        if CV_POS + vk in sd:
            g, v = (torch.as_tensor(np.asarray(sd[CV_POS + k]) if isinstance(sd[CV_POS + k], np.ndarray) else sd[CV_POS + k]).float()
                    for k in (gk, vk))
            out[CV_POS + "weight"] = torch._weight_norm(v, g.reshape(1, 1, -1), 2).contiguous()   # what the parametrization computes
            del out[CV_POS + gk], out[CV_POS + vk]
    if CV_POS + "weight" not in out:
        raise ValueError("the state dict has no positional conv weight (%sweight_g/_v or parametrizations)" % CV_POS)
    return out


def load_contentvec(path, config_json=None):
    """A Hugging Face ContentVec / HuBERT checkpoint: `path` a pytorch_model.bin (read with weights_only=True) or a directory
    holding it and config.json.  Returns (folded state dict, cv config): config.contentvec_config of the config.json
    (HubertConfig's defaults without one), the positional conv folded by fold_contentvec_pos_conv."""
    import os
    if os.path.isdir(path):
        if config_json is None and os.path.exists(os.path.join(path, "config.json")):
            config_json = os.path.join(path, "config.json")
        path = os.path.join(path, "pytorch_model.bin")
    cv = _config.contentvec_config(config_json)
    sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k[len("hubert."):] if k.startswith("hubert.") else k: v for k, v in sd.items()}
    return fold_contentvec_pos_conv(sd), cv


def _pack_contentvec(P, sd, cv, tc):
    """cv.* tensors of the engine's ContentVec (csrc/contentvec.cuh, engine.cu cv_enqueue).  Layers 1.. of the feature encoder
    are 1x1 convs over k consecutive rows ([k*C] inputs, tap-major), the positional conv two halves of its taps per group.
    tc: also the split-bf16 copies (.th / .tl) of the projection and the transformer's convs, which precision modes >= 1 run
    on the tensor cores."""
    g = lambda k: sd[k].detach().cpu().float().numpy() if hasattr(sd[k], "detach") else np.asarray(sd[k], np.float32)
    C, H, nl = cv["cv_conv_dim"], cv["cv_hidden"], len(cv["cv_conv_kernel"])
    fe = "feature_extractor.conv_layers.%d."
    w0 = g(fe % 0 + "conv.weight")
    if w0.shape != (C, 1, cv["cv_conv_kernel"][0]):
        raise ValueError("%sconv.weight has shape %s" % (fe % 0, w0.shape))
    P.add("cv.c0.w", w0[:, 0, :])
    P.add("cv.gn.g", g(fe % 0 + "layer_norm.weight"))
    P.add("cv.gn.b", g(fe % 0 + "layer_norm.bias"))
    for i in range(1, nl):
        w = g(fe % i + "conv.weight")                                   # [C, C, k]
        k = w.shape[2]
        P.conv("cv.c%d" % i, np.transpose(w, (0, 2, 1)).reshape(C, k * C)[:, :, None])
    P.add("cv.fp.ln.g", g("feature_projection.layer_norm.weight"))
    P.add("cv.fp.ln.b", g("feature_projection.layer_norm.bias"))
    conv = lambda name, w, b: (P.conv(name, w, b), tc and P.conv_tc(name, w))
    conv("cv.fp", g("feature_projection.projection.weight")[:, :, None], g("feature_projection.projection.bias"))
    pw = g(CV_POS + "weight")                                          # [H, H/G, K]
    G, K = cv["cv_pos_groups"], cv["cv_pos_k"]
    Cg, kh = H // G, K // 2
    if pw.shape != (H, Cg, K):
        raise ValueError("positional conv weight has shape %s, expected %s" % (pw.shape, (H, Cg, K)))
    halves = []
    for half in range(2):
        for gi in range(G):
            blk = pw[gi * Cg:(gi + 1) * Cg, :, half * kh:(half + 1) * kh]   # [Cg out, Cg in, kh]
            halves.append(np.transpose(blk, (2, 1, 0)))                    # [kh][Cg in][Cg out]
    P.add("cv.pos.w", np.stack(halves))
    P.add("cv.pos.b", g(CV_POS + "bias"))
    P.add("cv.enc.ln.g", g("encoder.layer_norm.weight"))
    P.add("cv.enc.ln.b", g("encoder.layer_norm.bias"))
    for l in range(cv["cv_layers"]):
        p = "encoder.layers.%d." % l
        a = p + "attention.%s_proj."
        qkv = np.concatenate([g(a % n + "weight") for n in "qkv"], 0)
        conv("cv.l%d.qkv" % l, qkv[:, :, None], np.concatenate([g(a % n + "bias") for n in "qkv"]))
        conv("cv.l%d.o" % l, g(a % "out" + "weight")[:, :, None], g(a % "out" + "bias"))
        P.add("cv.l%d.ln1.g" % l, g(p + "layer_norm.weight"))
        P.add("cv.l%d.ln1.b" % l, g(p + "layer_norm.bias"))
        conv("cv.l%d.ffn1" % l, g(p + "feed_forward.intermediate_dense.weight")[:, :, None], g(p + "feed_forward.intermediate_dense.bias"))
        conv("cv.l%d.ffn2" % l, g(p + "feed_forward.output_dense.weight")[:, :, None], g(p + "feed_forward.output_dense.bias"))
        P.add("cv.l%d.ln2.g" % l, g(p + "final_layer_norm.weight"))
        P.add("cv.l%d.ln2.b" % l, g(p + "final_layer_norm.bias"))


def pack_quickvc(w, cfg, tc=True, precision=None, contentvec=None, cv=None):
    """QuickVC state dict (folded) -> (blob, manifest) of a model_family "quickvc" engine.

    First the speaker encoder enc_spk and the mel front end of the target (vc/convert.py:60-69): each LSTM layer's input
    projection is a 1x1 conv whose bias is b_ih + b_hh folded; W_hh goes in the CTA-blocked layout of the recurrence kernel;
    the linear layer is stored transposed.  Then, when the state dict has enc_p (a full checkpoint, not an encoder alone), the
    conversion side of SynthesizerTrn.infer (vc/models.py:862-872), after every speaker-encoder tensor so that those keep
    their offsets: encp.* (the content encoder, laid out as pack's encq.*, without cond), flow.* and dec.* as pack lays them
    out, one stacked cond.w / cond.b (the flow's WN cond rows, then dec.cond, the decoder's Conv1d(256, 512, 1)), and
    dec.w2, the squared Hann window of the decoder's inverse STFT.  tc / precision: as in pack (the speaker encoder is fp32
    in every mode).  enc_q and the discriminators, which inference never reads, are left out.  contentvec: a ContentVec state
    dict (load_contentvec, or synthetic.make_random_contentvec) whose cv.* tensors go after everything else, with cv its
    config.contentvec_config (default: hubert-base); without it the blob is what it was before.  Unless tc is off or precision
    is 0, they include the split-bf16 copies of the convs that precision modes >= 1 run on the tensor cores."""
    g = lambda k: w[k].detach().cpu().numpy() if hasattr(w[k], "detach") else np.asarray(w[k])
    P = _Packer()
    for l in range(cfg.get("spk_layers", 3)):
        p = "enc_spk.lstm.%s_l%d"
        P.conv("spk.l%d.ih" % l, g(p % ("weight_ih", l))[:, :, None], g(p % ("bias_ih", l)) + g(p % ("bias_hh", l)))
        P.add("spk.l%d.hh" % l, spk_hh_layout(g(p % ("weight_hh", l))))
    P.add("spk.lin.w", np.ascontiguousarray(g("enc_spk.linear.weight").T))
    P.add("spk.lin.b", g("enc_spk.linear.bias"))
    n_fft = cfg["filter_length"]
    P.add("vc.stft", stft_basis(n_fft))
    P.add("vc.mel", mel_basis(cfg["sampling_rate"], n_fft, cfg["n_mel_channels"], cfg["mel_fmin"], cfg["mel_fmax"]))
    if "enc_p.pre.weight" in w:
        tc = tc and tc_supported(cfg) and precision != 0
        fw = not (tc and precision in (1, 2, 3))
        H = cfg["hidden_channels"]
        pre = g("enc_p.pre.weight")
        if pre.shape[1] != cfg["unit_channels"] or pre.shape[1] % 16:
            raise ValueError("enc_p.pre has %d input channels, expected %d content-unit channels" % (pre.shape[1], cfg["unit_channels"]))
        P.conv("encp.pre", pre, g("enc_p.pre.bias"))
        _pack_wn_encoder(P, g, "encp", "enc_p", H, tc, fw)
        _pack_flow_decoder(P, g, w, cfg, tc, fw)
        rows_w, rows_b = [], []
        _flow_cond_rows(g, cfg, rows_w, rows_b)
        rows_w.append(g("dec.cond.weight")[:, :, 0])
        rows_b.append(g("dec.cond.bias"))
        P.add("cond.w", np.concatenate(rows_w, 0))
        P.add("cond.b", np.concatenate(rows_b, 0))
        P.add("dec.w2", hann_squared(cfg["gen_istft_n_fft"]))
    if contentvec is not None:
        _pack_contentvec(P, fold_contentvec_pos_conv(contentvec) if CV_POS + "weight" not in contentvec else contentvec,
                         cv or _config.contentvec_config(), tc and precision != 0)
    return P.finish()


def _sd_getter(sd):
    g = lambda k: sd[k].detach().cpu().float().numpy() if hasattr(sd[k], "detach") else np.asarray(sd[k], np.float32)

    def want(name, shape):
        a = g(name)
        if tuple(a.shape) != tuple(shape):
            raise ValueError("%s has shape %s, expected %s" % (name, tuple(a.shape), tuple(shape)))
        return a
    return g, want


def _pack_dit_block(P, g, want, dst, src, H, F, k, convs=None):
    """qkv / o / ffn1 / ffn2 of one DiTConVBlock (diffusion_transformer.py:82-96) at state-dict prefix src -> tensors dst.*;
    convs: a dict that also receives each conv's weight [Co, Ci, k] under its tensor name, or None"""
    a = src + "attn.conv_%s."
    ws = {".qkv": (np.concatenate([want(a % n + "weight", (H, H, 1)) for n in "qkv"], 0), np.concatenate([g(a % n + "bias") for n in "qkv"])),
          ".o": (want(a % "o" + "weight", (H, H, 1)), g(a % "o" + "bias")),
          ".ffn1": (want(src + "mlp.conv_1.weight", (F, H, k)), g(src + "mlp.conv_1.bias")),
          ".ffn2": (want(src + "mlp.conv_2.weight", (H, F, k)), g(src + "mlp.conv_2.bias"))}
    for n, (w, b) in ws.items():
        P.conv(dst + n, w, b)
        if convs is not None:
            convs[dst + n] = w


def stabletts_tc_convs(cfg):
    """Names of the StableTTS decoder convs that precision mode 2 runs on the tensor cores (engine.cu bind_stabletts, the
    same rule): those whose input and output widths are both multiples of 64 (TC_BK, one 128-byte swizzle atom of bf16).
    in_proj (x | cond) and final_proj stay on the FFMA pipe: x, the Euler state, and the velocity stay fp32 rows."""
    NC, MC, H, F, NL = (int(cfg[k]) for k in ("noise_channels", "cond_channels", "hidden_channels", "filter_channels", "n_layers"))
    fits = lambda ci, co: ci % 64 == 0 and co % 64 == 0
    names = ["st.cp%d" % i for i, (ci, co) in enumerate(((MC, F), (F, F), (F, H))) if fits(ci, co)]
    for l in range(NL):
        names += ["st.l%d%s" % (l, n) for n, ci, co in ((".qkv", H, 3 * H), (".o", H, H), (".ffn1", H, F), (".ffn2", F, H)) if fits(ci, co)]
    names += ["st.lsc%d" % j for j in range(NL // 2) if fits(2 * H, H)]
    return names


def _pack_stabletts_decoder(P, sd, cfg, precision=1):
    """st.* tensors of the flow-matching decoder; precision 2 appends the split-bf16 copies (.th / .tl) of the convs in
    stabletts_tc_convs(cfg), which that mode runs on the tensor cores."""
    if precision not in (0, 1, 2, 3):
        raise ValueError("precision must be 0, 1, 2 or 3")
    g, want = _sd_getter(sd)
    e = "decoder.estimator."
    NC, MC, H, F, NL, G = (int(cfg[k]) for k in ("noise_channels", "cond_channels", "hidden_channels", "filter_channels", "n_layers",
                                                 "spk_emb_dim"))
    k = int(cfg["kernel_size"])
    convs = {}
    for i, (j, co, ci) in enumerate(((0, F, MC), (2, F, F), (4, H, F))):
        convs["st.cp%d" % i] = want(e + "cond_proj.%d.weight" % j, (co, ci, k))
        P.conv("st.cp%d" % i, convs["st.cp%d" % i], want(e + "cond_proj.%d.bias" % j, (co,)))
    P.conv("st.in", want(e + "in_proj.weight", (H, NC + H, 1)), g(e + "in_proj.bias"))
    P.conv("st.final", want(e + "final_proj.weight", (NC, H, 1)), g(e + "final_proj.bias"))
    P.add("st.time.w1", want(e + "time_mlp.layer.0.weight", (F, H)))
    P.add("st.time.b1", g(e + "time_mlp.layer.0.bias"))
    P.add("st.time.w2", want(e + "time_mlp.layer.2.weight", (H, F)))
    P.add("st.time.b2", g(e + "time_mlp.layer.2.bias"))
    b = e + "blocks.%d."
    P.add("st.film.w", np.stack([want(b % l + "time_fusion.film.weight", (2 * H, H, 1))[:, :, 0] for l in range(NL)]))
    P.add("st.film.b", np.stack([g(b % l + "time_fusion.film.bias") for l in range(NL)]))
    P.add("st.ada.w1", np.stack([want(b % l + "block.adaLN_modulation.0.weight", (H, G)) for l in range(NL)]))
    P.add("st.ada.b1", np.stack([g(b % l + "block.adaLN_modulation.0.bias") for l in range(NL)]))
    P.add("st.ada.w2", np.stack([want(b % l + "block.adaLN_modulation.2.weight", (6 * H, H)) for l in range(NL)]))
    P.add("st.ada.b2", np.stack([g(b % l + "block.adaLN_modulation.2.bias") for l in range(NL)]))
    P.add("st.spk_emb", want("spk_emb.weight", (int(cfg["n_spks"]), G)))
    P.add("st.fake_spk", want("fake_speaker", (1, G)))
    P.add("st.fake_content", want("fake_content", (1, MC, 1)))
    P.add("st.mel_mean", np.asarray(g("mel_mean"), np.float32).reshape(1))
    P.add("st.mel_std", np.asarray(g("mel_std"), np.float32).reshape(1))
    for l in range(NL):
        _pack_dit_block(P, g, want, "st.l%d" % l, b % l + "block.", H, F, k, convs)
    for j in range(NL // 2):
        convs["st.lsc%d" % j] = want(e + "lsc_layers.%d.weight" % j, (H, 2 * H, k))
        P.conv("st.lsc%d" % j, convs["st.lsc%d" % j], g(e + "lsc_layers.%d.bias" % j))
    if precision == 2:
        for name in stabletts_tc_convs(cfg):
            P.conv_tc(name, convs[name])


class _Inert:
    """What a global outside _STATE_DICT_GLOBALS unpickles to: it accepts any arguments and state and does nothing, so a
    checkpoint's hyper-parameters (Hydra configs, functools.partial of an optimizer) load as placeholders and nothing named
    in the file is imported or called."""

    def __init__(self, *args, **kwargs):
        pass

    def __call__(self, *args, **kwargs):
        return _Inert()

    def __setstate__(self, state):
        pass

    def __setitem__(self, key, value):
        pass

    def append(self, value):
        pass

    def extend(self, values):
        pass


# the globals a state dict of tensors needs; storages are resolved by torch.load itself
_STATE_DICT_GLOBALS = {
    ("collections", "OrderedDict"): "collections.OrderedDict",
    ("torch", "Size"): "torch.Size",
    ("torch._utils", "_rebuild_tensor"): "torch._utils._rebuild_tensor",
    ("torch._utils", "_rebuild_tensor_v2"): "torch._utils._rebuild_tensor_v2",
    ("torch._utils", "_rebuild_parameter"): "torch._utils._rebuild_parameter",
    ("torch._utils", "_rebuild_parameter_with_state"): "torch._utils._rebuild_parameter_with_state",
    ("torch._tensor", "_rebuild_from_type_v2"): "torch._tensor._rebuild_from_type_v2",
    ("torch._tensor", "Tensor"): "torch.Tensor",
    ("torch.nn.parameter", "Parameter"): "torch.nn.Parameter",
}


def _state_dict_pickle_module():
    import importlib
    import pickle
    import types

    class Unpickler(pickle.Unpickler):
        def find_class(self, module, name):
            if (module, name) not in _STATE_DICT_GLOBALS:
                return _Inert
            mod, _, attr = _STATE_DICT_GLOBALS[(module, name)].rpartition(".")
            return getattr(importlib.import_module(mod), attr)

    m = types.ModuleType("vtts_state_dict_pickle")
    m.Unpickler, m.load = Unpickler, pickle.load
    m.__dict__.update({k: getattr(pickle, k) for k in ("UnpicklingError", "HIGHEST_PROTOCOL")})
    return m


def load_lightning_state_dict(path):
    """The state dict of a PyTorch Lightning checkpoint (`{"state_dict": ..., "hyper_parameters": ..., ...}`, as the
    reference's training/stabletts writes `*.ckpt`), or of a file holding the state dict alone, with the weight norm folded.
    torch.load(weights_only=True) refuses such a checkpoint: its hyper_parameters hold Hydra configs and a functools.partial of
    the optimizer.  The file is read with an unpickler that resolves only the globals a state dict of tensors needs and turns
    every other one into an inert placeholder, so loading imports and runs nothing the file names."""
    ck = torch.load(path, map_location="cpu", weights_only=False, pickle_module=_state_dict_pickle_module())
    sd = ck["state_dict"] if isinstance(ck, dict) and "state_dict" in ck else ck
    if not isinstance(sd, dict) or not all(isinstance(v, torch.Tensor) for v in sd.values()):
        raise ValueError("%s holds no state dict of tensors" % path)
    return fold_weight_norm(sd)


def load_hifigan(path):
    """A HiFi-GAN checkpoint of StableTTS's vocoder (cli.py:65-71: `{"generator": state_dict}`, generator_v1 / hifigan_T2_v1)
    -> its state dict with the weight norm folded, as remove_weight_norm leaves it.  Read with weights_only=True."""
    ck = torch.load(path, map_location="cpu", weights_only=True)
    return fold_weight_norm(ck["generator"] if isinstance(ck, dict) and "generator" in ck else ck)


def _pack_hifigan(P, sd, h):
    """The Generator (matcha/hifigan/models.py:148-206) of a folded state dict under the decoder names csrc/engine.cu binds:
    dec.pre, dec.up<i>.p<r> (the polyphase phases of each ConvTranspose1d), dec.rb<n>.c1/c2.<d> (ResBlock1) or .c.<d>
    (ResBlock2) and dec.post.  Every conv is packed for the FFMA pipe; those whose input width is a multiple of 64 also as
    split-bf16 planes, which precision modes >= 1 read."""
    g, want = _sd_getter(sd)
    c0, nm = int(h["upsample_initial_channel"]), int(h["num_mels"])
    tc = lambda ci: ci % 64 == 0

    def conv(dst, w, b):
        P.conv(dst, w, b)
        if tc(w.shape[1]):
            P.conv_tc(dst, w)
    P.conv("dec.pre", want("conv_pre.weight", (c0, nm, 7)), g("conv_pre.bias"))
    ch = c0
    nk = len(h["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        wt = want("ups.%d.weight" % i, (ch, ch // 2, k))               # ConvTranspose1d: [Cin, Cout, K]
        for r, (pad, js) in enumerate(convt_phases(u, k, (k - u) // 2)):
            conv("dec.up%d.p%d" % (i, r), np.transpose(np.stack([wt[:, :, j] for j in js], axis=-1), (1, 0, 2)), g("ups.%d.bias" % i))
        ch //= 2
        for j, (ks, dils) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            n = i * nk + j
            for d in range(len(dils)):
                if h["resblock"] == "1":
                    for m in (1, 2):
                        src = "resblocks.%d.convs%d.%d." % (n, m, d)
                        conv("dec.rb%d.c%d.%d" % (n, m, d), want(src + "weight", (ch, ch, ks)), g(src + "bias"))
                else:
                    src = "resblocks.%d.convs.%d." % (n, d)
                    P.conv("dec.rb%d.c.%d" % (n, d), want(src + "weight", (ch, ch, ks)), g(src + "bias"))
    P.conv("dec.post", want("conv_post.weight", (1, ch, 7)), g("conv_post.bias"))


def pack_hifigan(sd, h):
    """The vocoder alone -> (blob, manifest) (see _pack_hifigan); h: config.hifigan_config."""
    P = _Packer()
    _pack_hifigan(P, sd, h)
    return P.finish()


def _bert_from_onnx(path, heads, layer_norm_eps):
    """The BERT graph bert-export.py writes (bert/model.onnx of a multistream model) -> (state dict, config.bert_config).
    Named initializers are taken as they are; each Linear's weight is recovered from the MatMul whose output the Add of its
    `<module>.bias` consumes (onnx_weights.state_dict_from_onnx).  The graph holds only the layers hidden_states[-3] depends on,
    and that count is the number that runs.  Widths and table rows follow from the tensors; the head count and the LayerNorm
    eps are not in the graph's weights, so they come from a config.json beside it or from the arguments (rubert-base's)."""
    import os
    import re
    from . import onnx_weights
    sd = onnx_weights.state_dict_from_onnx(path)
    layers = sorted({int(m.group(1)) for m in (re.match(r"encoder\.layer\.(\d+)\.", k) for k in sd) if m})
    if "embeddings.word_embeddings.weight" not in sd or not layers or layers != list(range(len(layers))):
        raise ValueError("%s is not a BERT graph of bert-export.py (no embeddings / encoder.layer.<i> tensors)" % path)
    cfg = {"num_attention_heads": heads, "layer_norm_eps": layer_norm_eps}
    side = os.path.join(os.path.dirname(os.path.abspath(path)), "config.json")
    if os.path.exists(side):
        with open(side) as f:
            cfg.update({k: v for k, v in json.load(f).items() if k in ("num_attention_heads", "layer_norm_eps", "hidden_act")})
    word, pos, typ = (sd["embeddings.%s_embeddings.weight" % n] for n in ("word", "position", "token_type"))
    cfg.update({"hidden_size": word.shape[1], "vocab_size": word.shape[0], "max_position_embeddings": pos.shape[0],
                "type_vocab_size": typ.shape[0], "intermediate_size": sd["encoder.layer.0.intermediate.dense.weight"].shape[0]})
    for l in layers:
        if "encoder.layer.%d.output.dense.weight" % l not in sd:
            raise ValueError("%s: the Linear weights of layer %d were not recovered from the graph" % (path, l))
    return sd, _config.bert_config(cfg, layers=len(layers))


def load_bert(path, heads=12, layer_norm_eps=1e-12):
    """A BERT checkpoint -> (state dict in BertModel's names, config.bert_config).  `path` is either
    - bert-export.py's ONNX graph (a .onnx file, or a directory holding model.onnx, as a multistream model's bert/ does): the
      layers that run are the ones the graph holds; heads and layer_norm_eps come from a config.json beside it, else from the
      arguments (rubert-base's 12 and 1e-12); or
    - a Hugging Face checkpoint directory (config.json and pytorch_model.bin, read with weights_only=True, or
      model.safetensors): the layers that run are num_hidden_layers - 2, as bert-export.py's hidden_states[-3] leaves them.
      A BertForMaskedLM / BertForPreTraining checkpoint's `bert.` prefix is dropped; its heads are not read."""
    import os
    if os.path.isfile(path) and path.endswith(".onnx"):
        return _bert_from_onnx(path, heads, layer_norm_eps)
    if not os.path.isdir(path):
        raise ValueError("%s: a BERT checkpoint is bert-export.py's .onnx graph or a directory holding model.onnx, or config.json "
                         "and pytorch_model.bin or model.safetensors" % path)
    st, pt = os.path.join(path, "model.safetensors"), os.path.join(path, "pytorch_model.bin")
    if not os.path.exists(st) and not os.path.exists(pt) and os.path.exists(os.path.join(path, "model.onnx")):
        return _bert_from_onnx(os.path.join(path, "model.onnx"), heads, layer_norm_eps)
    bt = _config.bert_config(os.path.join(path, "config.json") if os.path.exists(os.path.join(path, "config.json")) else None)
    if os.path.exists(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    elif os.path.exists(pt):
        sd = torch.load(pt, map_location="cpu", weights_only=True)
    else:
        raise ValueError("%s holds none of model.onnx, model.safetensors and pytorch_model.bin" % path)
    sd = {k[len("bert."):] if k.startswith("bert.") else k: v for k, v in sd.items()}
    return sd, bt


def _pack_bert(P, sd, bt, tc):
    """bt.* tensors of the engine's BERT (csrc/bert.cuh, engine.cu bt_enqueue): the three embedding tables row-major and their
    LayerNorm, then per layer that runs (bt["cv_layers"]) the fused q | k | v 1x1 conv, the attention's output conv, the FFN's
    two convs and both LayerNorms, laid out as ContentVec's.  tc: also the split-bf16 copies (.th / .tl) that precision modes
    >= 1 run on the tensor cores."""
    g, want = _sd_getter(sd)
    H, F, V, NP, NT = (int(bt[k]) for k in ("cv_hidden", "cv_ffn", "bt_vocab", "bt_max_pos", "bt_type_rows"))
    e = "embeddings."
    P.add("bt.emb.word", want(e + "word_embeddings.weight", (V, H)))
    P.add("bt.emb.pos", want(e + "position_embeddings.weight", (NP, H)))
    P.add("bt.emb.type", want(e + "token_type_embeddings.weight", (NT, H)))
    P.add("bt.emb.ln.g", want(e + "LayerNorm.weight", (H,)))
    P.add("bt.emb.ln.b", want(e + "LayerNorm.bias", (H,)))
    conv = lambda name, w, b: (P.conv(name, w[:, :, None], b), tc and P.conv_tc(name, w[:, :, None]))
    for l in range(int(bt["cv_layers"])):
        p = "encoder.layer.%d." % l
        a = p + "attention.self.%s."
        conv("bt.l%d.qkv" % l, np.concatenate([want(a % n + "weight", (H, H)) for n in ("query", "key", "value")], 0),
             np.concatenate([want(a % n + "bias", (H,)) for n in ("query", "key", "value")]))
        conv("bt.l%d.o" % l, want(p + "attention.output.dense.weight", (H, H)), want(p + "attention.output.dense.bias", (H,)))
        P.add("bt.l%d.ln1.g" % l, want(p + "attention.output.LayerNorm.weight", (H,)))
        P.add("bt.l%d.ln1.b" % l, want(p + "attention.output.LayerNorm.bias", (H,)))
        conv("bt.l%d.ffn1" % l, want(p + "intermediate.dense.weight", (F, H)), want(p + "intermediate.dense.bias", (F,)))
        conv("bt.l%d.ffn2" % l, want(p + "output.dense.weight", (H, F)), want(p + "output.dense.bias", (H,)))
        P.add("bt.l%d.ln2.g" % l, want(p + "output.LayerNorm.weight", (H,)))
        P.add("bt.l%d.ln2.b" % l, want(p + "output.LayerNorm.bias", (H,)))


def pack_bert(sd, bt, tc=True):
    """BERT alone -> (blob, manifest) (see _pack_bert); bt: config.bert_config.  StableTTS(..., bert=...) appends the same
    tensors to its blob through pack_stabletts(..., bert=...)."""
    P = _Packer()
    _pack_bert(P, sd, bt, tc)
    return P.finish()


def pack_stabletts_cfm(sd, cfg, vocoder=None, bert=None, precision=1):
    """The flow-matching decoder of a MatchaTTS (StableTTS) state dict -> (blob, manifest) of a model_family "stabletts" engine.
    sd: the checkpoint's `state_dict` entry (keys decoder.estimator.*, spk_emb.weight, fake_speaker, fake_content, mel_mean,
    mel_std); cfg: config.stabletts_cfm_config.  Convs go in the FFMA layout (q, k, v stacked into one 1x1 conv), the small
    linears of the conditioning path (time_mlp, each block's film conv and adaLN_modulation) row-major [out][in] and stacked
    over the blocks, all fp32.  precision: the engine's precision mode; 2 also packs the split-bf16 copies (.th / .tl) of the
    convs that mode runs on the tensor cores (stabletts_tc_convs), the other modes the same blob as each other.  vocoder:
    (folded Generator state dict, config.hifigan_config) appended as pack_hifigan lays it out, or None; bert: (BertModel
    state dict, config.bert_config, tc) appended as pack_bert lays it out, or None."""
    P = _Packer()
    _pack_stabletts_decoder(P, sd, cfg, precision)
    if vocoder is not None:
        _pack_hifigan(P, *vocoder)
    if bert is not None:
        _pack_bert(P, *bert)
    return P.finish()


def pack_stabletts(sd, cfg, vocoder=None, bert=None, precision=1):
    """A MatchaTTS (StableTTS) state dict without its vocoder -> (blob, manifest) of an engine that serves text-to-mel
    (vtts_stabletts_synthesise) and the decoder alone: the decoder part of pack_stabletts_cfm, then the text encoder
    (encoder.emb, encoder.punc_emb, encoder.bert_proj.1, both stacks encoder.encoder / encoder.dp_encoder with their proj) and
    dur_spk_emb.  Without encoder.encoder.* (a state dict read from an exported graph, onnx_weights.stabletts_from_onnx) the
    engine serves everything but the prior.  cfg: config.stabletts_config; vocoder and precision as in pack_stabletts_cfm (the
    text encoder is fp32 in every mode); bert: (BertModel state dict, config.bert_config, tc) appended as pack_bert lays it
    out, or None."""
    if "enc_n_layers" not in cfg:
        raise ValueError("pack_stabletts needs config.stabletts_config (the text encoder's constants), not stabletts_cfm_config")
    g, want = _sd_getter(sd)
    P = _Packer()
    _pack_stabletts_decoder(P, sd, cfg, precision)
    V, E, PD, BD, R, H, F, NE, G, DC = (int(cfg[k]) for k in ("n_vocab", "emb_dim", "punc_dim", "bert_dim", "bert_proj_dim",
                                                             "enc_hidden_channels", "enc_filter_channels", "enc_n_layers", "spk_emb_dim",
                                                             "dur_channels"))
    k = int(cfg["enc_kernel_size"])
    P.add("st.enc.emb", want("encoder.emb.weight", (V, E)))
    P.add("st.enc.punc", want("encoder.punc_emb.weight", (V, PD)))
    P.add("st.enc.bert.w", want("encoder.bert_proj.1.weight", (R, BD)))
    P.add("st.enc.bert.b", want("encoder.bert_proj.1.bias", (R,)))
    P.add("st.dur_spk_emb", want("dur_spk_emb.weight", (int(cfg["n_spks"]), G)))
    for dst, src, co in (("st.enc.mel", "encoder.encoder.", int(cfg["noise_channels"])), ("st.enc.dp", "encoder.dp_encoder.", DC)):
        if dst == "st.enc.mel" and src + "proj.weight" not in sd:
            continue            # the mel encoder feeds only the prior; an exported graph does not carry it
        b = src + "encoder.%d."
        for l in range(NE):
            _pack_dit_block(P, g, want, "%s.l%d" % (dst, l), b % l, H, F, k)
        P.add(dst + ".ada.w1", np.stack([want(b % l + "adaLN_modulation.0.weight", (H, G)) for l in range(NE)]))
        P.add(dst + ".ada.b1", np.stack([g(b % l + "adaLN_modulation.0.bias") for l in range(NE)]))
        P.add(dst + ".ada.w2", np.stack([want(b % l + "adaLN_modulation.2.weight", (6 * H, H)) for l in range(NE)]))
        P.add(dst + ".ada.b2", np.stack([g(b % l + "adaLN_modulation.2.bias") for l in range(NE)]))
        P.conv(dst + ".proj", want(src + "proj.weight", (co, H, 1)), g(src + "proj.bias"))
    if vocoder is not None:
        _pack_hifigan(P, *vocoder)
    if bert is not None:
        _pack_bert(P, *bert)
    return P.finish()


def load_t2s(path):
    """A GPT-SoVITS text-to-semantic checkpoint -> (fp32 state dict in Text2SemanticDecoder's names, config.t2s_config).  Both
    layouts the reference writes are read:
    - PyTorch Lightning's (`state_dict` with `model.*` keys, `hyper_parameters.config`), as inference_cli.py:85-97 loads it;
    - the half-weight export of s1_train.py:73-90 (`weight` in fp16, `config`), as onnx_export.py:89-92 loads it.
    The file is read with the restricted unpickler of load_lightning_state_dict: nothing it names is imported or called."""
    ck = torch.load(path, map_location="cpu", weights_only=False, pickle_module=_state_dict_pickle_module())
    if not isinstance(ck, dict):
        raise ValueError("%s is not a GPT-SoVITS text-to-semantic checkpoint" % path)
    if "state_dict" in ck:
        hp = ck.get("hyper_parameters")
        conf = hp.get("config") if isinstance(hp, dict) else None
        sd = {k[len("model."):]: v for k, v in ck["state_dict"].items() if k.startswith("model.")}
    elif "weight" in ck:
        conf, sd = ck.get("config"), ck["weight"]
    else:
        raise ValueError("%s holds neither `state_dict` (Lightning) nor `weight` (half-weight export)" % path)
    if not isinstance(conf, dict) or not isinstance(conf.get("model"), dict):
        raise ValueError("%s carries no config with a `model` block" % path)
    if not isinstance(sd, dict) or not sd or not all(isinstance(v, torch.Tensor) for v in sd.values()):
        raise ValueError("%s holds no state dict of tensors" % path)
    sd = {k: v.float() for k, v in sd.items()}
    return sd, _config.t2s_config(conf["model"], sd)


def t2s_sine_table(n, dim):
    """SinePositionalEmbedding.extend_pe (ar/modules/embedding.py:53-76) in fp32 on the host, with the reference's formula."""
    position = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe = torch.zeros(n, dim)
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe.numpy()


def pack_t2s(sd, cfg, tc=True):
    """Text2SemanticDecoder (config.t2s_config) -> (blob, manifest) of a model_family "t2s" engine: t2s.temb / t2s.aemb (the
    phone and semantic embedding tables), t2s.pe (the sine table, computed here), t2s.alpha (text, audio), t2s.bert_proj and
    t2s.pred (ar_predict_layer, zero bias) as 1x1 convs, then per layer the in_proj q | k | v conv, out_proj, norm1, linear1,
    linear2 and norm2.  tc: also the split-bf16 copies (.th / .tl) of the layer convs, which the prefill reads in precision
    modes >= 1."""
    g, want = _sd_getter(sd)
    H, F, V, PV, L = (int(cfg[k]) for k in ("cv_hidden", "cv_ffn", "t2s_vocab", "t2s_phone_vocab", "cv_layers"))
    P = _Packer()
    P.add("t2s.temb", want("ar_text_embedding.word_embeddings.weight", (PV, H)))
    P.add("t2s.aemb", want("ar_audio_embedding.word_embeddings.weight", (V, H)))
    P.add("t2s.pe", t2s_sine_table(int(cfg["t2s_positions"]), H))
    P.add("t2s.alpha", np.array([float(want("ar_text_position.alpha", (1,))[0]), float(want("ar_audio_position.alpha", (1,))[0])]))
    P.conv("t2s.bert_proj", want("bert_proj.weight", (H, 1024))[:, :, None], want("bert_proj.bias", (H,)))
    P.conv("t2s.pred", want("ar_predict_layer.weight", (V, H))[:, :, None], np.zeros(V, np.float32))
    conv = lambda name, w, b: (P.conv(name, w[:, :, None], b), tc and P.conv_tc(name, w[:, :, None]))
    for l in range(L):
        p = "h.layers.%d." % l
        conv("t2s.l%d.qkv" % l, want(p + "self_attn.in_proj_weight", (3 * H, H)), want(p + "self_attn.in_proj_bias", (3 * H,)))
        conv("t2s.l%d.o" % l, want(p + "self_attn.out_proj.weight", (H, H)), want(p + "self_attn.out_proj.bias", (H,)))
        P.add("t2s.l%d.ln1.g" % l, want(p + "norm1.weight", (H,)))
        P.add("t2s.l%d.ln1.b" % l, want(p + "norm1.bias", (H,)))
        conv("t2s.l%d.ffn1" % l, want(p + "linear1.weight", (F, H)), want(p + "linear1.bias", (F,)))
        conv("t2s.l%d.ffn2" % l, want(p + "linear2.weight", (H, F)), want(p + "linear2.bias", (H,)))
        P.add("t2s.l%d.ln2.g" % l, want(p + "norm2.weight", (H,)))
        P.add("t2s.l%d.ln2.b" % l, want(p + "norm2.bias", (H,)))
    return P.finish()
