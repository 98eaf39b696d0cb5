"""Checkpoint -> engine weights: weight-norm folding and the packed device blob.

Contract (SURVEY.md section 5 "Checkpoint / resume"; /root/reference/training/vits2/utils.py:18-50,
onnx_export.py:55,78-79): a ``G_*.pth`` holds ``{'model': state_dict, ...}`` with weight-normed convs
stored as ``weight_g`` / ``weight_v``; the exporter loads it and removes weight norm on ``dec`` and
``flow`` before tracing.  ``fold_weight_norm`` performs the same fold; ``pack`` (below) lays every
tensor out the way the CUDA kernels consume it.
"""
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
