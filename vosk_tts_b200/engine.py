"""ctypes binding of libvtts.so (include/vtts.h).  No CPU fallback: importing works without a GPU
(the library only needs libcudart), creating an Engine requires a CUDA device."""
import ctypes as C
import os

import numpy as np

from . import build as _build
from . import config as _config

_LIB = None


class VttsError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("vtts error %d: %s" % (code, msg))
        self.code = code


class VttsConfig(C.Structure):
    _fields_ = [
        ("n_vocab", C.c_int32), ("n_speakers", C.c_int32), ("gin_channels", C.c_int32),
        ("inter_channels", C.c_int32), ("hidden_channels", C.c_int32), ("filter_channels", C.c_int32),
        ("n_heads", C.c_int32), ("n_layers", C.c_int32), ("kernel_size", C.c_int32), ("window_size", C.c_int32),
        ("spk_cond_encoder", C.c_int32), ("cond_layer_idx", C.c_int32),
        ("use_transformer_flows", C.c_int32),
        ("flow_kernel_size", C.c_int32), ("flow_dilation_rate", C.c_int32), ("flow_wn_layers", C.c_int32),
        ("flow_n_flows", C.c_int32),
        ("dp_filter_channels", C.c_int32), ("dp_kernel_size", C.c_int32), ("dp_n_flows", C.c_int32),
        ("dp_num_bins", C.c_int32),
        ("dp_tail_bound", C.c_float),
        ("decoder_type", C.c_int32), ("resblock_type", C.c_int32),
        ("n_resblock_kernels", C.c_int32), ("resblock_kernel_sizes", C.c_int32 * 8),
        ("n_resblock_dilations", C.c_int32), ("resblock_dilations", (C.c_int32 * 8) * 8),
        ("n_upsamples", C.c_int32), ("upsample_rates", C.c_int32 * 8), ("upsample_kernel_sizes", C.c_int32 * 8),
        ("upsample_initial_channel", C.c_int32),
        ("subbands", C.c_int32), ("istft_n_fft", C.c_int32), ("istft_hop", C.c_int32),
        ("precision", C.c_int32), ("flow_n_heads", C.c_int32),
        ("spec_channels", C.c_int32), ("use_mel_posterior_encoder", C.c_int32),
        ("filter_length", C.c_int32), ("hop_length", C.c_int32), ("win_length", C.c_int32), ("n_mel_channels", C.c_int32),
        ("mel_fmin", C.c_float), ("mel_fmax", C.c_float),
        ("model_family", C.c_int32),
        ("cv_layers", C.c_int32), ("cv_hidden", C.c_int32), ("cv_heads", C.c_int32), ("cv_ffn", C.c_int32),
        ("cv_conv_dim", C.c_int32), ("cv_n_conv", C.c_int32), ("cv_conv_kernel", C.c_int32 * 8), ("cv_conv_stride", C.c_int32 * 8),
        ("cv_pos_k", C.c_int32), ("cv_pos_groups", C.c_int32), ("cv_ln_eps", C.c_float), ("cv_gn_eps", C.c_float),
    ]


EXPORTS = ["vtts_create", "vtts_destroy", "vtts_last_error", "vtts_durations", "vtts_synthesize",
           "vtts_durations_dev", "vtts_synthesize_dev", "vtts_hop", "vtts_stage_timings",
           "vtts_kernel_launches", "vtts_stream", "vtts_microbench", "vtts_debug_flags", "vtts_debug_read",
           "vtts_profile", "vtts_profile_read", "vtts_set_graphs", "vtts_graph_replays",
           "vtts_profile_read_tc", "vtts_timeline", "vtts_infer", "vtts_infer_dev",
           "vtts_decoder_halo", "vtts_flow", "vtts_decode_chunk", "vtts_debug_attention", "vtts_speculation_stats", "vtts_host_timings",
           "vtts_maximum_path", "vtts_maximum_path_dev", "vtts_convert", "vtts_convert_spec", "vtts_debug_conv",
           "vtts_debug_conv_log", "vtts_tc_split_plan", "vtts_align", "vtts_align_spec", "vtts_speaker_embedding",
           "vtts_speaker_embedding_mel", "vtts_quickvc_convert", "vtts_content_units",
           "vtts_quickvc_convert_wav"]

MODEL_FAMILIES = {"vits2": 0, "quickvc": 1}    # vtts_config.model_family

CONV_KEEP = -1000000     # VTTS_CONV_KEEP: leave a launch-shape setting at the engine's value


class ConvProblem(C.Structure):
    """vtts_conv_problem (include/vtts.h)."""
    _fields_ = [(n, C.c_int32) for n in ("Cin", "Cout", "k", "dil", "pad", "out_mul", "out_add", "in_extra", "out_seq_extra",
                                         "epi")] + \
        [("alpha", C.c_float), ("pl_slope", C.c_float), ("w_hi", C.c_void_p), ("w_mid", C.c_void_p), ("w_lo", C.c_void_p),
         ("w", C.c_void_p), ("bias", C.c_void_p), ("cond", C.c_void_p), ("cond_ld", C.c_int32)] + \
        [(n, C.c_int32) for n in ("y_on", "ldy", "yoff", "res", "ldr", "roff", "planes_on", "ldp", "poff", "ldx", "xoff",
                                  "reflect", "pro")] + [("slope", C.c_float)]


CONV_OVERRIDES = ("tc_bn", "tc_split", "tc_tall", "tc_mc", "tc_persist", "tc_wmc", "tc_min_steps", "conv_max_s", "conv_min_g",
                  "conv_max_g", "conv_big_g")


class ConvOverrides(C.Structure):
    _fields_ = [(n, C.c_int32) for n in CONV_OVERRIDES]


class ConvReport(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("use_tc", "bn", "split", "tall", "cn", "wmc", "persist", "np", "ast", "wst", "image",
                                         "S", "G", "grid_x", "grid_y", "grid_z")] + [("psplit", C.c_int32 * 4)]

    def as_dict(self):
        """psplit is a list of the per-problem splits (as many as the launch had problems)."""
        d = {n: int(getattr(self, n)) for n, _ in self._fields_ if n != "psplit"}
        d["psplit"] = [int(s) for s in self.psplit if s]
        return d


ATTN_KERNELS = {"auto": 0, "tc": 1, "split": 2, "r1": 3, "r4": 4, "ffma": 5}    # VTTS_ATTN_*


class AttnReport(C.Structure):
    """vtts_attn_report: the attention launch that ran."""
    _fields_ = [(n, C.c_int32) for n in ("kernel", "dk", "R", "grid_x", "grid_y", "grid_z", "smem")]

    def as_dict(self):
        d = {n: int(getattr(self, n)) for n, _ in self._fields_}
        d["kernel"] = {v: k for k, v in ATTN_KERNELS.items()}.get(d["kernel"], d["kernel"])
        return d


class _Missing:
    """Stand-in for an entry point an alternative build (VTTS_LIB) does not export: accepts the argtypes / restype
    assignments of load_library and raises when called."""

    def __init__(self, name):
        self._name = name

    def __call__(self, *a):
        raise RuntimeError("%s is not exported by the library selected with VTTS_LIB" % self._name)


class _TolerantLib:
    def __init__(self, lib):
        object.__setattr__(self, "_lib", lib)
        object.__setattr__(self, "_missing", {})

    def __getattr__(self, name):
        try:
            return getattr(self._lib, name)
        except AttributeError:
            return self._missing.setdefault(name, _Missing(name))


def lib_path():
    return _build.LIB


def load_library(build_if_missing=True):
    """dlopen the in-tree libvtts.so; fails loudly if it is missing and cannot be built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.environ.get("VTTS_LIB") or _build.LIB       # VTTS_LIB: load an alternative build (kernel A/B experiments)
    if not os.path.exists(path):
        if not build_if_missing:
            raise RuntimeError("libvtts.so is missing: run `python -m vosk_tts_b200.build`")
        _build.build()
    lib = C.CDLL(path)
    if os.environ.get("VTTS_LIB"):
        lib = _TolerantLib(lib)                 # an older build loaded for an A/B may lack the newest entry points
    vp, i32, i64p, fp = C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_float)
    lib.vtts_create.argtypes = [C.POINTER(VttsConfig), vp, C.c_size_t, C.c_char_p, i32, i32, C.POINTER(vp)]
    lib.vtts_create.restype = i32
    lib.vtts_destroy.argtypes = [vp]
    lib.vtts_destroy.restype = None
    lib.vtts_last_error.argtypes = [vp]
    lib.vtts_last_error.restype = C.c_char_p
    lib.vtts_durations.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, C.c_uint64, vp, vp]
    lib.vtts_durations.restype = i32
    lib.vtts_synthesize.argtypes = [vp, vp, i32, vp, C.c_int64, vp, i32]
    lib.vtts_synthesize.restype = i32
    lib.vtts_durations_dev.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, C.c_uint64, vp]
    lib.vtts_durations_dev.restype = i32
    lib.vtts_synthesize_dev.argtypes = [vp, vp, i32, vp, C.c_int64]
    lib.vtts_synthesize_dev.restype = i32
    lib.vtts_infer.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, i32, C.c_uint64, vp, vp, C.c_int64, vp, i32]
    lib.vtts_infer.restype = i32
    lib.vtts_infer_dev.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, vp, i32, C.c_uint64, vp, vp, C.c_int64]
    lib.vtts_infer_dev.restype = i32
    lib.vtts_decoder_halo.argtypes = [vp]
    lib.vtts_decoder_halo.restype = i32
    lib.vtts_flow.argtypes = [vp, vp, i32]
    lib.vtts_flow.restype = i32
    lib.vtts_decode_chunk.argtypes = [vp, i32, i32, vp, C.c_int64]
    lib.vtts_decode_chunk.restype = i32
    lib.vtts_hop.argtypes = [vp]
    lib.vtts_hop.restype = i32
    lib.vtts_stage_timings.argtypes = [vp, vp, i32]
    lib.vtts_stage_timings.restype = i32
    lib.vtts_kernel_launches.argtypes = [vp]
    lib.vtts_kernel_launches.restype = C.c_uint64
    lib.vtts_stream.argtypes = [vp]
    lib.vtts_stream.restype = vp
    lib.vtts_microbench.argtypes = [vp, C.c_char_p, i32]
    lib.vtts_microbench.restype = C.c_float
    lib.vtts_debug_flags.argtypes = [vp, i32]
    lib.vtts_debug_flags.restype = i32
    lib.vtts_debug_read.argtypes = [vp, C.c_char_p, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.vtts_debug_read.restype = i32
    lib.vtts_set_graphs.argtypes = [vp, i32]
    lib.vtts_set_graphs.restype = i32
    lib.vtts_graph_replays.argtypes = [vp]
    lib.vtts_graph_replays.restype = C.c_uint64
    lib.vtts_profile.argtypes = [vp, i32]
    lib.vtts_profile.restype = i32
    lib.vtts_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
    lib.vtts_timeline.argtypes = [vp, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.vtts_timeline.restype = i32
    lib.vtts_profile_read.restype = i32
    lib.vtts_profile_read_tc.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_double)]
    lib.vtts_profile_read_tc.restype = i32
    lib.vtts_debug_attention.argtypes = [vp, C.c_char_p, i32, vp, vp, vp, C.c_size_t, i32, vp, vp, i32, i32, fp,
                                         C.POINTER(AttnReport)]
    lib.vtts_debug_attention.restype = i32
    lib.vtts_debug_conv.argtypes = [vp, i32, i32, vp, i32, i32, C.POINTER(ConvProblem), vp, C.c_size_t, i32, vp, C.c_size_t, vp,
                                    C.c_size_t, vp, C.c_size_t, i32, C.POINTER(ConvOverrides), C.POINTER(ConvReport)]
    lib.vtts_debug_conv.restype = i32
    lib.vtts_debug_conv_log.argtypes = [vp, i32, C.POINTER(ConvReport), i32, C.POINTER(C.c_int)]
    lib.vtts_debug_conv_log.restype = i32
    lib.vtts_tc_split_plan.argtypes = [i32, vp, vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, i32, vp, vp]
    lib.vtts_tc_split_plan.restype = i32
    lib.vtts_speculation_stats.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.vtts_speculation_stats.restype = i32
    lib.vtts_host_timings.argtypes = [vp, C.POINTER(C.c_double), i32]
    lib.vtts_host_timings.restype = i32
    lib.vtts_maximum_path.argtypes = [vp, vp, vp, i32, i32, i32, vp, i32]
    lib.vtts_maximum_path.restype = i32
    lib.vtts_maximum_path_dev.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp]
    lib.vtts_maximum_path_dev.restype = i32
    for nm in ("vtts_convert", "vtts_convert_spec"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, vp, vp, i32, C.c_int64, vp, vp, C.c_float, vp, i32, C.c_uint64, vp, C.c_int64, vp]
        fn.restype = i32
    for nm in ("vtts_align", "vtts_align_spec"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, vp, vp, i32, vp, vp, vp, i32, C.c_int64, C.c_float, vp, i32, C.c_uint64, vp, vp, C.c_int64, vp, vp]
        fn.restype = i32
    for nm in ("vtts_speaker_embedding", "vtts_speaker_embedding_mel"):
        fn = getattr(lib, nm)
        fn.argtypes = [vp, vp, vp, i32, C.c_int64, vp]
        fn.restype = i32
    lib.vtts_quickvc_convert.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_float, vp, i32, C.c_uint64, vp, C.c_int64, vp]
    lib.vtts_quickvc_convert.restype = i32
    lib.vtts_content_units.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_int64, vp]
    lib.vtts_content_units.restype = i32
    lib.vtts_quickvc_convert_wav.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_float, vp, i32, C.c_uint64, vp, C.c_int64, vp]
    lib.vtts_quickvc_convert_wav.restype = i32
    _LIB = lib
    return lib


def tc_split_plan(problems, lens, rmul, n_sm, cluster_cap, max_len=None, bn=0, max_split=8, min_steps=2):
    """The engine's split-K plan of one grouped tensor-core conv launch (vtts_tc_split_plan), on the host alone.
    problems: list of dicts with Cin, Cout, k and optionally in_extra; cluster_cap: co-resident clusters of 2/4/8 CTAs at
    BN 64, then at BN 128 (6 ints).  Returns (BN, cluster size, [split of each problem])."""
    lib = load_library()
    ints = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    cin, cout, k = (ints([q[n] for q in problems]) for n in ("Cin", "Cout", "k"))
    extra, lens, cap = ints([q.get("in_extra", 0) for q in problems]), ints(lens), ints(cluster_cap)
    plan = np.zeros(6, np.int32)
    st = lib.vtts_tc_split_plan(len(problems), _ptr(cin), _ptr(cout), _ptr(k), _ptr(extra), lens.size, _ptr(lens), int(rmul),
                                int(lens.max() if max_len is None else max_len), int(bn), int(max_split), int(min_steps),
                                int(n_sm), _ptr(cap), _ptr(plan))
    if st != 0:
        raise VttsError(st, "vtts_tc_split_plan: invalid arguments")
    return int(plan[0]), int(plan[1]), [int(s) for s in plan[2:2 + len(problems)]]


def make_c_config(cfg, precision=0):
    c = VttsConfig()
    for k in ("n_vocab", "n_speakers", "gin_channels", "inter_channels", "hidden_channels", "filter_channels",
              "n_heads", "n_layers", "kernel_size", "window_size", "cond_layer_idx", "flow_kernel_size",
              "flow_dilation_rate", "flow_wn_layers", "flow_n_flows", "dp_filter_channels", "dp_kernel_size",
              "dp_n_flows", "dp_num_bins", "upsample_initial_channel", "subbands"):
        setattr(c, k, int(cfg[k]))
    c.spk_cond_encoder = int(bool(cfg["use_spk_conditioned_encoder"]) and cfg["gin_channels"] > 0 and cfg["n_speakers"] > 0)
    c.use_transformer_flows = int(bool(cfg["use_transformer_flows"]))
    c.dp_tail_bound = float(cfg["dp_tail_bound"])
    # 0: conv_post -> exp / pi*sin -> inverse STFT -> 63-tap filter bank (Multiband_ / Multistream_ / plain iSTFT_Generator differ only
    #    in the bank: fixed PQMF, learned, unit impulse; models.py:901-971, 974-1063, 1066-1169); 1: HiFi-GAN Generator
    c.decoder_type = 0 if cfg["decoder"] in ("mb_istft", "ms_istft", "istft") else 1
    c.resblock_type = 1 if str(cfg["resblock"]) == "1" else 2
    rk, rd = cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"]
    c.n_resblock_kernels = len(rk)
    c.n_resblock_dilations = len(rd[0])
    for j, k in enumerate(rk):
        c.resblock_kernel_sizes[j] = int(k)
        assert len(rd[j]) == len(rd[0])
        for d, v in enumerate(rd[j]):
            c.resblock_dilations[j][d] = int(v)
    c.n_upsamples = len(cfg["upsample_rates"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        c.upsample_rates[i] = int(u)
        c.upsample_kernel_sizes[i] = int(k)
    c.istft_n_fft = int(cfg["gen_istft_n_fft"])
    c.istft_hop = int(cfg["gen_istft_hop_size"])
    c.precision = int(precision)
    c.flow_n_heads = int(cfg.get("flow_n_heads", 2))
    d = _config.DEFAULT_CONFIG
    c.use_mel_posterior_encoder = int(bool(cfg.get("use_mel_posterior_encoder", d["use_mel_posterior_encoder"])))
    for k in ("filter_length", "hop_length", "win_length", "n_mel_channels"):
        setattr(c, k, int(cfg.get(k, d[k])))
    c.spec_channels = int(cfg.get("spec_channels", c.n_mel_channels if c.use_mel_posterior_encoder else c.filter_length // 2 + 1))
    c.mel_fmin = float(cfg.get("mel_fmin", 0.0) or 0.0)
    fmax = cfg.get("mel_fmax")
    c.mel_fmax = float(cfg.get("sampling_rate", 22050)) / 2 if fmax is None else float(fmax)
    c.model_family = MODEL_FAMILIES[cfg.get("model_family", "vits2")]
    cv = cfg.get("contentvec")
    if cv:
        for k in ("cv_layers", "cv_hidden", "cv_heads", "cv_ffn", "cv_conv_dim", "cv_pos_k", "cv_pos_groups"):
            setattr(c, k, int(cv[k]))
        c.cv_n_conv = len(cv["cv_conv_kernel"])
        for i, (k, s) in enumerate(zip(cv["cv_conv_kernel"], cv["cv_conv_stride"])):
            c.cv_conv_kernel[i], c.cv_conv_stride[i] = int(k), int(s)
        c.cv_ln_eps, c.cv_gn_eps = float(cv["cv_ln_eps"]), float(cv["cv_gn_eps"])
    return c


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Engine:
    """One engine = one GPU.  `blob` may be a numpy float32 array (host) or an (int device_ptr, n_floats) tuple."""

    def __init__(self, cfg, blob, manifest, device=0, precision=0):
        self.lib = load_library()
        self.cfg = cfg
        self.h = C.c_void_p()
        ccfg = make_c_config(cfg, precision)
        if isinstance(blob, tuple):
            ptr, n, on_dev = C.c_void_p(int(blob[0])), int(blob[1]), 1
        else:
            blob = np.ascontiguousarray(blob, dtype=np.float32)
            ptr, n, on_dev = _ptr(blob), blob.size, 0
        rc = self.lib.vtts_create(C.byref(ccfg), ptr, n, manifest.encode(), on_dev, int(device), C.byref(self.h))
        if rc != 0:
            msg = self.lib.vtts_last_error(self.h).decode() if self.h else "allocation failed"
            if self.h:
                self.lib.vtts_destroy(self.h)
                self.h = C.c_void_p()
            raise VttsError(rc, msg)
        self.hop = self.lib.vtts_hop(self.h)
        self.device = device
        import threading
        self._tls = threading.local()

    def close(self):
        if getattr(self, "h", None):
            self.lib.vtts_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise VttsError(rc, self.lib.vtts_last_error(self.h).decode())

    # ---- host-buffer path (what the reference-facing session calls)
    def durations(self, ids, lengths, sid, scales, noise_dp=None, seed=0, want_durations=False):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.ndim == 1:
            ids = ids[None, :]
        B, t_max = ids.shape
        lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
        sid = np.ascontiguousarray(sid, dtype=np.int64).reshape(B)
        scales = np.ascontiguousarray(scales, dtype=np.float32).reshape(3)
        if noise_dp is not None:
            noise_dp = np.ascontiguousarray(noise_dp, dtype=np.float32).reshape(B, 2, t_max)
        y_len = np.zeros(B, np.int64)
        dur = np.zeros((B, t_max), np.int32) if want_durations else None
        self._check(self.lib.vtts_durations(self.h, _ptr(ids), _ptr(lengths), _ptr(sid), B, t_max, _ptr(scales),
                                            _ptr(noise_dp), int(seed), _ptr(y_len), _ptr(dur)))
        self._B = B
        return (y_len, dur) if want_durations else y_len

    def synthesize(self, y_lengths, noise_z=None, want_alignment=False):
        B = self._B
        max_f = int(np.max(y_lengths))
        wav = np.zeros((B, max_f * self.hop), np.float32)
        z_ld = 0
        if noise_z is not None:
            noise_z = np.ascontiguousarray(noise_z, dtype=np.float32)
            assert noise_z.ndim == 3 and noise_z.shape[0] == B
            z_ld = noise_z.shape[2]
        idx = np.full((B, max_f), -1, np.int32) if want_alignment else None
        self._check(self.lib.vtts_synthesize(self.h, _ptr(noise_z), z_ld, _ptr(wav), wav.shape[1], _ptr(idx), max_f))
        return (wav, idx) if want_alignment else wav

    # Thread-safe variants of the two-phase pair: no per-Engine Python state (the batch size travels with the caller)
    def lib_durations_threadsafe(self, ids, lengths, sid, scales, noise_dp=None, seed=0):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        B, t_max = ids.shape
        lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
        sid = np.ascontiguousarray(sid, dtype=np.int64).reshape(B)
        scales = np.ascontiguousarray(scales, dtype=np.float32).reshape(3)
        if noise_dp is not None:
            noise_dp = np.ascontiguousarray(noise_dp, dtype=np.float32).reshape(B, 2, t_max)
        y_len = np.zeros(B, np.int64)
        self._check(self.lib.vtts_durations(self.h, _ptr(ids), _ptr(lengths), _ptr(sid), B, t_max, _ptr(scales), _ptr(noise_dp), int(seed),
                                            _ptr(y_len), None))
        return y_len

    def lib_synthesize_threadsafe(self, B, y_lengths, noise_z=None):
        max_f = int(np.max(y_lengths))
        wav = np.zeros((B, max_f * self.hop), np.float32)
        z_ld = 0
        if noise_z is not None:
            noise_z = np.ascontiguousarray(noise_z, dtype=np.float32)
            z_ld = noise_z.shape[2]
        self._check(self.lib.vtts_synthesize(self.h, _ptr(noise_z), z_ld, _ptr(wav), wav.shape[1], None, 0))
        return wav

    def infer(self, ids, lengths, sid, scales, noise_dp=None, noise_z=None, seed=0, frames_hint=None):
        """Both phases.  noise_z may be a callable(max_frames)->[B,C,max_frames] (T_y is data dependent).
        With `frames_hint` (an upper bound on max(y_lengths), e.g. from a previous call) and array/None noise, the
        fused C entry point vtts_infer is used: one ctypes call, no Python between the two phases."""
        if frames_hint is not None and not callable(noise_z):
            ids = np.ascontiguousarray(ids, dtype=np.int64)
            if ids.ndim == 1:
                ids = ids[None, :]
            B, t_max = ids.shape
            lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
            sid = np.ascontiguousarray(sid, dtype=np.int64).reshape(B)
            scales = np.ascontiguousarray(scales, dtype=np.float32).reshape(3)
            if noise_dp is not None:
                noise_dp = np.ascontiguousarray(noise_dp, dtype=np.float32).reshape(B, 2, t_max)
            z_ld = 0
            if noise_z is not None:
                noise_z = np.ascontiguousarray(noise_z, dtype=np.float32)
                z_ld = noise_z.shape[2]
            y_len = np.zeros(B, np.int64)
            # capacity-sized scratch rows, reused by this thread's calls (a fresh 1 MB numpy buffer per call costs mmap / page
            # faults / munmap -- 0.1-0.3 ms of a 1.7 ms call); the engine writes y_len*hop samples per row
            tl = self._tls
            need = int(frames_hint) * self.hop
            wav = getattr(tl, "wav", None)
            if wav is None or wav.shape[0] < B or wav.shape[1] < need:
                wav = np.empty((B, need), np.float32)
                tl.wav = wav
            wav = wav[:B]
            rc = self.lib.vtts_infer(self.h, _ptr(ids), _ptr(lengths), _ptr(sid), B, t_max, _ptr(scales), _ptr(noise_dp),
                                     _ptr(noise_z), z_ld, int(seed), _ptr(y_len), _ptr(wav), wav.shape[1], None, 0)
            self._B = B
            if rc == -4:            # capacity: durations are kept, finish with exact buffers
                if noise_z is not None and z_ld < int(y_len.max()):
                    self._check(rc)
                return self.synthesize(y_len, noise_z), y_len
            self._check(rc)
            n = int(y_len.max()) * self.hop
            out = np.zeros((B, n), np.float32)                           # contiguous result sized to max(y_len); rows are zero beyond their length
            for b in range(B):
                m = int(y_len[b]) * self.hop
                out[b, :m] = wav[b, :m]
            return out, y_len
        y_len = self.durations(ids, lengths, sid, scales, noise_dp, seed)
        if callable(noise_z):
            noise_z = noise_z(int(y_len.max()))
        wav = self.synthesize(y_len, noise_z)
        return wav, y_len

    def infer_dev(self, d_ids, lengths, d_sid, B, t_max, scales, d_wav, wav_ld, d_noise_dp=0, d_noise_z=0, z_ld=0, seed=0):
        lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
        scales = np.ascontiguousarray(scales, dtype=np.float32).reshape(3)
        y_len = np.zeros(B, np.int64)
        self._check(self.lib.vtts_infer_dev(self.h, C.c_void_p(d_ids), _ptr(lengths), C.c_void_p(d_sid), B, t_max, _ptr(scales),
                                            C.c_void_p(d_noise_dp) if d_noise_dp else None,
                                            C.c_void_p(d_noise_z) if d_noise_z else None, z_ld, int(seed), _ptr(y_len),
                                            C.c_void_p(d_wav), wav_ld))
        self._B = B
        return y_len

    def reserve(self, max_tokens=256, max_frames=1024, batch=1):
        """Sizes the engine's workspace (device buffers, plane pools, pinned staging) once for calls of up to `batch`
        utterances x `max_tokens` phonemes x `max_frames` frames, by synthesising one synthetic request of that size.
        Any LATER growth of the workspace moves buffers and therefore invalidates every captured CUDA graph (each length
        bucket then pays its capture again, ~15 ms); a service calls this once at start-up, like the reference server
        warms its ONNX session.  Returns the frame count that was reached."""
        T, B = int(max_tokens), int(batch)
        nv = int(self.cfg["n_vocab"])
        ids = (np.arange(B * T, dtype=np.int64).reshape(B, T) * 7 + 1) % nv
        lens, sid = [T] * B, [0] * B
        e1 = np.zeros((B, 2, T), np.float32)
        ls, F, yl = 1.0, 0, None
        for _ in range(5):
            yl = self.durations(ids, lens, sid, (0.667, ls, 0.8), e1)
            F = int(yl.max())
            if F >= max_frames:
                break
            ls *= max_frames / max(F, 1) * 1.05
        ez = np.zeros((B, int(self.cfg["inter_channels"]), F), np.float32)
        self.synthesize(yl, ez)
        self.infer(ids, lens, sid, (0.667, ls, 0.8), None, None, seed=1, frames_hint=F + 64)
        return F

    # ---- voice conversion (SynthesizerTrn.voice_conversion, models.py:1710-1718)
    def _convert(self, from_wav, x, lengths, ld, sid_src, sid_tgt, noise_scale, noise, seed):
        B = x.shape[0]
        lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
        src = np.ascontiguousarray(np.broadcast_to(np.asarray(sid_src, np.int64), (B,)))
        tgt = np.ascontiguousarray(np.broadcast_to(np.asarray(sid_tgt, np.int64), (B,)))
        q_ld = 0
        if noise is not None:
            noise = np.ascontiguousarray(noise, dtype=np.float32)
            if noise.ndim != 3 or noise.shape[0] != B or noise.shape[1] != int(self.cfg["inter_channels"]):
                raise ValueError("noise must be float32 [B, inter_channels, >= frames]")
            q_ld = noise.shape[2]
        frames = np.zeros(B, np.int64)
        cap = self.convert_frames(lengths) if from_wav else lengths
        fn = self.lib.vtts_convert if from_wav else self.lib.vtts_convert_spec
        out = np.zeros((B, max(1, int(np.max(cap))) * self.hop), np.float32)
        self._check(fn(self.h, _ptr(x), _ptr(lengths), B, ld, _ptr(src), _ptr(tgt), float(noise_scale), _ptr(noise), q_ld,
                       int(seed), _ptr(out), out.shape[1], _ptr(frames)))
        return out[:, : int(frames.max()) * self.hop], frames

    def convert_frames(self, wav_lengths):
        """Frames of the spectrogram of clips of `wav_lengths` samples (center=False after reflect padding by
        (filter_length - hop_length) / 2 on both sides, mel_processing.py:67-71): len // 256 for the reference configuration."""
        c = self.cfg
        n_fft, hop = int(c.get("filter_length", 1024)), int(c.get("hop_length", 256))
        pad = (n_fft - hop) // 2
        L = np.asarray(wav_lengths, np.int64)
        return np.maximum((L + 2 * pad - n_fft) // hop + 1, 0)

    def convert(self, wav, sid_src, sid_tgt, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Re-voices clips of speaker `sid_src` as speaker `sid_tgt` (vtts_convert).  wav: float32 [B, L] (or [L]) in [-1, 1],
        `lengths` the valid samples per row (default: all).  Returns (float32 [B, hop * max(frames)], frames [B]); row b holds
        hop * frames[b] samples.  noise: optional eps [B, inter_channels, >= frames] of the posterior sample."""
        wav = np.ascontiguousarray(wav, dtype=np.float32)
        if wav.ndim == 1:
            wav = wav[None, :]
        lengths = np.full(wav.shape[0], wav.shape[1], np.int64) if lengths is None else lengths
        return self._convert(True, wav, lengths, wav.shape[1], sid_src, sid_tgt, noise_scale, noise, seed)

    def convert_spec(self, spec, sid_src, sid_tgt, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Same from the posterior encoder's input features (the reference's `y`): float32 [B, spec_channels, T]."""
        spec = np.ascontiguousarray(spec, dtype=np.float32)
        if spec.ndim == 2:
            spec = spec[None]
        lengths = np.full(spec.shape[0], spec.shape[2], np.int64) if lengths is None else lengths
        return self._convert(False, spec, lengths, spec.shape[2], sid_src, sid_tgt, noise_scale, noise, seed)

    def reserve_convert(self, max_frames=1024, batch=1):
        """Workspace reservation for conversions of up to `batch` clips x `max_frames` frames (see reserve): one conversion
        from a waveform and one from a spectrogram of that size, so later calls within these bounds move no buffer."""
        hop = int(self.cfg.get("hop_length", 256))
        B, F = int(batch), int(max_frames)
        wav = np.zeros((B, F * hop), np.float32)
        n = int(self.cfg["n_speakers"])
        self.convert(wav, 0, min(1, n - 1), noise_scale=0.0)
        spec = np.zeros((B, int(self.cfg.get("spec_channels", 80)), F), np.float32)
        self.convert_spec(spec, 0, min(1, n - 1), noise_scale=0.0)
        return F

    # ---- QuickVC speaker embedding (SpeakerEncoder.embed_utterance, vc/models.py:728-767)
    def speaker_embedding(self, wav, lengths=None):
        """The QuickVC target embedding g of each clip (vtts_speaker_embedding): wav float32 [B, L] (or [L]) in [-1, 1] at the
        model's sampling rate, `lengths` the valid samples per row (default: all).  Returns float32 [B, gin_channels]."""
        wav = np.ascontiguousarray(wav, dtype=np.float32)
        if wav.ndim == 1:
            wav = wav[None, :]
        B = wav.shape[0]
        lengths = np.ascontiguousarray(np.full(B, wav.shape[1]) if lengths is None else lengths, dtype=np.int64).reshape(B)
        g = np.zeros((B, int(self.cfg["gin_channels"])), np.float32)
        self._check(self.lib.vtts_speaker_embedding(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(g)))
        return g

    def speaker_embedding_mel(self, mel, lengths=None):
        """Same from log-mel rows (mel_spectrogram_torch's output): float32 [B, n_mel_channels, T] (or [n_mel_channels, T])."""
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        if mel.ndim == 2:
            mel = mel[None]
        B = mel.shape[0]
        lengths = np.ascontiguousarray(np.full(B, mel.shape[2]) if lengths is None else lengths, dtype=np.int64).reshape(B)
        g = np.zeros((B, int(self.cfg["gin_channels"])), np.float32)
        self._check(self.lib.vtts_speaker_embedding_mel(self.h, _ptr(mel), _ptr(lengths), B, mel.shape[2], _ptr(g)))
        return g

    def reserve_quickvc(self, max_frames=1024, batch=1):
        """Workspace reservation for embeddings of up to `batch` clips x `max_frames` mel frames: one call of that size, so
        later calls within these bounds move no buffer."""
        hop = int(self.cfg["hop_length"])
        self.speaker_embedding(np.zeros((int(batch), int(max_frames) * hop), np.float32))
        return int(max_frames)

    # ---- QuickVC conversion (SynthesizerTrn.infer, vc/models.py:862-872)
    def quickvc_convert(self, units, g, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Content units -> waveforms in the voice of g (vtts_quickvc_convert).  units: one clip [T, 768] (ContentVec's
        last_hidden_state, vc/encode.py's .npy), a batch [B, T, 768] with `lengths`, or a list of ragged [T_b, 768] arrays;
        g: [gin_channels] (one target for every clip) or [B, gin_channels] (speaker_embedding's output).  noise: None
        (Philox from `seed`) or [B, inter_channels, >= max T] standing in for torch.randn_like.  Returns (wav float32
        [B, hop * max T], zeros past each clip's end; frames int64 [B])."""
        if isinstance(units, (list, tuple)):
            clips = [np.asarray(u, np.float32) for u in units]
            lengths = np.array([u.shape[0] for u in clips], np.int64)
            batch = np.zeros((len(clips), int(lengths.max()), 768), np.float32)
            for b, u in enumerate(clips):
                batch[b, :u.shape[0]] = u
            units = batch
        units = np.ascontiguousarray(units, dtype=np.float32)
        if units.ndim == 2:
            units = units[None]
        B, T = units.shape[0], units.shape[1]
        lengths = np.ascontiguousarray(np.full(B, T) if lengths is None else lengths, dtype=np.int64).reshape(B)
        G = int(self.cfg["gin_channels"])
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(g, np.float32).reshape(-1, G), (B, G)), dtype=np.float32)
        ld = 0
        if noise is not None:
            noise = np.ascontiguousarray(noise, dtype=np.float32)
            ld = noise.shape[2]
        wav = np.zeros((B, max(1, int(lengths.max())) * self.hop), np.float32)
        frames = np.zeros(B, np.int64)
        self._check(self.lib.vtts_quickvc_convert(self.h, _ptr(units), _ptr(lengths), B, T, _ptr(g), float(noise_scale), _ptr(noise),
                                                  ld, int(seed), _ptr(wav), wav.shape[1], _ptr(frames)))
        return wav, frames

    def reserve_quickvc_convert(self, max_frames=1024, batch=1):
        """Workspace reservation for conversions of up to `batch` clips x `max_frames` content frames: one call of that size,
        so later calls within these bounds move no buffer."""
        self.quickvc_convert(np.zeros((int(batch), int(max_frames), 768), np.float32), np.zeros(int(self.cfg["gin_channels"]), np.float32),
                             noise_scale=0.0)
        return int(max_frames)

    # ---- ContentVec (vc/contentvec.py) and conversion from source waveforms; cfg["contentvec"] is its shape
    @staticmethod
    def _clips(wav, lengths):
        if isinstance(wav, (list, tuple)):
            clips = [np.asarray(w, np.float32).reshape(-1) for w in wav]
            lengths = np.array([w.size for w in clips], np.int64)
            batch = np.zeros((len(clips), int(lengths.max())), np.float32)
            for b, w in enumerate(clips):
                batch[b, :w.size] = w
            wav = batch
        wav = np.ascontiguousarray(wav, dtype=np.float32)
        if wav.ndim == 1:
            wav = wav[None]
        B = wav.shape[0]
        lengths = np.ascontiguousarray(np.full(B, wav.shape[1]) if lengths is None else lengths, dtype=np.int64).reshape(B)
        return wav, lengths

    def content_units(self, wav, lengths=None):
        """ContentVec units of 16 kHz sources (vtts_content_units): wav [L], [B, L] with `lengths`, or a list of ragged clips.
        Returns (units float32 [B, max T, hidden], zeros past each clip's end; frames int64 [B])."""
        wav, lengths = self._clips(wav, lengths)
        B = wav.shape[0]
        T = max(1, max(_config.contentvec_frames(int(n), self.cfg.get("contentvec")) for n in lengths))
        units = np.zeros((B, T, int((self.cfg.get("contentvec") or _config.contentvec_config())["cv_hidden"])), np.float32)
        frames = np.zeros(B, np.int64)
        self._check(self.lib.vtts_content_units(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(units), T, _ptr(frames)))
        return units, frames

    def quickvc_convert_wav(self, wav, g, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Source waveforms -> waveforms in the voice of g in one call (vtts_quickvc_convert_wav): content_units, then
        quickvc_convert, without the units leaving the GPU.  Arguments as those two.  Returns (wav [B, hop * max T], frames)."""
        wav, lengths = self._clips(wav, lengths)
        B = wav.shape[0]
        T = max(1, max(_config.contentvec_frames(int(n), self.cfg.get("contentvec")) for n in lengths))
        G = int(self.cfg["gin_channels"])
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(g, np.float32).reshape(-1, G), (B, G)), dtype=np.float32)
        ld = 0
        if noise is not None:
            noise = np.ascontiguousarray(noise, dtype=np.float32)
            ld = noise.shape[2]
        out = np.zeros((B, T * self.hop), np.float32)
        frames = np.zeros(B, np.int64)
        self._check(self.lib.vtts_quickvc_convert_wav(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(g), float(noise_scale),
                                                      _ptr(noise), ld, int(seed), _ptr(out), out.shape[1], _ptr(frames)))
        return out, frames

    def reserve_contentvec(self, max_samples=160000, batch=1):
        """Workspace reservation for ContentVec calls of up to `batch` clips x `max_samples` samples (layer 0's rows at 3200 Hz
        are the large buffers): one call of that size, so later calls within these bounds move no buffer."""
        self.content_units(np.zeros((int(batch), int(max_samples)), np.float32))
        return int(max_samples)

    # ---- forced alignment (the alignment of SynthesizerTrn.forward, models.py:1632-1660)
    def _align(self, from_wav, ids, lengths, sid, x, x_lengths, noise_scale, noise, seed):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.ndim == 1:
            ids = ids[None, :]
        B, t_max = ids.shape
        if x.shape[0] != B:
            raise ValueError("ids and recordings must have the same batch size")
        lengths = np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int64), (B,)))
        sid = np.ascontiguousarray(np.broadcast_to(np.asarray(0 if sid is None else sid, np.int64), (B,)))
        ld = x.shape[-1]
        x_lengths = np.full(B, ld, np.int64) if x_lengths is None else \
            np.ascontiguousarray(np.broadcast_to(np.asarray(x_lengths, np.int64), (B,)))
        q_ld = 0
        if noise is not None:
            noise = np.ascontiguousarray(noise, dtype=np.float32)
            if noise.ndim != 3 or noise.shape[0] != B or noise.shape[1] != int(self.cfg["inter_channels"]):
                raise ValueError("noise must be float32 [B, inter_channels, >= frames]")
            q_ld = noise.shape[2]
        cap = self.convert_frames(x_lengths) if from_wav else x_lengths
        max_f = max(1, int(np.max(cap)))
        dur = np.zeros((B, t_max), np.int32)
        tof = np.full((B, max_f), -1, np.int32)
        score = np.zeros(B, np.float32)
        frames = np.zeros(B, np.int64)
        fn = self.lib.vtts_align if from_wav else self.lib.vtts_align_spec
        self._check(fn(self.h, _ptr(ids), _ptr(lengths), t_max, _ptr(sid), _ptr(x), _ptr(x_lengths), B, ld, float(noise_scale),
                       _ptr(noise), q_ld, int(seed), _ptr(dur), _ptr(tof), max_f, _ptr(score), _ptr(frames)))
        return dur, frames, tof[:, : int(frames.max())], score

    def align(self, ids, lengths, sid, wav, wav_lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Forced alignment (vtts_align): phoneme ids int64 [B, t_max] (`lengths` valid per row) of speaker `sid` against
        recordings float32 [B, L] in [-1, 1] (`wav_lengths` valid samples per row, default all).  Returns (durations int32
        [B, t_max] -- frames per token, 0 past lengths[b]; frames int64 [B]; token_of_frame int32 [B, max frames], -1 past
        frames[b]; score float32 [B], the best path's log-likelihood).  noise: optional eps [B, inter_channels, >= frames] of
        the posterior sample, else Philox(seed); noise_scale 1 is the reference's forward, 0 the posterior mean."""
        wav = np.ascontiguousarray(wav, dtype=np.float32)
        if wav.ndim == 1:
            wav = wav[None, :]
        return self._align(True, ids, lengths, sid, wav, wav_lengths, noise_scale, noise, seed)

    def align_spec(self, ids, lengths, sid, spec, spec_lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Same from the posterior encoder's input features (the reference's `y`): float32 [B, spec_channels, T]."""
        spec = np.ascontiguousarray(spec, dtype=np.float32)
        if spec.ndim == 2:
            spec = spec[None]
        return self._align(False, ids, lengths, sid, spec, spec_lengths, noise_scale, noise, seed)

    def reserve_align(self, max_tokens=256, max_frames=1024, batch=1):
        """Workspace reservation for alignments of up to `batch` utterances x `max_tokens` tokens x `max_frames` frames (see
        reserve): one alignment from a waveform and one from a spectrogram of that size, so that later calls within these
        bounds move no buffer (a move invalidates every captured CUDA graph)."""
        hop = int(self.cfg.get("hop_length", 256))
        B, T, F = int(batch), int(max_tokens), int(max_frames)
        if not 1 <= T <= F:
            raise ValueError("reserve_align needs 1 <= max_tokens <= max_frames")
        ids = (np.arange(B * T, dtype=np.int64).reshape(B, T) * 7 + 1) % int(self.cfg["n_vocab"])
        self.align(ids, T, 0, np.zeros((B, F * hop), np.float32), noise_scale=0.0)
        spec = np.zeros((B, int(self.cfg.get("spec_channels", 80)), F), np.float32)
        self.align_spec(ids, T, 0, spec, noise_scale=0.0)
        return F

    # ---- streaming (one utterance): flow once, then vocode chunk by chunk
    def synthesize_stream(self, ids, sid, scales, chunk_frames=64, noise_dp=None, noise_z=None, seed=0):
        """Generator of float32 chunks; concatenated they equal `infer(...)` of the same inputs."""
        ids = np.ascontiguousarray(ids, dtype=np.int64).reshape(1, -1)
        y_len = self.durations(ids, [ids.shape[1]], [sid], scales, noise_dp, seed)
        T = int(y_len[0])
        z_ld = 0
        if noise_z is not None:
            noise_z = np.ascontiguousarray(noise_z, dtype=np.float32)
            z_ld = noise_z.shape[2]
        self._check(self.lib.vtts_flow(self.h, _ptr(noise_z), z_ld))
        for f0 in range(0, T, chunk_frames):
            f1 = min(T, f0 + chunk_frames)
            out = np.zeros((f1 - f0) * self.hop, np.float32)
            self._check(self.lib.vtts_decode_chunk(self.h, f0, f1, _ptr(out), out.size))
            yield out

    # ---- device-buffer path (raw pointers, e.g. torch tensors' data_ptr())
    def durations_dev(self, d_ids, lengths, d_sid, B, t_max, scales, d_noise_dp=0, seed=0):
        lengths = np.ascontiguousarray(lengths, dtype=np.int64).reshape(B)
        scales = np.ascontiguousarray(scales, dtype=np.float32).reshape(3)
        y_len = np.zeros(B, np.int64)
        self._check(self.lib.vtts_durations_dev(self.h, C.c_void_p(d_ids), _ptr(lengths), C.c_void_p(d_sid), B, t_max,
                                                _ptr(scales), C.c_void_p(d_noise_dp) if d_noise_dp else None,
                                                int(seed), _ptr(y_len)))
        self._B = B
        return y_len

    def synthesize_dev(self, d_wav, wav_ld, d_noise_z=0, z_ld=0):
        self._check(self.lib.vtts_synthesize_dev(self.h, C.c_void_p(d_noise_z) if d_noise_z else None, z_ld,
                                                 C.c_void_p(d_wav), wav_ld))

    def stage_timings(self):
        ms = np.zeros(8, np.float32)
        self.lib.vtts_stage_timings(self.h, _ptr(ms), 8)
        return dict(encoder=float(ms[0]), duration=float(ms[1]), flow=float(ms[2]), decoder=float(ms[3]),
                    h2d=float(ms[4]), d2h=float(ms[5]))

    def kernel_launches(self):
        return int(self.lib.vtts_kernel_launches(self.h))

    def stream(self):
        return int(self.lib.vtts_stream(self.h) or 0)

    def microbench(self, what, iters=50):
        ms = float(self.lib.vtts_microbench(self.h, what.encode(), int(iters)))
        if ms < 0:
            raise VttsError(int(ms), self.lib.vtts_last_error(self.h).decode())
        return ms

    def timeline(self, mode):
        """mode 1: arm, 0: disarm, 2: read -> array [n,2] of (source line, globaltimer ns)."""
        if mode != 2:
            self._check(self.lib.vtts_timeline(self.h, int(mode), None, 0, None))
            return None
        out = np.zeros((4000, 2), np.uint64)
        n = C.c_size_t(0)
        self._check(self.lib.vtts_timeline(self.h, 2, _ptr(out), 4000, C.byref(n)))
        return out[: n.value].copy()

    def set_graphs(self, enable):
        self._check(self.lib.vtts_set_graphs(self.h, int(bool(enable))))

    def graph_replays(self):
        return int(self.lib.vtts_graph_replays(self.h))

    def speculation_stats(self):
        """(hits, misses) of the speculative second phase of single-utterance infer calls."""
        a, b = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.vtts_speculation_stats(self.h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def host_timings(self):
        """Host-side microseconds of the last single-utterance infer call (see vtts_host_timings)."""
        a = (C.c_double * 8)()
        self._check(self.lib.vtts_host_timings(self.h, a, 8))
        return [float(v) for v in a]

    def profile(self, enable):
        self._check(self.lib.vtts_profile(self.h, int(bool(enable))))

    def profile_read(self):
        ms, n, fl = C.c_double(0), C.c_uint64(0), C.c_double(0)
        self._check(self.lib.vtts_profile_read(self.h, C.byref(ms), C.byref(n), C.byref(fl)))
        out = dict(conv_ms=ms.value, conv_launches=int(n.value), conv_flops=fl.value)
        self._check(self.lib.vtts_profile_read_tc(self.h, C.byref(ms), C.byref(n), C.byref(fl)))
        out.update(tc_ms=ms.value, tc_launches=int(n.value), tc_flops=fl.value)
        return out

    def debug_attention(self, layer, qkv, lens=None, kernel="auto", launch_lens=None, out=True, planes=None, iters=0):
        """One attention launch of `layer` ("enc.<i>" / "flow.<f>.tr") through the engine's launch code (vtts_debug_attention).
        qkv: float32 [rows, 3H], every row of the packed batch (utterance b at row cr.offsets(lens)[b], 8 rows between
        utterances).  lens: lengths (default: one utterance of all rows); launch_lens: lengths >= lens the launch is sized for.
        kernel: "auto", "tc", "split", "r1", "r4" or "ffma" (the engine's choice among the FFMA kernels).
        out: True (zero-filled), an initial float32 [rows, H] (rows outside the utterances keep it) or False for none.
        planes: None, 2 / 3 (zero-filled) or an initial uint16 [p, rows * H].
        Returns (out [rows, H] or None, planes or None, launch report dict, ms or None)."""
        qkv = np.ascontiguousarray(qkv, dtype=np.float32)
        rows, H = qkv.shape[0], qkv.shape[1] // 3
        lens = np.ascontiguousarray([rows] if lens is None else lens, dtype=np.int32)
        ll = None if launch_lens is None else np.ascontiguousarray(launch_lens, dtype=np.int32)
        if out is True:
            out = np.zeros((rows, H), np.float32)
        elif out is not None and out is not False:
            out = np.ascontiguousarray(out, dtype=np.float32).reshape(rows, H).copy()
        else:
            out = None
        if isinstance(planes, int):
            planes = np.zeros((planes, rows * H), np.uint16)
        elif planes is not None:
            planes = np.ascontiguousarray(planes, dtype=np.uint16).copy()
        if kernel not in ATTN_KERNELS:
            raise ValueError("unknown attention kernel %r" % (kernel,))
        ms = C.c_float(0.0)
        rep = AttnReport()
        self._check(self.lib.vtts_debug_attention(
            self.h, layer.encode(), lens.size, _ptr(lens), _ptr(ll), _ptr(qkv), rows, ATTN_KERNELS[kernel], _ptr(out),
            _ptr(planes), 0 if planes is None else planes.shape[0], int(iters), C.byref(ms), C.byref(rep)))
        return out, planes, rep.as_dict(), (float(ms.value) if iters > 0 else None)

    def debug_conv(self, use_tc, lens, rmul, problems, x, y=None, res=None, planes=None, overrides=None):
        """One grouped launch of the tensor-core (use_tc) or FFMA conv kernel on host tensors (vtts_debug_conv).
        problems: list of dicts with the vtts_conv_problem fields; array fields (w_hi / w_mid / w_lo uint16 [k][Cout][Cin],
        w float32 [k][Cin][ldw], bias, cond) are numpy arrays.  x: tensor cores uint16 [np][rows][Cin] planes, FFMA float32
        (any shape, flat layout).  y / res: float32 buffers (y is in/out), planes: uint16 [2 or 3][n] (in/out).
        overrides: dict of CONV_OVERRIDES names.  Returns (y, planes, launch report dict)."""
        keep = []

        def arr(a, dt):
            a = np.ascontiguousarray(a, dtype=dt)
            keep.append(a)
            return a

        ps = (ConvProblem * len(problems))()
        for i, q in enumerate(problems):
            p = ps[i]
            p.out_mul, p.alpha, p.pl_slope = 1, 1.0, 1.0
            for key, v in q.items():
                if key in ("w_hi", "w_mid", "w_lo"):
                    setattr(p, key, None if v is None else arr(v, np.uint16).ctypes.data)
                elif key in ("w", "bias", "cond"):
                    setattr(p, key, None if v is None else arr(v, np.float32).ctypes.data)
                else:
                    setattr(p, key, v)
        if use_tc:
            x = arr(x, np.uint16)
            x_planes, x_n = x.shape[0], x.shape[1]
        else:
            x = arr(x, np.float32)
            x_planes, x_n = 0, x.size
        y = None if y is None else np.ascontiguousarray(y, dtype=np.float32).copy()
        res = None if res is None else arr(res, np.float32)
        planes = None if planes is None else np.ascontiguousarray(planes, dtype=np.uint16).copy()
        ov = None
        if overrides:
            ov = ConvOverrides(*[CONV_KEEP] * len(CONV_OVERRIDES))
            for key, v in overrides.items():
                if key not in CONV_OVERRIDES:
                    raise ValueError("unknown conv launch override %r" % key)
                setattr(ov, key, int(v))
        rep = ConvReport()
        lens = arr(lens, np.int32)
        self._check(self.lib.vtts_debug_conv(
            self.h, int(bool(use_tc)), lens.size, _ptr(lens), int(rmul), len(problems), ps, _ptr(x), x_n, x_planes,
            _ptr(y), 0 if y is None else y.size, _ptr(res), 0 if res is None else res.size,
            _ptr(planes), 0 if planes is None else planes.shape[1], 0 if planes is None else planes.shape[0],
            None if ov is None else C.byref(ov), C.byref(rep)))
        return y, planes, rep.as_dict()

    def conv_log(self, mode):
        """Launch-shape log of the dense conv launches (vtts_debug_conv_log): 1 clears and starts it, 0 stops it, 2 returns the
        list of report dicts recorded since it was started."""
        if mode != 2:
            self._check(self.lib.vtts_debug_conv_log(self.h, int(mode), None, 0, None))
            return None
        out = (ConvReport * 65536)()
        n = C.c_int(0)
        self._check(self.lib.vtts_debug_conv_log(self.h, 2, out, len(out), C.byref(n)))
        return [out[i].as_dict() for i in range(n.value)]

    def debug_flags(self, flags):
        self._check(self.lib.vtts_debug_flags(self.h, int(flags)))

    def debug_read(self, name, max_floats=1 << 26):
        out = np.zeros(max_floats, np.float32)
        n = C.c_size_t(0)
        self._check(self.lib.vtts_debug_read(self.h, name.encode(), _ptr(out), max_floats, C.byref(n)))
        return out[: n.value].copy()
