"""ctypes binding of libvtts.so (include/vtts.h).  No CPU fallback: importing works without a GPU
(the library only needs libcudart), creating an Engine requires a CUDA device."""
import ctypes as C
import math
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
        ("st_noise", C.c_int32), ("st_cond", C.c_int32), ("st_hidden", C.c_int32), ("st_filter", C.c_int32),
        ("st_layers", C.c_int32), ("st_heads", C.c_int32), ("st_kernel", C.c_int32), ("st_spk_dim", C.c_int32),
        ("st_n_spks", C.c_int32),
        ("st_n_vocab", C.c_int32), ("st_streams", C.c_int32), ("st_emb_dim", C.c_int32), ("st_punc_dim", C.c_int32),
        ("st_bert_dim", C.c_int32), ("st_bert_proj", C.c_int32), ("st_enc_hidden", C.c_int32), ("st_enc_filter", C.c_int32),
        ("st_enc_layers", C.c_int32), ("st_enc_heads", C.c_int32), ("st_enc_kernel", C.c_int32), ("st_dur_channels", C.c_int32),
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
           "vtts_quickvc_convert_wav", "vtts_debug_live_bytes", "vtts_resample", "vtts_cfm_decode", "vtts_stabletts_synthesise",
           "vtts_hifigan_vocode", "vtts_stabletts_synthesise_wav", "vtts_bert_features", "vtts_stabletts_synthesise_pieces_wav",
           "vtts_debug_dds", "vtts_debug_spline", "vtts_debug_durations", "vtts_debug_stt_durations", "vtts_t2s_decode",
           "vtts_debug_t2s_sample", "vtts_debug_front_end", "vtts_debug_istft", "vtts_debug_mrf_mean",
           "vtts_sovits_semantic", "vtts_sovits_latent"]

MODEL_FAMILIES = {"vits2": 0, "quickvc": 1, "stabletts": 2, "t2s": 3, "sovits": 4}    # vtts_config.model_family
CFM_MAX_STEPS = 64       # VTTS_CFM_MAX_STEPS

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
    lib.vtts_debug_dds.argtypes = [vp, C.c_char_p, i32, vp, C.c_size_t, vp, vp, vp, vp]
    lib.vtts_debug_dds.restype = i32
    lib.vtts_debug_spline.argtypes = [vp, i32, vp, C.c_size_t, vp, i32, vp]
    lib.vtts_debug_spline.restype = i32
    lib.vtts_debug_durations.argtypes = [vp, i32, vp, C.c_size_t, vp, C.c_float, i32, vp, vp, C.c_int64, C.c_float, vp, vp, vp, vp,
                                         vp, vp, C.c_size_t, vp, vp]
    lib.vtts_debug_durations.restype = i32
    lib.vtts_debug_stt_durations.argtypes = [vp, i32, vp, C.c_size_t, vp, vp, C.c_float, vp, vp, i32, vp, vp, vp, vp, C.c_size_t,
                                             vp, vp, vp, vp]
    lib.vtts_debug_stt_durations.restype = i32
    lib.vtts_debug_front_end.argtypes = [vp, i32, vp, vp, i32, C.c_int64, vp, C.c_size_t, vp, vp]
    lib.vtts_debug_front_end.restype = i32
    lib.vtts_debug_istft.argtypes = [vp, i32, vp, i32, C.c_size_t, vp, C.c_size_t, vp]
    lib.vtts_debug_istft.restype = i32
    lib.vtts_debug_mrf_mean.argtypes = [vp, i32, i32, vp, i32, i32, i32, C.c_size_t, vp, i32, vp, C.c_size_t, vp, vp]
    lib.vtts_debug_mrf_mean.restype = i32
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
    lib.vtts_debug_live_bytes.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.vtts_debug_live_bytes.restype = i32
    lib.vtts_resample.argtypes = [vp, vp, vp, i32, C.c_int64, i32, i32, C.c_float, vp, C.c_int64, vp, vp]
    lib.vtts_resample.restype = i32
    lib.vtts_cfm_decode.argtypes = [vp, vp, vp, i32, C.c_int64, vp, vp, i32, C.c_float, C.c_float, vp, C.c_int64, C.c_uint64, vp,
                                    C.c_int64, i32]
    lib.vtts_cfm_decode.restype = i32
    lib.vtts_stabletts_synthesise.argtypes = [vp, vp, vp, i32, C.c_int64, vp, vp, vp, i32, C.c_float, C.c_float, C.c_float, vp, C.c_int64,
                                              C.c_uint64, vp, C.c_int64, vp, vp, vp, i32]
    lib.vtts_stabletts_synthesise.restype = i32
    lib.vtts_stabletts_synthesise_wav.argtypes = lib.vtts_stabletts_synthesise.argtypes + [vp, C.c_int64, vp]
    lib.vtts_stabletts_synthesise_wav.restype = i32
    lib.vtts_hifigan_vocode.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_int64, vp]
    lib.vtts_hifigan_vocode.restype = i32
    lib.vtts_bert_features.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_int64]
    lib.vtts_bert_features.restype = i32
    st = lib.vtts_stabletts_synthesise_wav.argtypes
    lib.vtts_stabletts_synthesise_pieces_wav.argtypes = st[:5] + [vp, vp, C.c_int64, vp] + st[6:]
    lib.vtts_stabletts_synthesise_pieces_wav.restype = i32
    lib.vtts_t2s_decode.argtypes = [vp, vp, vp, i32, C.c_int64, vp, vp, vp, C.c_int64, i32, C.c_float, C.c_float, C.c_float, i32, i32,
                                    vp, vp, C.c_int64, vp, C.c_int64, vp, vp, vp, C.c_int64]
    lib.vtts_t2s_decode.restype = i32
    lib.vtts_debug_t2s_sample.argtypes = [vp, i32, vp, vp, vp, i32, i32, C.c_float, C.c_float, C.c_float, i32, i32, vp, vp, i32, vp, vp,
                                          vp, i32]
    lib.vtts_debug_t2s_sample.restype = i32
    for fn in (lib.vtts_sovits_semantic, lib.vtts_sovits_latent):
        fn.argtypes = [vp, vp, vp, i32, C.c_int64, vp, C.c_int64, vp]
        fn.restype = i32
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


def live_bytes():
    """(device bytes, pinned host bytes) the library holds in this process right now, over every engine (a test hook)."""
    dev, pin = C.c_uint64(), C.c_uint64()
    if load_library().vtts_debug_live_bytes(C.byref(dev), C.byref(pin)) != 0:
        raise VttsError(-1, "vtts_debug_live_bytes failed")
    return int(dev.value), int(pin.value)


def _set_decoder_shape(c, cfg):
    """resblock_* and upsample_* of the decoder (VITS2 / QuickVC) or of the vocoder (config.hifigan_config)."""
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
    c.upsample_initial_channel = int(cfg["upsample_initial_channel"])


def make_c_config(cfg, precision=0):
    c = VttsConfig()
    if cfg.get("model_family") == "t2s":               # config.t2s_config: the GPT's layers in the cv_* fields
        c.model_family = MODEL_FAMILIES["t2s"]
        c.precision = int(precision)
        for k in ("cv_layers", "cv_hidden", "cv_heads", "cv_ffn"):
            setattr(c, k, int(cfg[k]))
        c.cv_ln_eps = float(cfg["cv_ln_eps"])
        return c
    if cfg.get("model_family") == "sovits":            # config.sovits_config: the HuBERT in the cv_* fields, the codebook in n_vocab
        c.model_family = MODEL_FAMILIES["sovits"]
        c.precision = int(precision)
        _set_contentvec_shape(c, cfg)
        c.n_vocab = int(cfg["sv_codebook"])
        return c
    if cfg.get("model_family") == "stabletts":        # the flow-matching decoder reads none of the VITS2 fields
        c.model_family = MODEL_FAMILIES["stabletts"]
        c.precision = int(precision)
        for dst, src in (("st_noise", "noise_channels"), ("st_cond", "cond_channels"), ("st_hidden", "hidden_channels"),
                         ("st_filter", "filter_channels"), ("st_layers", "n_layers"), ("st_heads", "n_heads"),
                         ("st_kernel", "kernel_size"), ("st_spk_dim", "spk_emb_dim"), ("st_n_spks", "n_spks")):
            setattr(c, dst, int(cfg[src]))
        if "enc_n_layers" in cfg:                      # config.stabletts_config: the text encoder of weights.pack_stabletts
            for dst, src in (("st_n_vocab", "n_vocab"), ("st_streams", "n_streams"), ("st_emb_dim", "emb_dim"), ("st_punc_dim", "punc_dim"),
                             ("st_bert_dim", "bert_dim"), ("st_bert_proj", "bert_proj_dim"), ("st_enc_hidden", "enc_hidden_channels"),
                             ("st_enc_filter", "enc_filter_channels"), ("st_enc_layers", "enc_n_layers"), ("st_enc_heads", "enc_n_heads"),
                             ("st_enc_kernel", "enc_kernel_size"), ("st_dur_channels", "dur_channels")):
                setattr(c, dst, int(cfg[src]))
        voc = cfg.get("vocoder")
        if voc:                                        # config.hifigan_config: the vocoder in the decoder fields
            c.decoder_type = 1
            c.inter_channels = int(voc["num_mels"])
            _set_decoder_shape(c, voc)
        bt = cfg.get("bert")
        if bt:                                         # config.bert_config: BERT's transformer in the cv_* fields
            for k in ("cv_layers", "cv_hidden", "cv_heads", "cv_ffn"):
                setattr(c, k, int(bt[k]))
            c.cv_ln_eps = float(bt["cv_ln_eps"])
        return c
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
    _set_decoder_shape(c, cfg)
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
        _set_contentvec_shape(c, cv)
    return c


def _set_contentvec_shape(c, cv):
    """The cv_* fields of a HuBERT / ContentVec shape (config.contentvec_config)."""
    for k in ("cv_layers", "cv_hidden", "cv_heads", "cv_ffn", "cv_conv_dim", "cv_pos_k", "cv_pos_groups"):
        setattr(c, k, int(cv[k]))
    c.cv_n_conv = len(cv["cv_conv_kernel"])
    for i, (k, s) in enumerate(zip(cv["cv_conv_kernel"], cv["cv_conv_stride"])):
        c.cv_conv_kernel[i], c.cv_conv_stride[i] = int(k), int(s)
    c.cv_ln_eps, c.cv_gn_eps = float(cv["cv_ln_eps"]), float(cv["cv_gn_eps"])


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _batch(x, lengths, ndim, t_axis=-1, ragged=False):
    """A batch of recordings or rows as the C ABI reads it: `x` with `ndim` axes, or one item without the batch axis, as
    contiguous float32; `lengths` as int64 [B] (one value for every item; None: the full axis `t_axis`).  ragged: `x` may
    also be a list of items of different lengths along their first axis, zero-padded to the longest (their lengths are
    then the lengths)."""
    if ragged and isinstance(x, (list, tuple)):
        items = [np.asarray(u, np.float32) for u in x]
        if ndim == 2:
            items = [u.reshape(-1) for u in items]
        lengths = np.array([u.shape[0] for u in items], np.int64)
        x = np.zeros((len(items), int(lengths.max())) + items[0].shape[1:], np.float32)
        for b, u in enumerate(items):
            x[b, :u.shape[0]] = u
    x = np.ascontiguousarray(x, dtype=np.float32)
    if x.ndim == ndim - 1:
        x = x[None]
    B = x.shape[0]
    if lengths is None:
        return x, np.full(B, x.shape[t_axis], np.int64)
    return x, np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int64).reshape(-1), (B,)))


def _noise(noise, B, channels):
    """Caller noise standing in for a posterior sample's eps: (float32 [B, channels, >= 1], its row pitch), or (None, 0).
    The engine reads every [b, channel] row, so any other shape is refused."""
    if noise is None:
        return None, 0
    noise = np.ascontiguousarray(noise, dtype=np.float32)
    if noise.ndim != 3 or noise.shape[0] != B or noise.shape[1] != channels or noise.shape[2] < 1:
        raise ValueError("noise must be float32 [B, inter_channels, >= frames]")
    return noise, noise.shape[2]


def _per_item(v, B, width):
    """One row [width] for every item, or one per item [B, width] -> contiguous float32 [B, width]."""
    return np.ascontiguousarray(np.broadcast_to(np.asarray(v, np.float32).reshape(-1, width), (B, width)))


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
        src = np.ascontiguousarray(np.broadcast_to(np.asarray(sid_src, np.int64), (B,)))
        tgt = np.ascontiguousarray(np.broadcast_to(np.asarray(sid_tgt, np.int64), (B,)))
        noise, q_ld = _noise(noise, B, int(self.cfg["inter_channels"]))
        frames = np.zeros(B, np.int64)
        cap = self.convert_frames(lengths) if from_wav else lengths
        fn = self.lib.vtts_convert if from_wav else self.lib.vtts_convert_spec
        out = np.zeros((B, max(1, int(np.max(cap))) * self.hop), np.float32)
        self._check(fn(self.h, _ptr(x), _ptr(lengths), B, ld, _ptr(src), _ptr(tgt), float(noise_scale), _ptr(noise), q_ld,
                       int(seed), _ptr(out), out.shape[1], _ptr(frames)))
        return out[:, : int(frames.max()) * self.hop], frames

    def convert_frames(self, wav_lengths):
        """Frames of the spectrogram of clips of `wav_lengths` samples (center=False after reflect padding by
        (filter_length - hop_length) / 2 on both sides, mel_processing.py:67-71): len // 256 for the reference configuration.
        0 for a clip shorter than min_clip_samples(), which the engine refuses."""
        c = self.cfg
        n_fft, hop = int(c.get("filter_length", 1024)), int(c.get("hop_length", 256))
        pad = (n_fft - hop) // 2
        L = np.asarray(wav_lengths, np.int64)
        return np.where(L >= self.min_clip_samples(), (L + 2 * pad - n_fft) // hop + 1, 0)

    def min_clip_samples(self):
        """The shortest clip the spectrogram front end takes: more samples than the reflect padding (filter_length -
        hop_length) / 2, and at least one frame (hop_length samples)."""
        n_fft, hop = int(self.cfg.get("filter_length", 1024)), int(self.cfg.get("hop_length", 256))
        return max((n_fft - hop) // 2 + 1, hop)

    def convert(self, wav, sid_src, sid_tgt, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Re-voices clips of speaker `sid_src` as speaker `sid_tgt` (vtts_convert).  wav: float32 [B, L] (or [L]) in [-1, 1],
        `lengths` the valid samples per row (default: all).  Returns (float32 [B, hop * max(frames)], frames [B]); row b holds
        hop * frames[b] samples.  noise: optional eps [B, inter_channels, >= frames] of the posterior sample."""
        wav, lengths = _batch(wav, lengths, 2)
        return self._convert(True, wav, lengths, wav.shape[1], sid_src, sid_tgt, noise_scale, noise, seed)

    def convert_spec(self, spec, sid_src, sid_tgt, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Same from the posterior encoder's input features (the reference's `y`): float32 [B, spec_channels, T]."""
        spec, lengths = _batch(spec, lengths, 3)
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
        wav, lengths = _batch(wav, lengths, 2)
        B = wav.shape[0]
        g = np.zeros((B, int(self.cfg["gin_channels"])), np.float32)
        self._check(self.lib.vtts_speaker_embedding(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(g)))
        return g

    def speaker_embedding_mel(self, mel, lengths=None):
        """Same from log-mel rows (mel_spectrogram_torch's output): float32 [B, n_mel_channels, T] (or [n_mel_channels, T])."""
        mel, lengths = _batch(mel, lengths, 3)
        B = mel.shape[0]
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
        units, lengths = _batch(units, lengths, 3, t_axis=1, ragged=True)
        B, T = units.shape[0], units.shape[1]
        g = _per_item(g, B, int(self.cfg["gin_channels"]))
        noise, ld = _noise(noise, B, int(self.cfg["inter_channels"]))
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
    def content_units(self, wav, lengths=None):
        """ContentVec units of 16 kHz sources (vtts_content_units): wav [L], [B, L] with `lengths`, or a list of ragged clips.
        Returns (units float32 [B, max T, hidden], zeros past each clip's end; frames int64 [B])."""
        wav, lengths = _batch(wav, lengths, 2, ragged=True)
        B = wav.shape[0]
        T = max(1, max(_config.contentvec_frames(int(n), self.cfg.get("contentvec")) for n in lengths))
        units = np.zeros((B, T, int((self.cfg.get("contentvec") or _config.contentvec_config())["cv_hidden"])), np.float32)
        frames = np.zeros(B, np.int64)
        self._check(self.lib.vtts_content_units(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(units), T, _ptr(frames)))
        return units, frames

    def quickvc_convert_wav(self, wav, g, lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Source waveforms -> waveforms in the voice of g in one call (vtts_quickvc_convert_wav): content_units, then
        quickvc_convert, without the units leaving the GPU.  Arguments as those two.  Returns (wav [B, hop * max T], frames)."""
        wav, lengths = _batch(wav, lengths, 2, ragged=True)
        B = wav.shape[0]
        T = max(1, max(_config.contentvec_frames(int(n), self.cfg.get("contentvec")) for n in lengths))
        g = _per_item(g, B, int(self.cfg["gin_channels"]))
        noise, ld = _noise(noise, B, int(self.cfg["inter_channels"]))
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

    # ---- resampling of recordings (librosa.load(path, sr=...) and librosa.effects.trim, as vc/convert.py:65-66 uses them)
    def cfm_decode(self, mu, sid=None, lengths=None, n_timesteps=10, temperature=1.0, guidance_scale=0.5, noise=None, seed=0,
                   spk_rows=None, denormalise=False):
        """StableTTS flow-matching decoder (vtts_cfm_decode): mu frame-major [T, cond], [B, T, cond] with `lengths`, or a list
        of ragged [T_b, cond] items; sid int [B] (or one for all), or spk_rows float [B, spk_emb_dim]; noise like mu with
        noise_channels columns, or None for Philox(seed).  Returns (mel float32 [B, max T, noise_channels] frame-major, zeros
        past each utterance; lengths int64 [B]); denormalise: mel * mel_std + mel_mean."""
        mu, lengths = _batch(mu, lengths, 3, t_axis=1, ragged=True)
        B, T = mu.shape[0], mu.shape[1]
        NC, MC, G = (int(self.cfg[k]) for k in ("noise_channels", "cond_channels", "spk_emb_dim"))
        if mu.shape[2] != MC:
            raise ValueError("mu must be frame-major [.., T, %d]" % MC)
        noise_ld = 0
        if noise is not None:
            noise, _ = _batch(noise, None, 3, t_axis=1, ragged=True)
            if noise.shape[0] != B or noise.shape[2] != NC:
                raise ValueError("noise must be frame-major [B, >= T, %d]" % NC)
            noise_ld = noise.shape[1]
        if sid is not None:
            sid = np.ascontiguousarray(np.broadcast_to(np.asarray(sid, np.int64).reshape(-1), (B,)))
        if spk_rows is not None:
            spk_rows = _per_item(spk_rows, B, G)
        mel = np.zeros((B, T, NC), np.float32)
        self._check(self.lib.vtts_cfm_decode(self.h, _ptr(mu), _ptr(lengths), B, T, _ptr(sid), _ptr(spk_rows), int(n_timesteps),
                                             float(temperature), float(guidance_scale), _ptr(noise), noise_ld, int(seed),
                                             _ptr(mel), T, int(bool(denormalise))))
        return mel, lengths

    def hifigan_vocode(self, mel, lengths=None):
        """StableTTS vocoder (vtts_hifigan_vocode): mel frame-major [T, num_mels], [B, T, num_mels] with `lengths`, or a list of
        ragged [T_b, num_mels] items, denormalised.  Returns (wav float32 [B, hop * max T], zeros past each utterance;
        wav_lengths int64 [B] = hop * lengths)."""
        mel, lengths = _batch(mel, lengths, 3, t_axis=1, ragged=True)
        B, T = mel.shape[0], mel.shape[1]
        voc = self.cfg.get("vocoder")
        if not voc:
            raise ValueError("this engine has no vocoder")
        if mel.shape[2] != int(voc["num_mels"]):
            raise ValueError("mel must be frame-major [.., T, %d]" % int(voc["num_mels"]))
        hop = _config.hop_samples(voc)
        wav = np.zeros((B, T * hop), np.float32)
        wl = np.zeros(B, np.int64)
        self._check(self.lib.vtts_hifigan_vocode(self.h, _ptr(mel), _ptr(lengths), B, T, _ptr(wav), T * hop, _ptr(wl)))
        return wav, wl

    def stabletts_synthesise(self, ids, bert, sid, lengths=None, pause=None, n_timesteps=10, temperature=1.0, length_scale=1.0,
                             guidance_scale=0.5, noise=None, seed=0, mel_frames=None, want_prior=False, denormalise=False,
                             want_wav=False, pieces=None, bert_rows=None, piece_lengths=None):
        """StableTTS text-to-mel (vtts_stabletts_synthesise).  ids int [B, n_streams, T] (or [n_streams, T]); bert float [B, T,
        bert_dim] token-major; lengths int [B] (None: T for all); pause float [B, T] or None; sid int [B] (or one for all);
        noise float [B, >= ceil4(frames), noise_channels] frame-major over the padded frame axis, or None for Philox(seed).
        mel_frames: the frame capacity of the result; None asks the engine for the frame counts first (a call with no room,
        which ends after the text phase) and then runs the call with exactly enough.  Returns a dict: mel [B, frames,
        noise_channels] frame-major (zeros past each utterance), mel_lengths int64 [B], durations int32 [B, T], and prior (the
        expanded mel encoder output) when want_prior, and with want_wav the vocoder's wav [B, hop * frames] (zeros past each
        utterance) and wav_lengths int64 [B] (vtts_stabletts_synthesise_wav: the vocoder reads the denormalised mel on the
        device).
        pieces / bert_rows (with bert=None): each utterance's sentence of word pieces, a list of B sequences or int [B, L] with
        piece_lengths int [B] (None: every row is a whole sentence of L pieces), and int [B, T] the row among its own pieces that
        each token reads; BERT then runs on the device and its rows are gathered there (vtts_stabletts_synthesise_pieces_wav,
        which always vocodes: want_wav is implied)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.ndim == 2:
            ids = ids[None]
        B, S, T = ids.shape
        NC, BD = int(self.cfg["noise_channels"]), int(self.cfg.get("bert_dim", 0))
        if S != int(self.cfg.get("n_streams", S)):
            raise ValueError("ids must be [B, %d, T]" % int(self.cfg["n_streams"]))
        if (bert is None) == (pieces is None) or (pieces is None) != (bert_rows is None):
            raise ValueError("give either bert, or pieces with bert_rows")
        if pieces is None:
            bert = np.ascontiguousarray(bert, dtype=np.float32)
            if bert.ndim == 2:
                bert = bert[None]
            if bert.shape != (B, T, BD):
                raise ValueError("bert must be token-major [B, T, %d]" % BD)
        else:
            if not self.cfg.get("bert"):
                raise ValueError("this engine has no BERT")
            if isinstance(pieces, (list, tuple)):
                seqs = [np.asarray(u, np.int64).reshape(-1) for u in pieces] or [np.zeros(0, np.int64)]
                piece_len = np.array([u.size for u in seqs], np.int64)
                pieces = np.zeros((len(seqs), max(1, int(piece_len.max()))), np.int64)
                for b, u in enumerate(seqs):
                    pieces[b, :u.size] = u
            else:
                pieces = np.ascontiguousarray(pieces, dtype=np.int64)
                pieces = pieces[None] if pieces.ndim == 1 else pieces
                piece_len = np.full(pieces.shape[0], pieces.shape[-1], np.int64) if piece_lengths is None else \
                    np.ascontiguousarray(np.broadcast_to(np.asarray(piece_lengths, np.int64).reshape(-1), (pieces.shape[0],)))
            bert_rows = np.ascontiguousarray(bert_rows, dtype=np.int32)
            bert_rows = bert_rows[None] if bert_rows.ndim == 1 else bert_rows
            if pieces.ndim != 2 or pieces.shape[0] != B or pieces.shape[1] < 1 or (piece_len < 1).any() or (piece_len > pieces.shape[1]).any():
                raise ValueError("pieces must hold one sentence of at least one word piece per utterance")
            if bert_rows.shape != (B, T):
                raise ValueError("bert_rows must be [B, T]")
            want_wav = True
        lengths = np.full(B, T, np.int64) if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int64).reshape(-1), (B,)))
        sid = np.ascontiguousarray(np.broadcast_to(np.asarray(sid, np.int64).reshape(-1), (B,)))
        if pause is not None:
            pause = np.ascontiguousarray(pause, dtype=np.float32).reshape(-1, T)
            if pause.shape != (B, T):
                raise ValueError("pause must be [B, T]")
        noise_ld = 0
        if noise is not None:
            noise, _ = _batch(noise, None, 3, t_axis=1, ragged=True)
            if noise.shape[0] != B or noise.shape[2] != NC:
                raise ValueError("noise must be frame-major [B, >= ceil4(frames), %d]" % NC)
            noise_ld = noise.shape[1]
        mel_len = np.zeros(B, np.int64)
        dur = np.zeros((B, T), np.int32)
        if mel_frames is None:      # a token lasts at most max(sum of dur_channels sigmoids, its pause) * length_scale frames
            per = np.full((B, T), float(self.cfg["dur_channels"]), np.float64) if pause is None else np.maximum(pause, float(self.cfg["dur_channels"]))
            per = np.maximum(np.ceil(per * float(length_scale)) + 1, 1) * (np.arange(T)[None, :] < lengths[:, None])
            mel_frames = int(per.sum(1).max())
        mel = np.zeros((B, int(mel_frames), NC), np.float32)
        prior = np.zeros_like(mel) if want_prior else None
        args = (self.h, _ptr(ids), _ptr(lengths), B, T, _ptr(bert), _ptr(pause), _ptr(sid), int(n_timesteps), float(temperature),
                float(length_scale), float(guidance_scale), _ptr(noise), noise_ld, int(seed), _ptr(mel), int(mel_frames), _ptr(mel_len),
                _ptr(dur), _ptr(prior), int(bool(denormalise)))
        if want_wav:
            hop = _config.hop_samples(self.cfg["vocoder"]) if self.cfg.get("vocoder") else 1
            wav = np.zeros((B, int(mel_frames) * hop), np.float32)
            wl = np.zeros(B, np.int64)
            if pieces is not None:
                args = args[:5] + (_ptr(pieces), _ptr(piece_len), pieces.shape[1], _ptr(bert_rows)) + args[6:]
                self._check(self.lib.vtts_stabletts_synthesise_pieces_wav(*args, _ptr(wav), wav.shape[1], _ptr(wl)))
            else:
                self._check(self.lib.vtts_stabletts_synthesise_wav(*args, _ptr(wav), wav.shape[1], _ptr(wl)))
        else:
            self._check(self.lib.vtts_stabletts_synthesise(*args))
        top = int(mel_len.max())
        out = {"mel": np.ascontiguousarray(mel[:, :top]), "mel_lengths": mel_len, "durations": dur}
        if want_wav:
            out["wav"], out["wav_lengths"] = np.ascontiguousarray(wav[:, :top * hop]), wl
        if want_prior:
            out["prior"] = np.ascontiguousarray(prior[:, :top])
        return out

    def bert_features(self, ids, lengths=None):
        """BERT's last-layer rows of word-piece sentences (vtts_bert_features): ids int64 [B, L] with lengths, or a list of
        sequences.  Returns float32 [B, max length, hidden] (zeros after each sentence) and the lengths."""
        if isinstance(ids, (list, tuple)):
            if not ids:
                raise ValueError("bert_features needs at least one sentence")
            seqs = [np.asarray(u, np.int64).reshape(-1) for u in ids]
            lengths = np.array([u.size for u in seqs], np.int64)
            ids = np.zeros((len(seqs), max(1, int(lengths.max()))), np.int64)
            for b, u in enumerate(seqs):
                ids[b, :u.size] = u
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.ndim == 1:
            ids = ids[None]
        B, L = ids.shape
        if B == 0 or L == 0:
            raise ValueError("bert_features needs at least one sentence of at least one word piece")
        lengths = np.full(B, L, np.int64) if lengths is None else np.ascontiguousarray(np.broadcast_to(np.asarray(lengths, np.int64).reshape(-1), (B,)))
        H = int(self.cfg["bert"]["cv_hidden"]) if self.cfg.get("bert") else 1
        out = np.zeros((B, max(1, int(lengths.max())), H), np.float32)
        self._check(self.lib.vtts_bert_features(self.h, _ptr(ids), _ptr(lengths), B, L, _ptr(out), out.shape[1]))
        return out, lengths

    def t2s_decode(self, phones, prompts=None, bert=None, top_k=20, top_p=0.6, temperature=0.6, repetition_penalty=1.35,
                   early_stop_num=-1, step_cap=1500, seeds=0, q=None, logits_steps=0):
        """GPT-SoVITS text-to-semantic decoding (vtts_t2s_decode) of a ragged batch.  phones: a list of B phone-id sequences;
        prompts: None or a list of B semantic-token sequences (empty for none); bert: None or a list of B float [T_b, 1024]
        token-major features; seeds: B ints, or one int s giving sentence b the seed s + b (so that no two sentences of a call
        share a Philox stream; a sentence keeps its tokens in another batch when it keeps its seed); q: float [B, steps, V] replacing the Philox draws; logits_steps > 0 also
        returns the raw logits of the first that many sampling steps, float [B, logits_steps, V].
        Returns (tokens: list of B int64 arrays = y[:, :-1] with the prompt, idx: int64 [B][, logits])."""
        B = len(phones)
        if B < 1:
            raise ValueError("t2s_decode needs at least one sentence")
        lens = np.array([len(p) for p in phones], np.int64)
        L = max(1, int(lens.max()))
        ids = np.zeros((B, L), np.int64)
        for b, p in enumerate(phones):
            ids[b, :len(p)] = np.asarray(p, np.int64)
        pr = pl = None
        Pld = 0
        if prompts is not None:
            if len(prompts) != B:
                raise ValueError("one prompt per sentence")
            pl = np.array([len(p) for p in prompts], np.int64)
            Pld = max(1, int(pl.max()))
            pr = np.zeros((B, Pld), np.int64)
            for b, p in enumerate(prompts):
                pr[b, :len(p)] = np.asarray(p, np.int64)
        bt = None
        if bert is not None:
            bt = np.zeros((B, L, 1024), np.float32)
            for b, f in enumerate(bert):
                f = np.asarray(f, np.float32)
                if f.shape != (lens[b], 1024):
                    raise ValueError("bert[%d] must be [T, 1024] token-major" % b)
                bt[b, :lens[b]] = f
        V = int(self.cfg["t2s_vocab"])
        gen_max = step_cap if early_stop_num < 0 else min(step_cap, early_stop_num + 1)
        tok_ld = Pld + max(gen_max, 1)
        sd = None
        q_ld = 0
        if q is not None:
            q = np.ascontiguousarray(q, np.float32)
            if q.ndim != 3 or q.shape[0] != B or q.shape[2] != V:
                raise ValueError("q must be float32 [B, steps, V]")
            q_ld = q.shape[1]
        else:
            sd = np.asarray(seeds, np.uint64).reshape(-1)
            if sd.size == 1:
                sd = sd[0] + np.arange(B, dtype=np.uint64)
            if sd.size != B:
                raise ValueError("seeds: one int or one per sentence")
            sd = np.ascontiguousarray(sd)
        tokens = np.zeros((B, tok_ld), np.int64)
        n = np.zeros(B, np.int64)
        idx = np.zeros(B, np.int64)
        lg = np.zeros((B, logits_steps, V), np.float32) if logits_steps > 0 else None
        self._check(self.lib.vtts_t2s_decode(self.h, _ptr(ids), _ptr(lens), B, L, _ptr(bt), _ptr(pr), _ptr(pl), Pld, int(top_k),
                                             float(top_p), float(temperature), float(repetition_penalty), int(early_stop_num),
                                             int(step_cap), _ptr(sd), _ptr(q), q_ld, _ptr(tokens), tok_ld, _ptr(n), _ptr(idx),
                                             _ptr(lg), logits_steps))
        out = [tokens[b, :n[b]].copy() for b in range(B)]
        return (out, idx, lg) if lg is not None else (out, idx)

    # ---- GPT-SoVITS prompt tokens (HuBERT and SynthesizerTrn.extract_latent); cfg is config.sovits_config
    def sovits_semantic(self, wav, lengths=None):
        """Semantic codes of 16 kHz recordings, already padded (vtts_sovits_semantic): wav [L], [B, L] with `lengths`, or a list
        of ragged clips.  Returns (codes int64 [B, max n], -1 after each clip's codes; n int64 [B], HuBERT's frames // 2)."""
        wav, lengths = _batch(wav, lengths, 2, ragged=True)
        B = wav.shape[0]
        T = max(1, max(_config.contentvec_frames(int(n), self.cfg) // 2 for n in lengths))
        codes = np.zeros((B, T), np.int64)
        n = np.zeros(B, np.int64)
        self._check(self.lib.vtts_sovits_semantic(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], _ptr(codes), T, _ptr(n)))
        return codes, n

    def sovits_latent(self, feats, frames=None):
        """Semantic codes of HuBERT rows (vtts_sovits_latent): feats frame-major [T, hidden], [B, T, hidden] with `frames`, or a
        list of ragged [T_b, hidden] clips.  Returns (codes int64 [B, max T // 2], -1 after each clip's codes; n int64 [B])."""
        H = int(self.cfg["cv_hidden"])
        if isinstance(feats, (list, tuple)):
            items = [np.asarray(f, np.float32).reshape(-1, H) for f in feats]
            frames = np.array([f.shape[0] for f in items], np.int64)
            x = np.zeros((len(items), max(1, int(frames.max())), H), np.float32)
            for b, f in enumerate(items):
                x[b, :f.shape[0]] = f
        else:
            x = np.ascontiguousarray(feats, dtype=np.float32)
            if x.ndim == 2:
                x = x[None]
            if x.ndim != 3 or x.shape[2] != H:
                raise ValueError("feats must be [T, %d], [B, T, %d] or a list of [T_b, %d]" % (H, H, H))
            B = x.shape[0]
            frames = np.full(B, x.shape[1], np.int64) if frames is None else \
                np.ascontiguousarray(np.broadcast_to(np.asarray(frames, np.int64).reshape(-1), (B,)))
        B = x.shape[0]
        T = max(1, int(frames.max()) // 2)
        codes = np.zeros((B, T), np.int64)
        n = np.zeros(B, np.int64)
        self._check(self.lib.vtts_sovits_latent(self.h, _ptr(x), _ptr(frames), B, x.shape[1], _ptr(codes), T, _ptr(n)))
        return codes, n

    def resample(self, wav, from_rate, to_rate, lengths=None, trim_top_db=None, return_bounds=False):
        """Clips at `from_rate` Hz resampled to `to_rate` Hz (vtts_resample: scipy.signal.resample_poly's filter, not soxr), and
        with `trim_top_db` trimmed of leading and trailing silence as librosa.effects.trim(y, top_db=trim_top_db) does.  wav:
        one clip [L], a padded batch [B, L] with `lengths`, or a list of ragged clips.  Works on engines of every model family.
        Returns the list of float32 clips; with return_bounds also int64 [B, 2], the [start, end) kept of each resampled clip."""
        if min(int(from_rate), int(to_rate)) <= 0:
            raise ValueError("sample rates must be positive")
        wav, lengths = _batch(wav, lengths, 2, ragged=True)
        B = wav.shape[0]
        g = math.gcd(int(from_rate), int(to_rate))
        up, down = int(to_rate) // g, int(from_rate) // g
        out_len = -(-lengths * up // down)
        out = np.zeros((B, max(1, int(out_len.max()))), np.float32)
        n = np.zeros(B, np.int64)
        bounds = np.zeros((B, 2), np.int64)
        self._check(self.lib.vtts_resample(self.h, _ptr(wav), _ptr(lengths), B, wav.shape[1], int(from_rate), int(to_rate),
                                           float(trim_top_db or 0.0), _ptr(out), out.shape[1], _ptr(n), _ptr(bounds)))
        clips = [out[b, :int(n[b])].copy() for b in range(B)]
        return (clips, bounds) if return_bounds else clips

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
        noise, q_ld = _noise(noise, B, int(self.cfg["inter_channels"]))
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
        wav, wav_lengths = _batch(wav, wav_lengths, 2)
        return self._align(True, ids, lengths, sid, wav, wav_lengths, noise_scale, noise, seed)

    def align_spec(self, ids, lengths, sid, spec, spec_lengths=None, noise_scale=1.0, noise=None, seed=0):
        """Same from the posterior encoder's input features (the reference's `y`): float32 [B, spec_channels, T]."""
        spec, spec_lengths = _batch(spec, spec_lengths, 3)
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

    def _hook_arrays(self, spec):
        """Contiguous copies of a debug hook's arrays, each checked against its shape: spec is a list of (name, array or None,
        dtype, shape); a shape entry None takes any extent.  Raises ValueError before anything reaches the library."""
        out = []
        for name, a, dt, shape in spec:
            if a is None:
                out.append(None)
                continue
            a = np.ascontiguousarray(a, dtype=dt).copy()
            if a.ndim != len(shape) or any(n is not None and a.shape[i] != n for i, n in enumerate(shape)):
                raise ValueError("%s: shape %s, expected %s" % (name, a.shape, tuple("*" if n is None else n for n in shape)))
            out.append(a)
        return out

    def debug_dds(self, stack, lens, y, x=None, x0=None, cond=None):
        """The three DDSConv layers of `stack` ("dp.convs" with x, or "dp.flows.<i>.convs" with x0 and cond), launched as
        dds_stack launches them (vtts_debug_dds).  Rows packed as cr.offsets(lens); y: float32 [3, rows, D], rows outside the
        utterances keep it.  Returns the new y: the output of every layer, each computed from the previous one."""
        D = int(self.cfg["dp_filter_channels"])
        y = np.ascontiguousarray(y, dtype=np.float32)
        rows = y.shape[1] if y.ndim == 3 else -1
        y, x, x0, cond = self._hook_arrays([("y", y, np.float32, (3, rows, D)), ("x", x, np.float32, (rows, D)),
                                            ("x0", x0, np.float32, (rows,)), ("cond", cond, np.float32, (rows, D))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        self._check(self.lib.vtts_debug_dds(self.h, stack.encode(), lens.size, _ptr(lens), rows, _ptr(x), _ptr(x0), _ptr(cond),
                                            _ptr(y)))
        return y

    def debug_spline(self, lens, params, x1):
        """spline_inverse_kernel on params float32 [rows, ldh] and x1 float32 [rows] (vtts_debug_spline).  Returns the new x1."""
        params = np.ascontiguousarray(params, dtype=np.float32)
        if params.ndim != 2:
            raise ValueError("params: shape %s, expected (rows, ldh)" % (params.shape,))
        x1, = self._hook_arrays([("x1", x1, np.float32, (params.shape[0],))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        self._check(self.lib.vtts_debug_spline(self.h, lens.size, _ptr(lens), x1.shape[0], _ptr(params), params.shape[1], _ptr(x1)))
        return x1

    def debug_front_end(self, x, lengths, feat, mag=None, from_spec=False):
        """The spectrogram front end of conversion, alignment and the speaker encoder (vtts_debug_front_end) on waveforms x
        float32 [B, ld] (or caller features [B, spec_channels, ld] with from_spec).  feat float32 [rows, spec_pad] and, for a
        mel engine's waveform input, mag float32 [rows, filter_length // 2 + 1]: initial contents that rows outside the clips
        keep.  Returns (frames int32 [B], mag, feat), rows packed from the frame counts."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        lengths = np.ascontiguousarray(lengths, dtype=np.int64)
        feat = np.ascontiguousarray(feat, dtype=np.float32).copy()
        if feat.ndim != 2:
            raise ValueError("feat: shape %s, expected (rows, spec_pad)" % (feat.shape,))
        mag, = self._hook_arrays([("mag", mag, np.float32, (feat.shape[0], None))])
        frames = np.zeros(lengths.size, np.int32)
        self._check(self.lib.vtts_debug_front_end(self.h, int(bool(from_spec)), _ptr(x), _ptr(lengths), lengths.size, x.shape[-1],
                                                  _ptr(frames), feat.shape[0], _ptr(mag), _ptr(feat)))
        return frames, mag, feat

    def debug_istft(self, lens, post, wav, first=0):
        """The decoder tail istft_pqmf_kernel (vtts_debug_istft) on conv_post rows post float32 [rows, subbands * (n_fft + 2)]
        of utterances of lens frames packed from row `first`.  wav float32 [n]: initial contents that samples outside the
        utterances keep.  Returns the new wav."""
        post = np.ascontiguousarray(post, dtype=np.float32)
        if post.ndim != 2:
            raise ValueError("post: shape %s, expected (rows, channels)" % (post.shape,))
        wav, = self._hook_arrays([("wav", wav, np.float32, (None,))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        self._check(self.lib.vtts_debug_istft(self.h, lens.size, _ptr(lens), int(first), post.shape[0], _ptr(post), wav.size, _ptr(wav)))
        return wav

    def debug_mrf_mean(self, lens, rmul, x, out=None, hi=None, lo=None, use_tc=False, last=False):
        """The MRF mean (vtts_debug_mrf_mean) of x float32 [n, rows, C]: mrf_mean_kernel into out float32 [rows, C], or with
        use_tc mrf_mean_planes_kernel into the planes hi / lo uint16 [plane_rows, C] (and out, if given).  Initial contents
        are kept where the kernel does not write.  Returns (out, hi, lo)."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        if x.ndim != 3:
            raise ValueError("x: shape %s, expected (n, rows, C)" % (x.shape,))
        n, rows, Cc = x.shape
        out, hi, lo = self._hook_arrays([("out", out, np.float32, (rows, Cc)), ("hi", hi, np.uint16, (None, Cc)),
                                         ("lo", lo, np.uint16, (None, Cc))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        self._check(self.lib.vtts_debug_mrf_mean(self.h, int(bool(use_tc)), lens.size, _ptr(lens), int(rmul), Cc, n, rows, _ptr(x),
                                                 int(bool(last)), _ptr(out), 0 if hi is None else hi.shape[0], _ptr(hi), _ptr(lo)))
        return out, hi, lo

    def debug_t2s_sample(self, logits, state, y, top_k=20, top_p=0.6, temperature=0.6, repetition_penalty=1.35, early_stop_num=-1,
                         step_cap=1500, seeds=None, q=None, raw=None):
        """One t2s_sample_kernel launch (vtts_debug_t2s_sample) on logits float32 [B, V], state int32 [B, 8] (P, NY, GEN, STOP,
        YOFF at the indices of t2s.cuh T2sSt; YOFF becomes b * y_ld) and y int32 [B, y_ld], whose first P + GEN entries of a
        row are its previous tokens.  Exactly one of seeds (uint64 [B]) and q (float32 [B, q_ld, V]); raw: float32
        [B, raw_ld, V] raw-logit rows to fill, or None.  Returns a dict of state, y, seen (uint32 [B, (V + 31) // 32]),
        n_stopped and raw."""
        V = int(self.cfg["t2s_vocab"])
        logits = np.ascontiguousarray(logits, dtype=np.float32)
        if logits.ndim != 2 or logits.shape[1] != V:
            raise ValueError("logits: shape %s, expected (B, %d)" % (logits.shape, V))
        B = logits.shape[0]
        y = np.ascontiguousarray(y, dtype=np.int32)
        state, y, seeds, q, raw = self._hook_arrays([("state", state, np.int32, (B, 8)), ("y", y, np.int32, (B, None)),
                                                     ("seeds", seeds, np.uint64, (B,)), ("q", q, np.float32, (B, None, V)),
                                                     ("raw", raw, np.float32, (B, None, V))])
        seen = np.zeros((B, (V + 31) // 32), np.uint32)
        ns = np.zeros(1, np.int32)
        self._check(self.lib.vtts_debug_t2s_sample(self.h, B, _ptr(logits), _ptr(state), _ptr(y), y.shape[1], int(top_k), float(top_p),
                                                   float(temperature), float(repetition_penalty), int(early_stop_num), int(step_cap),
                                                   _ptr(seeds), _ptr(q), 0 if q is None else q.shape[1], _ptr(seen), _ptr(ns),
                                                   _ptr(raw), 0 if raw is None else raw.shape[1]))
        return dict(state=state, y=y, seen=seen, n_stopped=int(ns[0]), raw=raw)

    def debug_durations(self, lens, z, length_scale, stats, eps, noise_scale, frame_rows, frame_cap=0, wceil=None, cum=None, z_p=None,
                        frame_token=None):
        """duration_kernel then sample_prior_kernel (vtts_debug_durations).  z float32 [rows]; stats float32 [rows, 2I]; eps
        float32 [B, I, eps_ld]; wceil / cum int32 [rows], z_p float32 [frame_rows, I], frame_token int32 [frame_rows]: initial
        contents (default zeros) that rows outside the utterances keep.  Returns a dict of wceil, cum, ylen, ylen_real, frm_off,
        published (host-read lengths [B] then offsets [B + 1]), z_p, frame_token."""
        z = np.ascontiguousarray(z, dtype=np.float32)
        rows, B, I, F = z.shape[0], len(lens), int(self.cfg["inter_channels"]), int(frame_rows)
        if z.ndim != 1:
            raise ValueError("z: shape %s, expected (rows,)" % (z.shape,))
        zeros = lambda a, shape, dt: np.zeros(shape, dt) if a is None else a
        stats, eps, wceil, cum, z_p, frame_token = self._hook_arrays([
            ("stats", stats, np.float32, (rows, 2 * I)), ("eps", eps, np.float32, (B, I, None)),
            ("wceil", zeros(wceil, rows, np.int32), np.int32, (rows,)), ("cum", zeros(cum, rows, np.int32), np.int32, (rows,)),
            ("z_p", zeros(z_p, (F, I), np.float32), np.float32, (F, I)),
            ("frame_token", zeros(frame_token, F, np.int32), np.int32, (F,))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        o = dict(wceil=wceil, cum=cum, ylen=np.zeros(B, np.int32), ylen_real=np.zeros(B, np.int32), frm_off=np.zeros(B + 1, np.int32),
                 published=np.zeros(2 * B + 1, np.int32), z_p=z_p, frame_token=frame_token)
        self._check(self.lib.vtts_debug_durations(
            self.h, B, _ptr(lens), rows, _ptr(z), float(length_scale), int(frame_cap), _ptr(stats), _ptr(eps), eps.shape[-1],
            float(noise_scale), _ptr(o["wceil"]), _ptr(o["cum"]), _ptr(o["ylen"]), _ptr(o["ylen_real"]), _ptr(o["frm_off"]),
            _ptr(o["published"]), F, _ptr(o["z_p"]), _ptr(o["frame_token"])))
        return o

    def debug_stt_durations(self, lens, mu_dp, pause, length_scale, x, frame_rows, mu_mel=None, denormalise=False, prior=True,
                            init=None):
        """stt_dur_kernel, stt_expand_kernel and stt_pause_fill_kernel (vtts_debug_stt_durations).  mu_dp float32 [rows, DC],
        pause [rows], x [rows, MC], mu_mel [rows, NC].  init: dict of initial dur / first / logw / mu / pau / prior / mel
        buffers (default zeros), which rows outside the utterances keep.  Returns a dict of those and ylen."""
        c = self.cfg
        if "dur_channels" not in c:
            raise ValueError("debug_stt_durations needs a StableTTS engine with a text encoder")
        DC, MC, NC = int(c["dur_channels"]), int(c["cond_channels"]), int(c["noise_channels"])
        mu_dp = np.ascontiguousarray(mu_dp, dtype=np.float32)
        rows, B, F = mu_dp.shape[0], len(lens), int(frame_rows)
        init = init or {}
        buf = lambda k, shape, dt: init[k] if k in init else np.zeros(shape, dt)
        (mu_dp, pause, x, mu_mel, dur, first, logw, mu, pau, pr, mel) = self._hook_arrays([
            ("mu_dp", mu_dp, np.float32, (rows, DC)), ("pause", pause, np.float32, (rows,)), ("x", x, np.float32, (rows, MC)),
            ("mu_mel", mu_mel, np.float32, (rows, NC)), ("dur", buf("dur", rows, np.int32), np.int32, (rows,)),
            ("first", buf("first", rows, np.int32), np.int32, (rows,)), ("logw", buf("logw", rows, np.float32), np.float32, (rows,)),
            ("mu", buf("mu", (F, MC), np.float32), np.float32, (F, MC)), ("pau", buf("pau", F, np.float32), np.float32, (F,)),
            ("prior", buf("prior", (F, NC), np.float32) if prior else None, np.float32, (F, NC)),
            ("mel", buf("mel", (F, NC), np.float32), np.float32, (F, NC))])
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        o = dict(dur=dur, first=first, ylen=np.zeros(B, np.int32), logw=logw, mu=mu, pau=pau, prior=pr, mel=mel)
        self._check(self.lib.vtts_debug_stt_durations(
            self.h, B, _ptr(lens), rows, _ptr(mu_dp), _ptr(pause), float(length_scale), _ptr(x), _ptr(mu_mel), int(bool(denormalise)),
            _ptr(o["dur"]), _ptr(o["first"]), _ptr(o["ylen"]), _ptr(o["logw"]), F, _ptr(o["mu"]), _ptr(o["pau"]),
            _ptr(o["prior"]), _ptr(o["mel"])))
        return o

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
