"""QuickVC conversion on the host: the float64 oracle against the reference's SynthesizerTrn.infer
(tests/golden/ref_quickvc_convert.npz, written from the unmodified vc/models.py by oracle/make_golden_quickvc_convert.py),
QuickVC's upsampling pads in the engine's polyphase split, the torch.istft tail as the engine's kernel computes it, the
synthetic checkpoint, the packed layout, the config refusals, the C entry point and the CLI."""
import copy
import ctypes
import math
import wave

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from oracle import quickvc_convert_oracle as O
from vosk_tts_b200 import config as C, engine as E, quickvc, weights

REF = np.load(QI.GOLDEN + "/ref_quickvc_convert.npz")


@pytest.fixture(scope="module")
def folded():
    return O.as_float64(weights.fold_weight_norm(QC.model()))


@pytest.mark.parametrize("i", range(len(QC.CASES)))
def test_oracle_matches_reference(i, folded):
    T, _ = QC.CASES[i]
    case = "T%d" % T
    r = O.infer(QC.units(T, i), REF[case + "/g"], folded, QI.config(), QC.eps(T, i))
    keep = QC.kept_frames(T)
    errs = {k: float(np.abs(r[k][:, keep] - REF[case + "/" + k]).max()) for k in ("m_p", "logs_p", "z_p", "z")}
    errs["o"] = float(np.abs(r["o"] - REF[case + "/o"]).max())
    print(case, errs)
    assert r["o"].shape == (320 * T,)
    assert max(errs.values()) < 1e-6, errs
    assert np.abs(REF[case + "/o"]).max() >= 0.1


@pytest.mark.parametrize("i", [0, 1])
def test_polyphase_split_with_quickvc_pads(i):
    cfg = QI.config()
    u, K = cfg["upsample_rates"][i], cfg["upsample_kernel_sizes"][i]
    p, op = C.convt_pad(cfg, i)
    assert (p, op) == [(6, 1), (6, 0)][i]
    g = torch.Generator().manual_seed(i)
    T, Ci, Co = 9, 3, 2
    x = torch.randn(1, Ci, T, generator=g, dtype=torch.float64)
    W = torch.randn(Ci, Co, K, generator=g, dtype=torch.float64)
    ref = F.conv_transpose1d(x, W, stride=u, padding=p, output_padding=op)[0]
    assert ref.shape[1] == u * T
    y = torch.zeros(Co, u * T, dtype=torch.float64)
    for r, (pad, js) in enumerate(weights.convt_phases(u, K, p)):
        for t in range(T):
            for m, j in enumerate(js):
                s = t - pad + m
                if 0 <= s < T:
                    y[:, u * t + r] += x[0, :, s] @ W[:, :, j]
    assert float((ref - y).abs().max()) < 1e-12


def tail_numpy(spec, phase, n_fft=16, hop=4):
    """The inverse STFT as istft_pqmf_kernel computes it with its w2 table (one band): for every kept sample m, the frames
    fa..fb that cover it, sum_f basis . rec_f at position m + n_fft/2 - f*hop, times scale / sum_f w2[pos]."""
    basis = weights.istft_inverse_basis(n_fft, hop).astype(np.float64)
    w2 = weights.hann_squared(n_fft).astype(np.float64)
    rec = np.concatenate([spec * np.cos(phase), spec * np.sin(phase)], 0)         # [2 nb][L]
    L1 = rec.shape[1]
    M = (L1 - 1) * hop
    y = np.zeros(M)
    for m in range(M):
        u = m + n_fft // 2
        fa = max(0, -(-(u - (n_fft - 1)) // hop))
        fb = min(u // hop, L1 - 1)
        a = env = 0.0
        for f in range(fa, fb + 1):
            pos = u - f * hop
            a += rec[:, f] @ basis[:, pos]
            env += w2[pos]
        y[m] = a * (n_fft / hop) / env
    return y


@pytest.mark.parametrize("T", [1, 50])
def test_envelope_tail_equals_torch_istft(T):
    rng = np.random.RandomState(T)
    L = 20 * T + 1                                     # conv_post frames of T content frames
    x = rng.randn(18, L)
    spec, phase = np.exp(x[:9] * 0.5), math.pi * np.sin(x[9:])
    ref = O.istft(torch.from_numpy(spec)[None], torch.from_numpy(phase)[None], 16, 4)[0].numpy()
    y = tail_numpy(spec, phase)
    assert y.shape == ref.shape == (80 * T,)
    assert np.abs(y - ref).max() < 1e-5 * np.abs(ref).max()


def test_synthetic_names_and_shapes_match_reference():
    sd = QC.model()
    names = sorted(sd)
    assert names == list(REF["names"])
    assert [",".join(map(str, sd[k].shape)) for k in names] == list(REF["shapes"])


def test_packed_layout():
    cfg = QI.config()
    w = weights.fold_weight_norm(QC.model())
    blob, man = weights.pack_quickvc(w, cfg)
    blob0, man0 = weights.pack_quickvc(weights.fold_weight_norm(QI.speaker_encoder()), cfg)
    assert man.startswith(man0) and np.array_equal(blob[:blob0.size], blob0)       # the conversion side comes after
    ent = {n: (int(o), int(c)) for n, o, c in (l.split() for l in man.splitlines())}
    get = lambda n: blob[ent[n][0]:ent[n][0] + ent[n][1]]
    H, G = 192, 256
    assert ent["encp.pre.w"][1] == 768 * H and "encp.cond.w" not in ent and "encq.pre.w" not in ent
    assert all("encp.in%d.th" % i in ent and "encp.rss%d.b" % i in ent for i in range(16))
    assert all("flow.%d.in3.w" % f in ent for f in range(4)) and "dec.up0.p4.th" in ent and "dec.pqmf" in ent
    # the stacked cond rows: 4 flows x 4 WN layers x 2H (gate-interleaved), then dec.cond
    cw = get("cond.w").reshape(-1, G)
    assert cw.shape[0] == 4 * 4 * 2 * H + 512
    il = np.arange(2 * H).reshape(2, H).T.reshape(-1)
    assert np.array_equal(cw[:2 * H], w["flow.flows.0.enc.cond_layer.weight"][:2 * H, :, 0].numpy()[il])
    assert np.array_equal(cw[-512:], w["dec.cond.weight"][:, :, 0].numpy())
    assert np.allclose(get("dec.w2"), (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(16) / 16)) ** 2)
    # stage 0's phases follow QuickVC's pad 6 (taps 3, 3, 3, 3, 4), not VITS2's 5
    taps = [ent["dec.up0.p%d.w" % r][1] // (512 * 256) for r in range(5)]
    assert taps == [len(js) for _, js in weights.convt_phases(5, 16, 6)] == [3, 3, 3, 3, 4]
    # precision 0 leaves out every split-bf16 copy, 1 every fp32 copy of the convs on the tensor cores
    _, man_0 = weights.pack_quickvc(w, cfg, precision=0)
    _, man_1 = weights.pack_quickvc(w, cfg, precision=1)
    assert ".th " not in man_0 and "encp.in0.w " not in man_1 and "encp.pre.w " in man_1


@pytest.mark.parametrize("change", [{"upsample_rates": [5, 4, 2], "upsample_kernel_sizes": [16, 16, 4]},
                                    {"upsample_rates": [5], "upsample_kernel_sizes": [16]},
                                    {"upsample_kernel_sizes": [15, 16]}])
def test_config_refusals(change):
    j = copy.deepcopy(QI.QUICKVC_JSON)
    j["model"].update(change)
    with pytest.raises(ValueError):
        C.from_quickvc_json(j)


def test_config():
    cfg = QI.config()
    assert cfg["flow_n_flows"] == 4 and cfg["flow_wn_layers"] == 4 and not cfg["use_transformer_flows"]
    assert [C.convt_pad(cfg, i) for i in range(2)] == [(6, 1), (6, 0)]
    assert [C.convt_pad(C.DEFAULT_CONFIG, i) for i in range(2)] == [(6, 0), (6, 0)]
    assert C.hop_total(cfg) == 320


def test_abi_symbol_exported():
    assert "vtts_quickvc_convert" in E.EXPORTS
    lib = ctypes.CDLL(E.lib_path())
    assert hasattr(lib, "vtts_quickvc_convert")
    with open(E._build.CSRC + "/../../include/vtts.h") as f:
        assert "int vtts_quickvc_convert(vtts_handle h, const float* units, const int64_t* unit_lengths" in f.read()


def _write(path, sr, n=1600):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.zeros(n, np.int16).tobytes())


def test_cli_arguments(tmp_path, capsys):
    import json
    cfgp = tmp_path / "quickvc.json"
    cfgp.write_text(json.dumps(QI.QUICKVC_JSON))
    units = tmp_path / "src.npy"
    np.save(units, np.zeros((5, 768), np.float32))
    base = ["--config", str(cfgp), "--checkpoint", str(tmp_path / "G.pth"), "--units", str(units), "--out-dir", str(tmp_path / "o")]
    with pytest.raises(SystemExit):
        quickvc.main(base)                                          # --target missing
    _write(tmp_path / "t22.wav", 22050)
    with pytest.raises(SystemExit):
        quickvc.main(base + ["--target", str(tmp_path / "t22.wav")])
    assert "22050 Hz" in capsys.readouterr().err
    _write(tmp_path / "t16.wav", 16000)
    bad = tmp_path / "bad.npy"
    np.save(bad, np.zeros((5, 1024), np.float32))
    with pytest.raises(SystemExit):
        quickvc.main(base[:5] + [str(bad)] + base[6:] + ["--target", str(tmp_path / "t16.wav")])
    assert "768" in capsys.readouterr().err


def test_wav_io_clips(tmp_path):
    p = tmp_path / "x.wav"
    quickvc.write_wav(str(p), np.array([0.5, 1.5, -2.0, 0.0], np.float32))
    with wave.open(str(p)) as f:
        x = np.frombuffer(f.readframes(4), np.int16)
    assert list(x) == [16384, 32767, -32768, 0]
    assert np.allclose(quickvc.read_wav(str(p)), x / 32768.0)
