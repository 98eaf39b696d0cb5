"""QuickVC speaker encoder on the host: the float64 oracle against the reference's g and log-mel (tests/golden/ref_quickvc.npz,
written from the unmodified vc/models.py by oracle/make_golden_quickvc.py), the slicing of embed_utterance, the config
refusals, the synthetic checkpoint's names and shapes, and the packed layout of the recurrence kernel."""
import copy

import numpy as np
import pytest
import torch

from oracle import quickvc_oracle as O, vc_oracle
from vosk_tts_b200 import config as C, engine as E, weights
import quickvc_inputs as QI

REF = np.load(QI.GOLDEN + "/ref_quickvc.npz")


@pytest.mark.parametrize("key", [k for k, _, _, _ in QI.TARGETS])
def test_oracle_matches_reference(key):
    cfg = QI.config()
    y = torch.from_numpy(QI.wav_float(QI.targets()[key]))[None].double()
    mel = vc_oracle.mel_spectrogram(y, cfg["filter_length"], cfg["n_mel_channels"], cfg["sampling_rate"], cfg["hop_length"],
                                    cfg["win_length"], cfg["mel_fmin"], cfg["mel_fmax"])[0].numpy()
    ref_mel = REF[key + "/mel"]
    assert mel.shape == ref_mel.shape
    assert np.abs(mel - ref_mel).max() < 2e-3
    g = O.embed(ref_mel, QI.speaker_encoder())
    assert np.abs(g - REF[key + "/g"]).max() < 1e-6
    assert abs(np.linalg.norm(g) - 1.0) < 0.2


def test_target_lengths_cover_the_slicing_cases():
    frames = {k: REF[k + "/mel"].shape[1] for k, _, _, _ in QI.TARGETS}
    assert frames["short"] < 128 and frames["t129"] == 129 and frames["long"] >= 400


def test_slices():
    assert O.slices(1) == [(0, 1)]
    assert O.slices(128) == [(0, 128)]
    assert O.slices(129) == [(0, 128), (1, 128)]
    assert O.slices(192) == [(0, 128), (64, 128)]
    assert O.slices(193) == [(0, 128), (64, 128), (65, 128)]
    for T in range(129, 1000, 7):
        s = O.slices(T)
        assert s[-1] == (T - 128, 128) and [a for a, _ in s[:-1]] == list(range(0, T - 128, 64))


def test_config():
    cfg = QI.config()
    assert cfg["model_family"] == "quickvc" and cfg["gin_channels"] == 256 and cfg["n_mel_channels"] == 80
    assert cfg["filter_length"] == 1280 and cfg["hop_length"] == 320 and cfg["sampling_rate"] == 16000
    c = E.make_c_config(cfg)
    assert c.model_family == 1 and c.spec_channels == 80 and c.use_mel_posterior_encoder == 1
    assert E.make_c_config(C.DEFAULT_CONFIG).model_family == 0


@pytest.mark.parametrize("flags", [{"ms_istft_vits": False, "mb_istft_vits": True}, {"ms_istft_vits": False, "istft_vits": True},
                                   {"ms_istft_vits": False}, {"gin_channels": 192}])
def test_config_refusals(flags):
    j = copy.deepcopy(QI.QUICKVC_JSON)
    j["model"].update(flags)
    with pytest.raises(ValueError):
        C.from_quickvc_json(j)


def test_synthetic_names_and_shapes_match_reference():
    sd = QI.speaker_encoder()
    names = sorted(sd)
    assert names == list(REF["enc_spk_names"])
    assert [",".join(map(str, sd[k].shape)) for k in names] == list(REF["enc_spk_shapes"])


def test_packed_layout():
    cfg = QI.config()
    sd = QI.speaker_encoder()
    blob, manifest = weights.pack_quickvc(weights.fold_weight_norm(sd), cfg)
    ent = {n: (int(o), int(c)) for n, o, c in (l.split() for l in manifest.splitlines())}
    assert set(ent) == {"spk.l%d.%s" % (l, t) for l in range(3) for t in ("ih.w", "ih.b", "hh")} | {"spk.lin.w", "spk.lin.b", "vc.stft", "vc.mel"}
    get = lambda n: blob[ent[n][0]:ent[n][0] + ent[n][1]]
    whh = sd["enc_spk.lstm.weight_hh_l1"].numpy()
    hh = get("spk.l1.hh").reshape(8, 256, 4, 32)                 # [rank][k][gate][unit]
    for rank, k, gate, unit in [(0, 0, 0, 0), (3, 17, 2, 31), (7, 255, 3, 5)]:
        assert hh[rank, k, gate, unit] == whh[gate * 256 + rank * 32 + unit, k]
    b = sd["enc_spk.lstm.bias_ih_l2"].numpy() + sd["enc_spk.lstm.bias_hh_l2"].numpy()
    assert np.array_equal(get("spk.l2.ih.b"), b)
    assert np.array_equal(get("spk.l0.ih.w").reshape(80, 1024), sd["enc_spk.lstm.weight_ih_l0"].numpy().T)
    assert np.array_equal(get("spk.lin.w").reshape(256, 256), sd["enc_spk.linear.weight"].numpy().T)


def test_abi_exports():
    hdr = open(E._build.os.path.join(E._build.HERE, "..", "include", "vtts.h")).read()
    for nm in ("vtts_speaker_embedding", "vtts_speaker_embedding_mel"):
        assert nm in E.EXPORTS and nm + "(" in hdr
