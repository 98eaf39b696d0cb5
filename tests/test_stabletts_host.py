"""Host-side tests of StableTTS text-to-mel: the oracle restatement (with the padded extent synthesise gives the decoder)
against the reference's stored durations and mel, the duration rule's corner cases, the weight packing and the refusals
that need no device."""
import numpy as np
import pytest
import torch

import stabletts_inputs as SI
from oracle import stabletts_cfm_oracle as so
from oracle import stabletts_oracle as st
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import VttsConfig, make_c_config
from vosk_tts_b200.stabletts import StableTTS


@pytest.fixture(scope="module")
def golden():
    return SI.load_golden()


@pytest.fixture(scope="module")
def model():
    cfg = SI.config()
    return cfg, SI.model(cfg)


def test_fixture_holds_the_seeded_inputs_and_every_residue(golden):
    assert int(golden["seed"]) == SI.SEED and list(golden["cases"]) == [c[0] for c in SI.CASES]
    residues = set()
    for case in SI.CASES:
        for b, (ids, bert, pause, noise) in enumerate(SI.case_inputs(case)):
            k = case[0] + ".%s" + str(b)
            assert np.array_equal(golden[k % "ids"], ids) and np.array_equal(golden[k % "pause"], pause)
            assert str(golden[k % "bert_sha1"]) == SI.sha1(bert) and str(golden[k % "noise_sha1"]) == SI.sha1(noise)
            T = int(golden[k % "mel_lengths"][0])
            assert st.ceil4(T) <= SI.MAX_FRAMES          # the reference drew the noise's first ceil4(T) columns
            assert int(golden[k % "w_round"].sum()) == T and golden[k % "mel"].shape == golden[k % "encoder_outputs"].shape == (80, T)
            residues.add(T % 4)
    assert residues == {0, 1, 2, 3}


SMALL = [c for c in SI.CASES if c[0] in ("t1", "short_n1", "pause", "slow", "mod_a", "mod_b", "mod_c", "mod_d")]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c[0])
def test_oracle_equals_reference(case, golden, model):
    """fp32: the reference's durations exactly, its mel within 2e-5 (6.3e-6 measured at most); float64 on the reference's
    durations (what the GPU tests compare against): within the fp32 rounding the reference itself carries (2.5e-5 measured)."""
    cfg, sd = model
    name, lens, sids, n, temp, ls, pauses = case
    for b, (ids, bert, pause, noise) in enumerate(SI.case_inputs(case)):
        k = name + ".%s" + str(b)
        p = pause if pauses.get(b) else None
        r32 = st.synthesise(sd, cfg, ids, bert, sids[b], noise, p, n, temp, ls, 0.5, torch.float32)
        assert np.array_equal(r32["durations"], golden[k % "w_round"])
        assert np.abs(r32["decoder_outputs"] - golden[k % "decoder_outputs"]).max() < 2e-5
        assert np.abs(r32["mel"] - golden[k % "mel"]).max() < 5e-5
        assert np.abs(r32["encoder_outputs"] - golden[k % "encoder_outputs"]).max() < 2e-5
        r64 = st.synthesise(sd, cfg, ids, bert, sids[b], noise, p, n, temp, ls, 0.5, torch.float64, durations=golden[k % "w_round"])
        assert np.abs(r64["decoder_outputs"] - golden[k % "decoder_outputs"]).max() < 6e-5


def test_the_padded_extent_matters_and_only_off_multiples_of_four(golden, model):
    """Decoding on the utterance's own T columns (what vtts_cfm_decode does) is the reference only when T % 4 == 0: otherwise
    the padded columns' noise and cond_proj reach every frame through the last long-skip conv and the attention."""
    cfg, sd = model
    for name, same in (("mod_a", True), ("mod_b", False)):
        case = next(c for c in SI.CASES if c[0] == name)
        (ids, bert, pause, noise), = SI.case_inputs(case)
        r = st.synthesise(sd, cfg, ids, bert, 0, noise, pause, 10, 1.0, 1.0, 0.5, torch.float32)
        T = r["mu_y"].shape[1]
        own = so.decode(sd, cfg, r["mu_y"], 0, noise[:, :T], 10, 1.0, 0.5, torch.float32)
        pad = st.decode(sd, cfg, r["mu_y"], 0, noise, None, 10, 1.0, 0.5, torch.float32)
        assert np.array_equal(st.decode(sd, cfg, r["mu_y"], 0, noise, T, 10, 1.0, 0.5, torch.float32), own)
        assert (np.abs(own - pad).max() == 0) if same else (np.abs(own - pad).max() > 0.1)


def test_duration_rule_corner_cases():
    logw = np.array([0.5, 1.5, 2.5, 3.5, 0.2, 7.49, 4.0, 4.0], np.float32)
    w, _ = st.duration_rule(logw, None, 1.0)
    assert list(w) == [1, 2, 2, 4, 1, 7, 4, 4]            # half to even, then at least 1 (0.5 -> 0 -> 1)
    pause = np.array([0, 6.5, 0, 0.25, 0, 0, 3.0, 0], np.float32)
    w, pre = st.duration_rule(logw, pause, 1.0)
    assert list(w) == [1, 6, 2, 1, 1, 7, 3, 4]            # the pause replaces the prediction where it is not 0: 6.5 -> 6, 0.25 -> 1
    w, pre = st.duration_rule(logw, pause, 1.5)
    assert list(w) == [1, 10, 4, 1, 1, 11, 4, 6]          # length_scale applies to pauses too: 9.75 -> 10, 0.375 -> 0 -> 1, 4.5 -> 4
    assert pre.dtype == np.float32


def _tensors(blob, man):
    out = {}
    for line in man.strip().split("\n"):
        name, off, n = line.split()
        out[name] = blob[int(off):int(off) + int(n)]
    return out


def test_packing_round_trips_and_shares_the_decoder(model):
    cfg, sd = model
    blob, man = weights.pack_stabletts(sd, cfg)
    t = _tensors(blob, man)
    H, F, G = cfg["enc_hidden_channels"], cfg["enc_filter_channels"], cfg["spk_emb_dim"]
    assert np.array_equal(t["st.enc.emb"].reshape(-1, 160), sd["encoder.emb.weight"].numpy())
    assert np.array_equal(t["st.enc.punc"].reshape(-1, 16), sd["encoder.punc_emb.weight"].numpy())
    assert np.array_equal(t["st.enc.bert.w"].reshape(32, 768), sd["encoder.bert_proj.1.weight"].numpy())
    assert np.array_equal(t["st.dur_spk_emb"].reshape(-1, G), sd["dur_spk_emb.weight"].numpy())
    w = sd["encoder.dp_encoder.encoder.2.mlp.conv_1.weight"].numpy()
    assert np.array_equal(t["st.enc.dp.l2.ffn1.w"].reshape(3, H, F), np.transpose(w, (2, 1, 0)))
    assert np.array_equal(t["st.enc.mel.ada.w2"].reshape(4, 6 * H, H)[3], sd["encoder.encoder.encoder.3.adaLN_modulation.2.weight"].numpy())
    p = t["st.enc.dp.proj.w"].reshape(1, H, 52)[0]        # 50 output channels padded to the FFMA layout's multiple of 4
    assert np.array_equal(p[:, :50], sd["encoder.dp_encoder.proj.weight"].numpy()[:, :, 0].T) and not p[:, 50:].any()
    assert all(int(line.split()[1]) % 64 == 0 for line in man.strip().split("\n"))
    dec = _tensors(*weights.pack_stabletts_cfm(sd, C.stabletts_cfm_config()))
    assert all(np.array_equal(t[k], v) for k, v in dec.items()) and "st.enc.emb" not in dec


def test_packing_and_config_refusals(model):
    cfg, sd = model
    with pytest.raises(ValueError, match="needs config.stabletts_config"):
        weights.pack_stabletts(sd, C.stabletts_cfm_config())
    bad = dict(sd)
    bad["encoder.bert_proj.1.weight"] = sd["encoder.bert_proj.1.weight"][:, :-1]
    with pytest.raises(ValueError, match="bert_proj.1.weight has shape"):
        weights.pack_stabletts(bad, cfg)
    with pytest.raises(KeyError):
        weights.pack_stabletts(synthetic.make_random_stabletts_cfm(cfg, 1), cfg)
    with pytest.raises(ValueError, match="must equal cond_channels"):
        C.stabletts_config({"bert_proj_dim": 48})
    with pytest.raises(ValueError, match="head width enc_hidden_channels"):
        C.stabletts_config({"enc_n_heads": 16})
    with pytest.raises(ValueError, match="bert_dim and dur_channels"):
        C.stabletts_config({"bert_dim": 2048})


def test_c_config_carries_the_text_fields_behind_the_decoder_fields():
    names = [f[0] for f in VttsConfig._fields_]
    assert names.index("st_n_vocab") == names.index("st_n_spks") + 1 and names.index("cv_layers") == names.index("st_dur_channels") + 1
    c = make_c_config(SI.config())
    assert (c.st_n_vocab, c.st_streams, c.st_emb_dim, c.st_punc_dim, c.st_bert_dim, c.st_bert_proj) == (120, 5, 160, 16, 768, 32)
    assert (c.st_enc_hidden, c.st_enc_filter, c.st_enc_layers, c.st_enc_heads, c.st_enc_kernel, c.st_dur_channels) == (256, 1024, 4, 4, 3, 50)
    assert make_c_config(C.stabletts_cfm_config()).st_enc_layers == 0          # a decoder-only engine


def test_synthetic_encoder_has_live_gates_and_is_seeded(model):
    cfg, sd = model
    assert float(sd["encoder.dp_encoder.encoder.0.adaLN_modulation.2.weight"].abs().max()) > 0
    again = synthetic.make_random_stabletts(cfg, SI.SEED)
    assert all(torch.equal(sd[k], again[k]) for k in sd)


def test_scales_follow_the_exported_forward():
    assert StableTTS.from_scales([0.667, 1.2, 0.7]) == {"temperature": 0.667, "length_scale": 1.2}
