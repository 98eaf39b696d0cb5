"""GPU tests of the StableTTS vocoder (vtts_hifigan_vocode) and of text-to-waveform (vtts_stabletts_synthesise_wav): against
the reference's stored waveforms and the float64 oracle in precision modes 0 and 1, batch independence and graph replay, and
the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import hifigan_inputs as HI
import stabletts_inputs as SI
from oracle import hifigan_oracle as O
from vosk_tts_b200 import config, synthetic, weights
from vosk_tts_b200.engine import Engine, live_bytes
from vosk_tts_b200.stabletts import StableTTS

pytestmark = pytest.mark.gpu

# max |wav - float64 oracle| and |wav - reference fp32 wav| on waveforms of max |wav| 0.3-0.9 (tests/hifigan_inputs.py mels):
# fp32 FFMA (mode 0) and split-bf16 tensor cores (mode 1).  Measured maxima are in DESIGN.md 4.n.
BUDGET = {0: 2e-5, 1: 2e-4}
ERR_INVALID, ERR_CAPACITY = -1, -4


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(HI.GOLDEN))


@pytest.fixture(scope="module")
def sd():
    return HI.folded()


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "mode1"])
def tts(request):
    cfg = SI.config()
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, SI.model(cfg), device=0, precision=request.param, vocoder=HI.checkpoint())
    t.precision = request.param
    yield t
    t.close()


@pytest.mark.parametrize("case", HI.CASES, ids=lambda c: c[0])
def test_vocode_fixture_cases(tts, case, golden, sd):
    mels = HI.case_mels(case)
    wavs = tts.vocode(mels)
    for b, (m, w) in enumerate(zip(mels, wavs)):
        ref = golden["%s.wav%d" % (case[0], b)]
        o64 = O.generator(sd, HI.config(), m, torch.float64).numpy()
        assert w.shape == (256 * m.shape[1],)
        e_ref, e64 = float(np.abs(w - ref).max()), float(np.abs(w - o64).max())
        print("%s[%d] mode %d: max|wav| %.3f  |wav - ref| %.2e  |wav - f64| %.2e" % (case[0], b, tts.precision, np.abs(ref).max(), e_ref, e64))
        assert e_ref < BUDGET[tts.precision] and e64 < BUDGET[tts.precision]


def test_wav_lengths_and_padding(tts):
    mels = [HI.mel("len", b, T) for b, T in enumerate([3, 17, 9])]
    wav, wl = tts.engine.hifigan_vocode([np.ascontiguousarray(m.T) for m in mels])
    assert list(wl) == [256 * 3, 256 * 17, 256 * 9] and wav.shape == (3, 256 * 17)
    assert not wav[0, 256 * 3:].any() and not wav[2, 256 * 9:].any()


def test_batch_and_replay(tts):
    mels = [HI.mel("batch", b, T) for b, T in enumerate([40, 7, 133, 64])]
    first = tts.vocode(mels)
    again = tts.vocode(mels)                               # the bucket's graph replays
    for a, b in zip(first, again):
        assert np.array_equal(a, b)
    alone = [tts.vocode(m) for m in mels]
    diff = max(float(np.abs(a - b).max()) for a, b in zip(first, alone))
    print("mode %d: max |batched - alone| %.2e" % (tts.precision, diff))
    if tts.precision == 0:
        assert diff == 0.0
    else:                  # the tensor-core split-K plans follow the batch shape (DESIGN.md 4.n)
        assert diff < BUDGET[1]


def test_text_fixture_cases(tts, golden):
    st = SI.load_golden()
    for key in HI.TEXT_CASES:
        w = tts.vocode(st[key])
        ref = golden["text." + key + ".wav"]
        err = float(np.abs(w - ref).max())
        print("text %s mode %d: |wav - ref| %.2e" % (key, tts.precision, err))
        assert err < BUDGET[tts.precision]


@pytest.mark.parametrize("which", [None, 2], ids=["ragged3", "alone"])
def test_synthesise_wav_equals_synthesise_then_vocode(tts, which):
    case = [c for c in SI.CASES if c[0] == "ragged3"][0]
    name, lens, sids, n, temp, ls, pauses = case
    ins = SI.case_inputs(case)
    idx = list(range(len(lens))) if which is None else [which]
    kw = dict(n_timesteps=n, temperature=temp, length_scale=ls, noise=[ins[b][3] for b in idx])
    args = ([ins[b][0] for b in idx], [ins[b][1] for b in idx], [sids[b] for b in idx], [ins[b][2] for b in idx])
    r = tts.synthesise(*args, return_wav=True, **kw)
    r0 = tts.synthesise(*args, **kw)
    voc = tts.vocode(r0["mel"])
    for b in range(len(idx)):
        assert np.array_equal(r["mel"][b], r0["mel"][b]) and np.array_equal(r["decoder_outputs"][b], r0["decoder_outputs"][b])
        assert r["wav_lengths"][b] == 256 * r["mel_lengths"][b] == r["wav"][b].size
        d = float(np.abs(r["wav"][b] - voc[b]).max())
        print("mode %d utterance %d: |synthesise_wav - vocode(synthesise)| %.2e" % (tts.precision, b, d))
        if tts.precision == 0:
            assert d == 0.0
        else:
            assert d < BUDGET[1]
    again = tts.synthesise(*args, return_wav=True, **kw)          # replay of the mel phase's graph with the vocoder
    assert all(np.array_equal(a, b) for a, b in zip(again["wav"], r["wav"]))


def _synth_wav_raw(t, wav_ld):
    cfg = t.cfg
    ids, bert, pause, noise = SI.inputs("cap", 9)
    B, S, T = 1, ids.shape[0], ids.shape[1]
    ids = np.ascontiguousarray(ids[None], np.int64)
    bert = np.ascontiguousarray(bert.T[None], np.float32)
    lens, sid = np.array([T], np.int64), np.array([0], np.int64)
    mel_len = np.zeros(1, np.int64)
    wav = np.zeros((1, max(wav_ld, 1)), np.float32)
    wl = np.zeros(1, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = t.engine.lib.vtts_stabletts_synthesise_wav(t.engine.h, p(ids), p(lens), B, T, p(bert), None, p(sid), 2, 1.0, 1.0, 0.5, None, 0, 0,
                                                    None, 0, p(mel_len), None, None, 1, p(wav), wav_ld, p(wl))
    return rc, int(mel_len[0])


def test_refusals():
    cfg = SI.config()
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, SI.model(cfg), device=0, precision=0)          # no vocoder
    try:
        m = np.ascontiguousarray(HI.mel("x", 0, 5).T)
        L = np.array([5], np.int64)
        wav, wl = np.zeros((1, 2048), np.float32), np.zeros(1, np.int64)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert t.engine.lib.vtts_hifigan_vocode(t.engine.h, p(m), p(L), 1, 5, p(wav), 2048, p(wl)) == ERR_INVALID
        assert _synth_wav_raw(t, 1 << 20)[0] == ERR_INVALID
    finally:
        t.close()
    vc = dict(config.DEFAULT_CONFIG)
    blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(vc)), vc)
    e = Engine(vc, blob, man, device=0, precision=0)
    try:
        assert e.lib.vtts_hifigan_vocode(e.h, p(m), p(L), 1, 5, p(wav), 2048, p(wl)) == ERR_INVALID
        assert "StableTTS" in e.lib.vtts_last_error(e.h).decode()
    finally:
        e.close()


def test_small_wav_ld_returns_capacity_with_lengths(tts):
    rc, frames = _synth_wav_raw(tts, 1)
    assert rc == ERR_CAPACITY and frames >= 1
    rc2, frames2 = _synth_wav_raw(tts, 256 * frames)
    assert rc2 == 0 and frames2 == frames


def test_live_bytes_back_to_baseline():
    cfg = SI.config()
    base = live_bytes()
    for p in (0, 1):
        t = StableTTS({"n_vocab": cfg["n_vocab"]}, SI.model(cfg), device=0, precision=p, vocoder=HI.checkpoint())
        t.vocode([HI.mel("lb", b, T) for b, T in enumerate([30, 11])])
        t.synthesise(SI.inputs("lb", 6)[0], SI.inputs("lb", 6)[1], 0, return_wav=True)
        t.close()
        assert live_bytes() == base
