"""GPU tests of StableTTS text-to-mel (vtts_stabletts_synthesise) against the reference's stored durations and mel and the
float64 oracle, of its batch independence, and of what it must leave alone: the decoder called on its own."""
import numpy as np
import pytest
import torch

import stabletts_cfm_inputs as CI
import stabletts_inputs as SI
from oracle import stabletts_oracle as st
from vosk_tts_b200 import weights
from vosk_tts_b200.engine import Engine, VttsError, live_bytes
from vosk_tts_b200.stabletts import StableTTS

pytestmark = pytest.mark.gpu

# max |mel - float64 oracle| and |mel - reference fp32 mel| on the normalised mel: the decoder's budget (test_gpu_stabletts_cfm.py);
# the text side adds gathers and exact copies only.  Measured maxima are in DESIGN.md 4.m.
BUDGET = 1.6e-4
# |fp32 sum of the 50 sigmoids - float64| measured at most 4e-6 (CPU fp32) and below 2e-5 on the GPU: tokens closer than this
# to a rounding boundary are not compared
DUR_MARGIN = 1e-4


@pytest.fixture(scope="module")
def golden():
    return SI.load_golden()


@pytest.fixture(scope="module")
def model():
    cfg = SI.config()
    return cfg, SI.model(cfg)


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "mode1"])
def tts(request, model):
    cfg, sd = model
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=request.param)
    t.precision = request.param
    yield t
    t.close()


@pytest.fixture(scope="module")
def tts0(model):
    cfg, sd = model
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=0)
    yield t
    t.close()


def run(t, case, which=None, **kw):
    name, lens, sids, n, temp, ls, pauses = case
    ins = SI.case_inputs(case)
    idx = list(range(len(lens))) if which is None else [which]
    r = t.synthesise([ins[b][0] for b in idx], [ins[b][1] for b in idx], [sids[b] for b in idx],
                     [ins[b][2] for b in idx] if pauses else None, n_timesteps=n, temperature=temp, length_scale=ls,
                     noise=[ins[b][3] for b in idx], **kw)
    return r


@pytest.mark.parametrize("case", SI.CASES, ids=lambda c: c[0])
def test_fixture_cases(tts, case, golden, model):
    cfg, sd = model
    name, lens, sids, n, temp, ls, pauses = case
    r = run(tts, case, return_prior=True)
    worst, margin = 0.0, 1.0
    for b, (ids, bert, pause, noise) in enumerate(SI.case_inputs(case)):
        k = name + ".%s" + str(b)
        w = golden[k % "w_round"]
        o = st.synthesise(sd, cfg, ids, bert, sids[b], noise, pause if pauses.get(b) else None, n, temp, ls, 0.5, torch.float64, durations=w)
        pre = o["pre_round"].astype(np.float64)
        dist = np.abs(pre - np.floor(pre) - 0.5)
        dist[pre < 1.5] = np.minimum(dist, np.abs(pre - 0.5))[pre < 1.5]
        sure = dist > DUR_MARGIN
        margin = min(margin, float(dist.min()))
        assert np.array_equal(r["durations"][b][sure], w[sure]), (name, b)
        assert sure.all(), "a fixture token sits on a rounding boundary: choose another seed"
        assert r["mel_lengths"][b] == int(golden[k % "mel_lengths"][0])
        for key, ref in (("decoder_outputs", golden[k % "decoder_outputs"]), ("mel", golden[k % "mel"]),
                         ("encoder_outputs", golden[k % "encoder_outputs"])):
            e64 = float(np.abs(r[key][b] - o[key]).max())
            eref = float(np.abs(r[key][b] - ref).max())
            scale = float(sd["mel_std"]) if key == "mel" else 1.0
            worst = max(worst, e64 / scale, eref / scale)
            assert e64 < BUDGET * scale and eref < BUDGET * scale, (name, b, key, e64, eref)
        if pauses.get(b):
            tok = np.repeat(np.arange(len(w)), w)
            hit = pause[tok] > 0
            assert hit.any() and np.array_equal(r["mel"][b][:, hit], np.repeat(r["mel"][b][:, :1], int(hit.sum()), 1))
    print("stabletts %s mode %d: frames %s (mod 4: %s) max err %.2e, smallest rounding margin %.4f"
          % (name, tts.precision, r["mel_lengths"], [v % 4 for v in r["mel_lengths"]], worst, margin))


def test_token_and_mu_rows(tts0, golden, model):
    cfg, sd = model
    case = next(c for c in SI.CASES if c[0] == "pause")
    (ids, bert, pause, noise), = SI.case_inputs(case)
    tts0.engine.debug_flags(1)
    try:
        r = run(tts0, case)
        T = r["mel_lengths"][0]
        x = tts0.engine.debug_read("st_tok_x").reshape(-1, 256)
        mu = tts0.engine.debug_read("st_mu").reshape(-1, 256)
        logw = tts0.engine.debug_read("st_logw")
        mu_dp = tts0.engine.debug_read("st_mu_dp").reshape(-1, 50)
    finally:
        tts0.engine.debug_flags(0)
    o = st.synthesise(sd, cfg, ids, bert, 0, noise, pause, case[3], case[4], case[5], 0.5, torch.float64, durations=golden["pause.w_round0"])
    assert x.shape[0] == ids.shape[1] and np.abs(x.T - o["x"]).max() < 2e-5
    assert np.abs(mu_dp.T - o["mu_dp"]).max() < 2e-4
    free = pause == 0
    assert np.abs(logw[free] - o["logw"][free]).max() < DUR_MARGIN and np.array_equal(logw[~free], pause[~free])
    # the decoder's mu rows: the token rows repeated by the durations, bit for bit, then zero rows up to the padded extent
    tok = np.repeat(np.arange(ids.shape[1]), r["durations"][0])
    assert np.array_equal(mu[:T], x[tok]) and not mu[T:st.ceil4(T)].any()
    assert np.abs(mu[:T].T - o["mu_y"]).max() < 2e-5


def test_alone_equals_batched_and_eager_equals_replay(tts):
    case = next(c for c in SI.CASES if c[0] == "ragged3")
    first = run(tts, case)                      # eager (and the capture behind it)
    r0 = tts.engine.graph_replays()
    again = run(tts, case)
    assert tts.engine.graph_replays() == r0 + 2          # the text phase and the mel phase
    for b in range(3):
        assert np.array_equal(first["mel"][b], again["mel"][b]) and np.array_equal(first["durations"][b], again["durations"][b])
        alone = run(tts, case, which=b)
        assert np.array_equal(alone["durations"][0], first["durations"][b]), b
        assert np.array_equal(alone["mel"][0], first["mel"][b]), b


def test_philox_noise_is_seeded_and_needs_no_caller_noise(tts0):
    case = next(c for c in SI.CASES if c[0] == "short")
    (ids, bert, pause, noise), = SI.case_inputs(case)
    a = tts0.synthesise(ids, bert, 1, seed=7, n_timesteps=2)
    b = tts0.synthesise(ids, bert, 1, seed=7, n_timesteps=2)
    c = tts0.synthesise(ids, bert, 1, seed=8, n_timesteps=2)
    assert np.array_equal(a["mel"], b["mel"]) and not np.array_equal(a["mel"], c["mel"]) and np.isfinite(a["mel"]).all()


# SHA-1 of vtts_cfm_decode's mel on the decoder fixture's ragged batch (guided, 10 steps, precision 0; H100), taken from the code
# before the decoder learnt extents: with extent == length it must not change by a bit
CFM_SHA1 = {"ragged3": "c0e4f6aa1ef16da04a9f4c88df9b98c6f2e5a648"}


def test_decoder_alone_is_unchanged():
    import hashlib
    cfg = CI.config()
    blob, man = weights.pack_stabletts_cfm(CI.model(cfg), cfg)
    e = Engine(cfg, blob, man, device=0, precision=0)
    try:
        for name, want in CFM_SHA1.items():
            case = next(c for c in CI.CASES if c[0] == name)
            ins = CI.case_inputs(case)
            mel, _ = e.cfm_decode([m.T for m, _ in ins], case[5], n_timesteps=case[2], temperature=case[4], guidance_scale=case[3],
                                  noise=[z.T for _, z in ins])
            got = hashlib.sha1(np.ascontiguousarray(mel).tobytes()).hexdigest()
            print("cfm_decode %s sha1 %s" % (name, got))
            assert got == want, name
    finally:
        e.close()


def test_refusals(tts0, model):
    cfg, sd = model
    case = next(c for c in SI.CASES if c[0] == "short")
    (ids, bert, pause, noise), = SI.case_inputs(case)
    e = tts0.engine
    feats = np.ascontiguousarray(bert.T)[None]
    with pytest.raises(VttsError, match="token id out of range"):
        e.stabletts_synthesise(np.where(ids == ids[1, 2], cfg["n_vocab"], ids)[None], feats, 0)
    with pytest.raises(VttsError, match="speaker id out of range"):
        e.stabletts_synthesise(ids[None], feats, 2)
    with pytest.raises(VttsError, match="pause durations"):
        e.stabletts_synthesise(ids[None], feats, 0, pause=np.full((1, 9), -1.0, np.float32))
    with pytest.raises(VttsError, match="length_scale"):
        e.stabletts_synthesise(ids[None], feats, 0, length_scale=0.0)
    with pytest.raises(VttsError, match="mel_ld is smaller") as ex:
        e.stabletts_synthesise(ids[None], feats, 1, mel_frames=5)
    assert ex.value.code == -4
    with pytest.raises(VttsError, match="noise has fewer frames") as ex:
        e.stabletts_synthesise(ids[None], feats, 1, noise=np.zeros((1, 47, 80), np.float32))       # 47 frames need 48 columns
    assert ex.value.code == -4
    # a decoder-only blob refuses the call and says why
    dcfg = CI.config()
    blob, man = weights.pack_stabletts_cfm(sd, dcfg)
    d = Engine(dict(dcfg, n_streams=5, bert_dim=768, dur_channels=50), blob, man, device=0, precision=0)
    try:
        with pytest.raises(VttsError, match="flow-matching decoder only") as ex:
            d.stabletts_synthesise(ids[None], feats, 0)
        assert ex.value.code == -1
    finally:
        d.close()


def test_memory_returns_to_baseline(model):
    cfg, sd = model
    base = live_bytes()
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=0)
    run(t, next(c for c in SI.CASES if c[0] == "ragged3"), return_prior=True)
    assert live_bytes()[0] > base[0]
    t.close()
    assert live_bytes() == base
