"""GPT-SoVITS prompt tokens on the GPU (vtts_sovits_semantic / vtts_sovits_latent, gpt_sovits.SemanticEncoder) against the
reference's codes (tests/golden/ref_sovits_semantic.npz: transformers' HubertModel and the reference's
SynthesizerTrn.extract_latent, in float64), in precision modes 0 and 1."""
import numpy as np
import pytest
import torch

import sovits_inputs as SI
from oracle import sovits_oracle as O

pytestmark = pytest.mark.gpu

_ENC = {}
U = 2.0 ** -24                      # fp32 unit roundoff


def _fixture():
    return np.load(SI.FIXTURE)


def _enc(precision, s2_config=SI.S2_32K, ties=False):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.gpt_sovits import SemanticEncoder
    key = (precision, s2_config["data"]["sampling_rate"], ties)
    if key not in _ENC:
        sd = SI.s2_ties() if ties else SI.s2()
        _ENC[key] = SemanticEncoder((sd, SI.cfg(s2_config)), (SI.hubert(), SI.cv()), device=0, precision=precision)
    return _ENC[key]


def teardown_module(module):
    for e in _ENC.values():
        e.close()
    _ENC.clear()


def _bound(x, sd):
    """The fp32 error bound of every row's score difference (best minus any other), by the probabilistic rounding-error bound
    (Higham and Mary, 2019): a dot product of n terms within sqrt(n) u of the sum of its terms' magnitudes, for the
    projection's 2 H terms and the scores' H.  (The worst-case n u is some 10^4 times the error the kernels make here.)"""
    g = lambda k: sd[k].double().numpy()
    w, b, E = g("ssl_proj.weight"), g("ssl_proj.bias"), g("quantizer.vq.layers.0._codebook.embed")
    H = w.shape[0]
    T2 = x.shape[0] // 2
    a = np.abs(np.asarray(x, np.float64)[:2 * T2]).reshape(T2, 2, H)
    p = O.project(x, w, b)
    ep = np.sqrt(2 * H + 1) * U * (a[:, 0] @ np.abs(w[:, :, 0]).T + a[:, 1] @ np.abs(w[:, :, 1]).T + np.abs(b))
    es = 2 * ep @ np.abs(E).T + np.sqrt(H + 1) * U * (np.abs(p) @ np.abs(2 * E).T + (E * E).sum(1))
    return 2 * es.max(1)


@pytest.mark.parametrize("precision", [0, 1])
def test_tail_alone(precision):
    """extract_latent on HuBERT-like rows: the float64 argmax on every row whose margin exceeds the fp32 error bound, and the
    reference's codes on the rows of the fixture."""
    f = _fixture()
    enc = _enc(precision)
    sd = SI.s2()
    for name in ("f_odd", "f_even"):
        x = SI.feats(name)
        codes = enc.extract_latent(x.T[None])
        assert codes.shape == (1, 1, x.shape[0] // 2) and codes.dtype == np.int64
        ref = f[name + "/codes"]
        keep = f[name + "/margin"] > _bound(x, sd)
        print("mode %d, %s: %d of %d rows above the bound" % (precision, name, keep.sum(), keep.size))
        assert keep.mean() >= 0.5 and np.array_equal(codes[0, 0][keep], ref[keep])


@pytest.mark.parametrize("precision", [0, 1])
def test_ties_give_the_lowest_index(precision):
    """Duplicated codewords and a row equidistant from two codewords: exact ties, where the reference's (lowest) index is
    the ground truth, on every row."""
    f = _fixture()
    enc = _enc(precision, ties=True)
    codes = enc.extract_latent(SI.feats("ties").T[None])[0, 0]
    ref = f["ties/codes"]
    assert (f["ties/margin"] == 0).sum() >= 3
    assert ref[SI.ZERO_ROWS[0] // 2] == min(SI.TIE_PAIR)
    assert np.array_equal(codes, ref), (codes, ref)


def _score_rounding(proj, E, codes):
    """The probabilistic bound (as _bound) on the fp32 rounding of the scores of `codes`, per row: H products and the bias."""
    H = proj.shape[1]
    Ec = E[codes]
    return np.sqrt(H + 1) * U * ((np.abs(proj) * np.abs(2 * Ec)).sum(1) + (Ec * Ec).sum(1))


@pytest.mark.parametrize("precision", [0, 1])
def test_waveform_matches_reference(precision):
    """Recording in, codes out.  The reference's code on every frame whose margin exceeds 4x the score error measured in the
    same case plus the fp32 rounding of the two decisive scores; at least 95 % of all frames equal.  The measured error is that
    of the decisive difference: the float64 scores, from the engine's projected rows (which carry HuBERT's error), of the
    reference's code minus its runner-up's, against the reference's margin.  (The scores themselves carry an error common to
    all codes that no argmax sees.)  With this seeded HuBERT neighbouring frames are close, so a frame's margin is often near
    the rounding of scores some 10^3 larger: at least half the frames must be checked."""
    f = _fixture()
    E = SI.s2()["quantizer.vq.layers.0._codebook.embed"].double().numpy()
    for name, (n, seed, s2c) in SI.WAVE.items():
        enc = _enc(precision, s2c)
        enc.engine.debug_flags(1)
        try:
            p, = enc.prompts([SI.clip(name)])
            proj = enc.engine.debug_read("sv_proj").reshape(-1, 768)[: p.size].astype(np.float64)
        finally:
            enc.engine.debug_flags(0)
        ref, margin, second = f[name + "/codes"], f[name + "/margin"], f[name + "/second"]
        assert p.shape == ref.shape
        s = O.scores(proj, E)
        t = np.arange(ref.size)
        err = float(np.abs(s[t, ref] - s[t, second] - margin).max())
        keep = margin > 4 * err + _score_rounding(proj, E, ref) + _score_rounding(proj, E, second)
        agree = float((p == ref).mean())
        print("mode %d, %s: %d codes (%d distinct), score error %.3g, %d checked, %.1f %% equal overall"
              % (precision, name, p.size, int(f[name + "/distinct"]), err, keep.sum(), 100 * agree))
        assert keep.mean() >= 0.5 and agree >= 0.95, (keep.mean(), agree)
        assert np.array_equal(p[keep], ref[keep])


@pytest.mark.parametrize("precision", [0, 1])
def test_batch_equals_single(precision):
    """A ragged, shuffled batch of 8 gives each clip's codes bit for bit as alone."""
    enc = _enc(precision)
    rng = np.random.default_rng(9)
    ns = [48000, 320000, 52345, 160000, 48001, 99999, 200000, 70000]
    clips = [SI.CI.speech(int(n), 300 + i) for i, n in enumerate(rng.permutation(ns))]
    batch = enc.prompts(clips)
    for x, c in zip(clips, batch):
        one, = enc.prompts([x])
        assert np.array_equal(one, c)


def test_resampling():
    """A 44.1 kHz recording through prompts(..., sampling_rate=44100) equals Engine.resample then prompts at 16 kHz."""
    enc = _enc(1)
    x = SI.CI.speech(44100 * 4, 17)
    a, = enc.prompts([x], sampling_rate=44100)
    y, = enc.engine.resample(x, 44100, 16000)
    b, = enc.prompts([y])
    assert np.array_equal(a, b) and a.size > 0


def test_range_check():
    enc = _enc(0)
    for n in (47999, 320001):
        with pytest.raises(ValueError, match="Prompt audio length must be longer than 3 seconds and shorter than 20 seconds!"):
            enc.prompts([np.zeros(n, np.float32)])


def test_family_guards():
    """The SoVITS entry points refuse a text-to-semantic engine; a SoVITS engine refuses codes_ld below a clip's code count."""
    import ctypes as C
    import t2s_inputs as T2I
    from vosk_tts_b200.gpt_sovits import Text2Semantic
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    wav, lens = np.zeros((1, 48000), np.float32), np.array([48000], np.int64)
    codes, n = np.zeros((1, 100), np.int64), np.zeros(1, np.int64)
    t2s = Text2Semantic(T2I.model(), device=0, precision=0)
    try:
        e = t2s.engine
        for fn in (e.lib.vtts_sovits_semantic, e.lib.vtts_sovits_latent):
            assert fn(e.h, p(wav), p(lens), 1, 48000, p(codes), 100, p(n)) == -1
            assert "GPT-SoVITS SoVITS" in e.lib.vtts_last_error(e.h).decode()
    finally:
        t2s.close()
    e = _enc(0).engine
    assert e.lib.vtts_sovits_semantic(e.h, p(wav), p(lens), 1, 48000, p(codes), 10, p(n)) == -4      # 74 codes > 10


def test_chaining_into_text2semantic():
    """Codes the engine gives equal to the reference's (extract_latent of "f_even", checked whole) prompt
    Text2Semantic.decode to the same tokens as the reference's codes, for a fixed q; and prompts()'s tokens go straight in."""
    import t2s_inputs as T2I
    from vosk_tts_b200.gpt_sovits import Text2Semantic
    f = _fixture()
    enc = _enc(1)
    mine = enc.extract_latent(SI.feats("f_even").T[None])[0, 0]
    assert np.array_equal(mine, f["f_even/codes"])
    sd, cfg = T2I.model(T2I.UPSTREAM, seed=7)
    t2s = Text2Semantic((sd, cfg), device=0, precision=1)
    try:
        ph = T2I.phones(cfg, 20, 3)
        q = T2I.q_draws(cfg, 60, 4)[None]
        a, _ = t2s.decode([ph], prompts=[mine], q=q, step_cap=50)
        b, _ = t2s.decode([ph], prompts=[f["f_even/codes"]], q=q, step_cap=50)
        assert np.array_equal(a[0], b[0]) and a[0].size > mine.size
        pr = enc.prompts([SI.clip("w48000")])
        c, _ = t2s.decode([ph], prompts=pr, q=q, step_cap=50)
        assert np.array_equal(c[0][: pr[0].size], pr[0])
    finally:
        t2s.close()
