"""GPU tests of precision mode 2 on StableTTS engines: the mel phase's convs and attention on the tensor cores (split-bf16
wgmma), against the float64 oracle and the reference's fp32 mel, with the text phase left exactly as in mode 1; text to
waveform, the voice loaded from its exported graph, the word-piece path, and each plane-writing kernel on its own rows."""
import os

import numpy as np
import pytest
import torch

import bert_inputs as BI
import hifigan_inputs as HI
import stabletts_cfm_inputs as CI
import stabletts_inputs as SI
import stabletts_onnx_inputs as OI
from oracle import stabletts_cfm_oracle as so
from oracle import stabletts_oracle as st
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine, live_bytes
from vosk_tts_b200.stabletts import StableTTS

pytestmark = pytest.mark.gpu

# max |mel - float64 oracle| and |mel - reference fp32 mel| on the normalised mel (|mel| up to 10) in mode 2.  Measured on an
# H100 80GB HBM3 at 700 W: 2.4e-4 over the fixture cases, 3.3e-4 at 3000 frames (DESIGN.md 4.r); the budget is about 4x that.
BUDGET = 1.3e-3
# max |wav - reference| of text to waveform (ref_hifigan.npz: the reference's vocoder on the reference's mel): mode 2's mel
# error through the vocoder.  Measured on an H100 80GB HBM3 at 700 W: 2.2e-5 (DESIGN.md 4.r); the budget is about 4x that.
WAV_BUDGET = 1e-4


@pytest.fixture(scope="module")
def cfm():
    cfg = CI.config()
    sd = CI.model(cfg)
    return cfg, sd


@pytest.fixture(scope="module")
def eng2(cfm):
    cfg, sd = cfm
    blob, man = weights.pack_stabletts_cfm(sd, cfg, precision=2)
    e = Engine(cfg, blob, man, device=0, precision=2)
    yield e
    e.close()


def decode(e, case):
    name, lens, n, s, temp, sids = case
    ins = CI.case_inputs(case)
    mel, ln = e.cfm_decode([m.T for m, _ in ins], sids, n_timesteps=n, temperature=temp, guidance_scale=s, noise=[z.T for _, z in ins])
    assert list(ln) == lens
    return [mel[b, :lens[b]].T for b in range(len(lens))]


@pytest.mark.parametrize("case", CI.CASES, ids=lambda c: c[0])
def test_cfm_fixture_cases(eng2, cfm, case):
    cfg, sd = cfm
    golden = np.load(CI.GOLDEN)
    name, lens, n, s, temp, sids = case
    out = decode(eng2, case)
    worst = 0.0
    for b, (mu, nz) in enumerate(CI.case_inputs(case)):
        o64 = so.decode(sd, cfg, mu, sids[b], nz, n, temp, s, torch.float64)
        e64 = float(np.abs(out[b] - o64).max())
        eref = float(np.abs(out[b] - golden["%s.mel%d" % (name, b)]).max())
        worst = max(worst, e64, eref)
        assert e64 < BUDGET and eref < BUDGET, (name, b, e64, eref)
    print("cfm %s mode 2: max err %.2e" % (name, worst))


def test_cfm_alone_equals_batched_and_eager_equals_replay(eng2):
    case = CI.CASES[5]
    first = decode(eng2, case)                   # eager (and the capture behind it)
    r0 = eng2.graph_replays()
    again = decode(eng2, case)
    assert eng2.graph_replays() == r0 + 1
    for a, b in zip(first, again):
        assert np.array_equal(a, b)
    name, lens, n, s, temp, sids = case
    for b in range(len(lens)):
        mu, nz = CI.inputs(name + str(b), lens[b])
        mel, _ = eng2.cfm_decode(mu.T, sids[b], n_timesteps=n, temperature=temp, guidance_scale=s, noise=nz.T)
        assert np.array_equal(mel[0].T, first[b]), b


def test_cfm_long_utterance(eng2, cfm):
    """3000 frames: many row tiles per conv, attention over many key tiles."""
    cfg, sd = cfm
    mu, nz = CI.inputs("long3000", 3000)
    mel, _ = eng2.cfm_decode(mu.T, 1, n_timesteps=2, guidance_scale=0.5, noise=nz.T)
    err = float(np.abs(mel[0].T - so.decode(sd, cfg, mu, 1, nz, 2, 1.0, 0.5, torch.float64)).max())
    print("cfm 3000 frames mode 2: max err %.2e" % err)
    assert err < BUDGET


@pytest.mark.parametrize("over", [{"filter_channels": 720}, {"hidden_channels": 96, "n_heads": 3}], ids=["filter720", "hidden96"])
def test_mixed_pipes_where_widths_fall_back_to_ffma(over):
    """filter 720: cond_proj and the FFN convs on the FFMA pipe beside tensor-core qkv / o / long skips and attention.
    hidden 96 (3 heads of 32): every conv that reads or writes the hidden width on the FFMA pipe, the qkv conv's epilogue
    writing the planes the tensor-core attention reads, beside cond_proj's first two convs on the tensor cores."""
    cfg = C.stabletts_cfm_config(over)
    sd = synthetic.make_random_stabletts_cfm(cfg, 77)
    blob, man = weights.pack_stabletts_cfm(sd, cfg, precision=2)
    e = Engine(cfg, blob, man, device=0, precision=2)
    try:
        mu, nz = CI.inputs("mixed", 45, cfg)
        mel, _ = e.cfm_decode(mu.T, 1, n_timesteps=3, guidance_scale=0.5, noise=nz.T)
        err = float(np.abs(mel[0].T - so.decode(sd, cfg, mu, 1, nz, 3, 1.0, 0.5, torch.float64)).max())
        print("cfm %s mode 2: max err %.2e" % (over, err))
        assert err < BUDGET
    finally:
        e.close()


def test_blob_without_planes_is_refused(cfm):
    cfg, sd = cfm
    blob, man = weights.pack_stabletts_cfm(sd, cfg)
    with pytest.raises(Exception, match="tensor-core weights"):
        Engine(cfg, blob, man, device=0, precision=2)


@pytest.fixture(scope="module")
def text():
    cfg = SI.config()
    sd = SI.model(cfg)
    t1 = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=1)
    t2 = StableTTS({"n_vocab": cfg["n_vocab"]}, sd, device=0, precision=2)
    yield cfg, sd, t1, t2
    t1.close()
    t2.close()


def synth(t, case, which=None):
    name, lens, sids, n, temp, ls, pauses = case
    ins = SI.case_inputs(case)
    idx = list(range(len(lens))) if which is None else [which]
    return t.synthesise([ins[b][0] for b in idx], [ins[b][1] for b in idx], [sids[b] for b in idx],
                        [ins[b][2] for b in idx] if pauses else None, n_timesteps=n, temperature=temp, length_scale=ls,
                        noise=[ins[b][3] for b in idx])


@pytest.mark.parametrize("case", SI.CASES, ids=lambda c: c[0])
def test_text_cases(text, case):
    """Durations and frame counts equal mode 1's bit for bit; the mel within the budget of the oracle and the reference."""
    cfg, sd, t1, t2 = text
    golden = SI.load_golden()
    name, lens, sids, n, temp, ls, pauses = case
    r1, r2 = synth(t1, case), synth(t2, case)
    assert r2["mel_lengths"] == r1["mel_lengths"]
    worst = 0.0
    for b, (ids, bert, pause, noise) in enumerate(SI.case_inputs(case)):
        assert np.array_equal(r2["durations"][b], r1["durations"][b]), (name, b)
        k = name + ".%s" + str(b)
        w = golden[k % "w_round"]
        o = st.synthesise(sd, cfg, ids, bert, sids[b], noise, pause if pauses.get(b) else None, n, temp, ls, 0.5, torch.float64, durations=w)
        e64 = float(np.abs(r2["decoder_outputs"][b] - o["decoder_outputs"]).max())
        eref = float(np.abs(r2["decoder_outputs"][b] - golden[k % "decoder_outputs"]).max())
        worst = max(worst, e64, eref)
        assert e64 < BUDGET and eref < BUDGET, (name, b, e64, eref)
    print("text %s mode 2: max err %.2e" % (name, worst))


def test_text_alone_equals_batched(text):
    cfg, sd, t1, t2 = text
    case = SI.CASES[-1]
    both = synth(t2, case)
    for b in range(len(case[1])):
        one = synth(t2, case, which=b)
        assert np.array_equal(one["decoder_outputs"][0], both["decoder_outputs"][b]), b


def test_memory_returns_to_baseline(cfm):
    cfg, sd = cfm
    torch.cuda.synchronize()
    before = live_bytes()
    tts = StableTTS(None, sd, device=0, precision=2)
    mu, nz = CI.inputs("short0", 23)
    out = tts.refine([mu, mu[:, :9]], [1, 0], noise=[nz, nz[:, :9]])
    assert np.array_equal(tts.refine(mu, 1, noise=nz), out[0])
    assert live_bytes()[0] > before[0]
    tts.close()
    assert live_bytes() == before


def test_mode2_runs_on_the_tensor_cores(eng2, cfm):
    """A silent fallback to the FFMA pipe would give mode 1's bits: mode 2's mel must differ from them (and stay close)."""
    cfg, sd = cfm
    blob, man = weights.pack_stabletts_cfm(sd, cfg)
    e1 = Engine(cfg, blob, man, device=0, precision=1)
    try:
        mu, nz = CI.inputs("tc_used", 120)
        m1, _ = e1.cfm_decode(mu.T, 1, n_timesteps=3, noise=nz.T)
        m2, _ = eng2.cfm_decode(mu.T, 1, n_timesteps=3, noise=nz.T)
        d = float(np.abs(m1 - m2).max())
        print("mode 2 vs mode 1: max |diff| %.2e" % d)
        assert 0.0 < d < BUDGET
    finally:
        e1.close()


def split_bf16(x):
    """kernels.cuh split_bf16 on float32 rows: (hi, lo) bf16 bit patterns"""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    h = (u + np.uint32(0x8000)) & np.uint32(0xFFFF0000)
    r = (x - h.view(np.float32)).astype(np.float32)
    lo = r.view(np.uint32) + np.uint32(0x8000)
    return (h >> 16).astype(np.uint16), (lo >> 16).astype(np.uint16)


def test_plane_kernels_alone(eng2, cfm):
    """Block 0 at step 0 through the debug taps: each plane-writing kernel's fp32 rows against a restatement of its inputs
    (float32 where the kernel's op order is exact, float64 otherwise), and its planes equal to the split of those rows."""
    cfg, sd = cfm
    H, F, NL, heads = cfg["hidden_channels"], cfg["filter_channels"], cfg["n_layers"], cfg["n_heads"]
    dk = H // heads
    T = 64              # a whole frame bucket: the unconditional sequence's rows start at T + SEQ_GAP (8)
    mu, nz = CI.inputs("planes", T)
    eng2.debug_flags(1)
    try:
        eng2.cfm_decode(mu.T, 1, n_timesteps=2, guidance_scale=0.5, noise=nz.T)
        tap = lambda n, w: eng2.debug_read(n).reshape(-1, w)
        pl = lambda n, w: (eng2.debug_read(n + "_hi").view(np.uint16).reshape(-1, w), eng2.debug_read(n + "_lo").view(np.uint16).reshape(-1, w))
        film = eng2.debug_read("st_film").reshape(2, NL, 2 * H)[0, 0]
        ada = eng2.debug_read("st_ada").reshape(2, NL, 6 * H)[:, 0]
        rope = eng2.debug_read("st_rope").reshape(-1, dk // 4, 2)
        norm_in, norm, norm_pl = tap("tc_norm_in", H), tap("st_norm1", H), pl("tc_norm", H)
        qkv_in, qkv, qkv_pl = tap("tc_qkv_in", 3 * H), tap("st_qkv", 3 * H), pl("tc_qkv", 3 * H)
        silu_in, silu, silu_pl = tap("tc_silu_in", F), tap("tc_silu", F), pl("tc_silu", F)
        gx, gy, gate, gate_pl = tap("tc_gate_x", H), tap("tc_gate_y", H), tap("tc_gate", H), pl("tc_gate", H)
    finally:
        eng2.debug_flags(0)

    def same_planes(x, p, what):
        hi, lo = split_bf16(x)
        assert np.array_equal(hi, p[0]) and np.array_equal(lo, p[1]), what

    f32 = np.float32
    for s, off in enumerate((0, T + 8)):             # the conditional sequence, then the unconditional one
        rows = slice(off, off + T)
        # dit_norm_planes_kernel: FiLM, LayerNorm without affine, modulate
        u = (film[:H] * norm_in[rows] + film[H:]).astype(np.float64)
        ln = (u - u.mean(1, keepdims=True)) / np.sqrt(u.var(1, keepdims=True) + 1e-5)
        want = ln * (1.0 + ada[s, H:2 * H]) + ada[s, :H]
        assert np.abs(norm[rows] - want).max() < 1e-4
        same_planes(norm[rows], (norm_pl[0][rows], norm_pl[1][rows]), "norm")
        # dit_rope_planes_kernel: the first dk/2 features of each q and k head rotated in fp32, two rounded products and a sum
        want = qkv_in[rows].copy()
        cs, sn = rope[:T, :, 0], rope[:T, :, 1]
        hd = dk // 4
        for h in range(2 * heads):
            c0 = (h // heads) * H + (h % heads) * dk
            a, b = qkv_in[rows, c0:c0 + hd], qkv_in[rows, c0 + hd:c0 + 2 * hd]
            want[:, c0:c0 + hd] = (a * cs).astype(f32) + ((-b) * sn).astype(f32)
            want[:, c0 + hd:c0 + 2 * hd] = (b * cs).astype(f32) + (a * sn).astype(f32)
        assert np.array_equal(qkv[rows], want)
        same_planes(qkv[rows], (qkv_pl[0][rows], qkv_pl[1][rows]), "qkv")
        # dit_silu_planes_kernel
        x = silu_in[rows].astype(np.float64)
        assert np.abs(silu[rows] - x / (1.0 + np.exp(-x))).max() <= 2e-6 * max(1.0, float(np.abs(x).max()))
        same_planes(silu[rows], (silu_pl[0][rows], silu_pl[1][rows]), "silu")
        # dit_gate_planes_kernel: x + gate * y in fp32
        assert np.array_equal(gate[rows], gx[rows] + (ada[s, 5 * H:6 * H] * gy[rows]).astype(f32))
        same_planes(gate[rows], (gate_pl[0][rows], gate_pl[1][rows]), "gate")


@pytest.fixture(scope="module")
def voc_tts():
    cfg = SI.config()
    t = StableTTS({"n_vocab": cfg["n_vocab"]}, SI.model(cfg), device=0, precision=2, vocoder=HI.checkpoint())
    yield t
    t.close()


def test_text_to_waveform(voc_tts):
    """ref_hifigan.npz's text cases: the reference's vocoder on the reference's mel of the same utterances."""
    golden = np.load(HI.GOLDEN)
    worst = 0.0
    for key in HI.TEXT_CASES:
        name, b = key.split(".mel")
        case = [c for c in SI.CASES if c[0] == name][0]
        ids, bert, sid, pause, noise = synth_args(case, int(b))
        r = voc_tts.synthesise(ids, bert, sid, pause if case[6] else None, n_timesteps=case[3], temperature=case[4],
                               length_scale=case[5], noise=noise, return_wav=True)
        ref = golden["text." + key + ".wav"]
        assert r["wav"].shape == ref.shape
        err = float(np.abs(r["wav"] - ref).max())
        worst = max(worst, err)
        assert err < WAV_BUDGET, (key, err)
    print("text to waveform mode 2: max |wav - ref| %.2e" % worst)


def synth_args(case, b):
    """(ids, bert, sid, pause, noise) of utterance b of a stabletts_inputs case"""
    ids, bert, pause, noise = SI.case_inputs(case)[b]
    return ids, bert, case[2][b], pause, noise


def test_onnx_voice(tmp_path):
    """The voice read from its exported graph (widths 64: every conv and the attention on the tensor cores) against what the
    reference's synthesise and vocoder give, durations bit for bit."""
    from test_stabletts_onnx_host import GOLDEN
    fix = dict(np.load(os.path.join(GOLDEN, "ref_stabletts_onnx.npz")))
    t = StableTTS.from_onnx(OI.write_graph(tmp_path, fix), device=0, precision=2)
    try:
        std = float(t.mel_std)
        e_mel = e_wav = 0.0
        for i in range(4):
            u = [fix["u%d.%s" % (i, k)] for k in ("ids", "bert", "pause", "sid", "noise")]
            r = t.synthesise([u[0]], [u[1]], [int(u[3])], [u[2]], n_timesteps=t.n_timesteps, temperature=float(fix["temperature"]),
                             length_scale=float(fix["length_scale"]), noise=[u[4]], return_wav=True)
            w = fix["u%d.w_round" % i]
            assert np.array_equal(r["durations"][0], w.astype(r["durations"][0].dtype)), i
            e_mel = max(e_mel, float(np.abs(r["mel"][0] - fix["u%d.mel" % i]).max()) / std)
            e_wav = max(e_wav, float(np.abs(r["wav"][0] - fix["u%d.wav" % i]).max()))
        print("onnx voice mode 2: |mel - ref| / mel_std %.2e  |wav - ref| %.2e" % (e_mel, e_wav))
        assert e_mel < BUDGET and e_wav < WAV_BUDGET
    finally:
        t.close()


def test_pieces_equal_bert_then_host_gather():
    """vtts_stabletts_synthesise_pieces_wav in mode 2: the bits of BERT's features, the gather on the host and
    vtts_stabletts_synthesise_wav."""
    bt = BI.tiny()
    cfg = C.stabletts_config({"n_vocab": 120, "bert_dim": bt["cv_hidden"]})
    t = StableTTS({"n_vocab": 120, "bert_dim": bt["cv_hidden"]}, synthetic.make_random_stabletts(cfg, 8642), device=0, precision=2,
                  vocoder=HI.checkpoint(), bert=(BI.model(bt), bt))
    try:
        rng = np.random.default_rng(3)
        us = []
        for i, L in enumerate((9, 40, 5)):
            T = int(rng.integers(2, 48))
            rows = np.sort(rng.integers(0, L, T)).astype(np.int32)
            rows[0], rows[-1] = 0, L - 1
            us.append((rng.integers(0, 120, (5, T)).astype(np.int64), BI.sentence(bt, L, salt=i), rows,
                       rng.standard_normal((80, SI.MAX_FRAMES)).astype(np.float32), i % 2))
        fused = t.synthesise([u[0] for u in us], None, [u[4] for u in us], n_timesteps=3, noise=[u[3] for u in us],
                             pieces=[u[1] for u in us], bert_rows=[u[2] for u in us])
        feats = t.bert_features([u[1] for u in us])
        berts = [np.ascontiguousarray(f[u[2]].T) for f, u in zip(feats, us)]
        comp = t.synthesise([u[0] for u in us], berts, [u[4] for u in us], n_timesteps=3, noise=[u[3] for u in us], return_wav=True)
        for b in range(len(us)):
            for k in ("durations", "mel", "wav"):
                assert np.array_equal(fused[k][b], comp[k][b]), (k, b)
    finally:
        t.close()
