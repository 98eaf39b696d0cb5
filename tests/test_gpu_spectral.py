"""GPU (-m gpu): the spectral kernels one launch at a time through the engine's own launch code, against the float64
references and error bounds of tests/spectral_ref.py:
  vtts_debug_front_end   clip_frames -> staging -> stft_mag_kernel (-> mel_log_kernel), or spec_pack_kernel
  vtts_debug_istft       istft_pqmf_kernel, as both decoders launch it (istft_tail)
  vtts_debug_mrf_mean    mrf_mean_kernel (FFMA decoder) / mrf_mean_planes_kernel (tensor-core decoder)
Every case runs twice and must give the same bits.  Rows and samples outside the clips / utterances hold a sentinel that
must survive; the staged waveform is NaN behind every clip, so any read outside a clip shows as NaN in its rows."""
import json
import zlib

import numpy as np
import pytest
import torch

import golden_ref as GR
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
import spectral_ref as S
from vosk_tts_b200 import config as C, synthetic, weights
from vosk_tts_b200.engine import Engine, VttsError

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
WORST = {}                   # largest error / bound seen per kernel
FRONT = {c[0]: c for c in S.FRONT_CONFIGS}
TAILS = ["mb_istft", "ms_istft", "istft", "quickvc"]


def _note(kernel, r):
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(r))


def _blob_tensor(blob, man, name):
    for line in man.strip().splitlines():
        p = line.split()
        if p[0] == name:
            return blob[int(p[1]):int(p[1]) + int(p[2])]
    raise KeyError(name)


def _front_cfg(name):
    _, nfft, hop, nmel, model = FRONT[name]
    if model == "quickvc":
        return QI.config()
    j = GR.tiny_training_json()
    j["data"].update(filter_length=nfft, hop_length=hop, win_length=nfft, n_mel_channels=nmel or 80)
    for d in ("data", "model"):
        j[d]["use_mel_posterior_encoder"] = nmel > 0
    return C.from_training_json(j, n_vocab=GR.N_VOCAB)


@pytest.fixture(scope="module")
def engines():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    made = {}

    def get(name):
        if name not in made:
            if name in FRONT:
                cfg = _front_cfg(name)
                if FRONT[name][4] == "quickvc":
                    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QI.speaker_encoder()), cfg)
                else:
                    sd = synthetic.make_random_checkpoint(cfg, 11, posterior=True)
                    blob, man = weights.pack(weights.fold_weight_norm(sd), cfg, posterior=True)
            elif name == "quickvc":
                cfg = QI.config()
                blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), cfg)
            else:
                cfg = C.from_training_json(GR.training_json(name + "_vits"), n_vocab=GR.N_VOCAB)
                blob, man = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 11)), cfg)
            made[name] = (Engine(cfg, blob, man, device=0, precision=0), cfg, blob, man)
        return made[name]
    yield get
    for e in made.values():
        e[0].close()
    print("\nspectral kernels error / bound, largest per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


# ---------------------------------------------------------------------------------------------------- front end
def _speech(L, rng):
    d = GR.load("vc_speech.npz")
    x = np.concatenate([d["a"], d["b"]] * (L // (len(d["a"]) + len(d["b"])) + 1)).astype(np.float32) / 32768.0
    s = int(rng.integers(0, len(x) - L + 1))
    return x[s:s + L]


def _clip(kind, L, nfft, rng):
    return _speech(L, rng) if kind == "speech" else S.signal(kind, L, nfft, rng)


def run_front(ent, clips, from_spec=False, C_in=None):
    """The hook on the clips (float32 arrays), twice, with NaN behind every clip in the caller's buffer; returns (frames, the
    magnitude rows (None for features), the feature rows, row offsets)."""
    e, cfg, blob, man = ent
    B = len(clips)
    lens = np.array([c.shape[-1] for c in clips], np.int64)
    ld = int(lens.max()) + 37
    if from_spec:
        x = np.full((B, C_in, ld), np.nan, np.float32)
        for b, c in enumerate(clips):
            x[b, :, :c.shape[-1]] = c
        frames = lens
    else:
        x = np.full((B, ld), np.nan, np.float32)
        for b, c in enumerate(clips):
            x[b, :len(c)] = c
        frames = e.convert_frames(lens)
    offs = S.offsets(frames)
    rows = offs[-1] + 5
    nbins = cfg["filter_length"] // 2 + 1
    spec_pad = cfg["n_mel_channels"] if cfg.get("model_family") == "quickvc" else (cfg["spec_channels"] + 15) // 16 * 16
    mel = not from_spec and bool(cfg.get("use_mel_posterior_encoder"))
    feat0 = np.full((rows, spec_pad), SENT, np.float32)
    mag0 = np.full((rows, nbins), SENT, np.float32) if mel else None
    out = e.debug_front_end(x, lens, feat0, mag0, from_spec=from_spec)
    out2 = e.debug_front_end(x, lens, feat0, mag0, from_spec=from_spec)
    for a, b2 in zip(out[1:], out2[1:]):
        assert a is None or np.array_equal(a.view(np.uint32), b2.view(np.uint32)), "two launches differ"
    fr, mag, feat = out
    assert np.array_equal(fr, frames), "frame counts differ from Engine.convert_frames"
    inside = np.zeros(rows, bool)
    for b in range(B):
        inside[offs[b]:offs[b] + frames[b]] = True
    for a in (mag, feat):
        if a is not None:
            assert np.all(a[~inside].view(np.uint32) == SENT.view(np.uint32)), "rows outside the clips written"
            assert np.isfinite(a[inside]).all(), "non-finite rows: a read outside a clip"
    return fr, (mag if mel else feat[:, :nbins] if not from_spec else None), feat, offs


def check_front(ent, clips):
    e, cfg, blob, man = ent
    nfft, hop = cfg["filter_length"], cfg["hop_length"]
    nbins = nfft // 2 + 1
    fr, mag, feat, offs = run_front(ent, clips)
    mel = bool(cfg.get("use_mel_posterior_encoder"))
    fb = _blob_tensor(blob, man, "vc.mel").reshape(-1, nbins) if mel else None
    worst_m = worst_l = 0.0
    for b, x in enumerate(clips):
        rows = slice(offs[b], offs[b] + fr[b])
        ref, bound = S.magnitude(x, nfft, hop)
        err = np.abs(mag[rows].astype(np.float64) - ref)
        r = float((err / bound).max())
        assert r <= 1.0, "clip %d (L=%d): magnitude error %.3g x the bound" % (b, len(x), r)
        worst_m = max(worst_m, r)
        if mel:
            v, lo, hi = S.log_mel(mag[rows], fb)
            got = feat[rows, :fb.shape[0]].astype(np.float64)
            bad = (got < lo) | (got > hi)
            assert not bad.any(), "clip %d: log-mel outside its interval at %s" % (b, np.argwhere(bad)[:4].tolist())
            worst_l = max(worst_l, float(np.max(np.where(got >= v, (got - v) / (hi - v), (v - got) / (v - lo)))))
            assert np.all(feat[rows, fb.shape[0]:] == 0)
        else:
            assert np.all(feat[rows, nbins:].view(np.uint32) == 0), "pad columns not exactly 0"
    _note("stft_mag_kernel", worst_m)
    if mel:
        _note("mel_log_kernel", worst_l)
    return fr, mag, feat, offs


def _lengths(nfft, hop, rng):
    """The minimum clip, clips of 1, 63, 64, 65, 128, 129 frames at lengths that are not multiples of hop."""
    out = [S.min_clip(nfft, hop)]
    for F in (1, 63, 64, 65, 128, 129):
        out.append(S.length_for_frames(F, nfft, hop, int(rng.integers(1, hop))))
    return out


@pytest.mark.parametrize("name", list(FRONT))
@pytest.mark.parametrize("kind", ["noise", "silence", "dc", "nyquist", "tone", "speech"])
def test_front_end_clips_alone_and_in_a_ragged_batch(engines, name, kind):
    ent = engines(name)
    cfg = ent[1]
    nfft, hop = cfg["filter_length"], cfg["hop_length"]
    rng = np.random.default_rng(zlib.crc32((name + kind).encode()))
    clips = [_clip(kind, L, nfft, rng) for L in _lengths(nfft, hop, rng)]
    alone = [check_front(ent, [c]) for c in clips]
    order = rng.permutation(len(clips))
    batch = [clips[i] for i in order] + [_clip(kind, int(rng.integers(S.min_clip(nfft, hop), 9 * nfft)), nfft, rng) for _ in range(16 - len(clips))]
    fr, mag, feat, offs = check_front(ent, batch)
    for j, i in enumerate(order):         # each clip's rows bit-identical alone and in the batch
        a = alone[i]
        assert np.array_equal(feat[offs[j]:offs[j] + fr[j]].view(np.uint32), a[2][:a[0][0]].view(np.uint32))
        assert np.array_equal(mag[offs[j]:offs[j] + fr[j]].view(np.uint32), a[1][:a[0][0]].view(np.uint32))


@pytest.mark.parametrize("name", ["mel1024", "qvc1280", "lin1024"])
def test_front_end_long_clip(engines, name):
    ent = engines(name)
    cfg = ent[1]
    rng = np.random.default_rng(30)
    L = 30 * cfg["sampling_rate"] + 77
    check_front(ent, [_clip("speech", L, cfg["filter_length"], rng), _clip("noise", 5000, cfg["filter_length"], rng)])


@pytest.mark.parametrize("name", ["lin1024", "mel1024", "qvc1280"])
def test_spec_pack_is_an_exact_transpose(engines, name):
    ent = engines(name)
    cfg = ent[1]
    Cc = cfg["spec_channels"]
    rng = np.random.default_rng(7)
    lens = [1, 63, 64, 65, 200, 3]
    clips = [rng.standard_normal((Cc, T)).astype(np.float32) for T in lens]
    fr, _, feat, offs = run_front(ent, clips, from_spec=True, C_in=Cc)
    for b, c in enumerate(clips):
        rows = feat[offs[b]:offs[b] + lens[b]]
        assert np.array_equal(rows[:, :Cc].view(np.uint32), c.T.view(np.uint32))
        assert np.all(rows[:, Cc:].view(np.uint32) == 0)


@pytest.mark.parametrize("name", list(FRONT))
def test_front_end_refuses_clips_without_a_frame(engines, name):
    e, cfg, _, _ = engines(name)
    nfft, hop = cfg["filter_length"], cfg["hop_length"]
    lo = S.min_clip(nfft, hop)
    assert e.min_clip_samples() == lo
    assert list(e.convert_frames([lo - 1, lo])) == [0, 1]
    spec_pad = cfg["n_mel_channels"] if cfg.get("model_family") == "quickvc" else (cfg["spec_channels"] + 15) // 16 * 16
    mel = bool(cfg.get("use_mel_posterior_encoder"))

    def call(lens):
        x = np.zeros((len(lens), max(lens)), np.float32)
        return e.debug_front_end(x, lens, np.zeros((20, spec_pad), np.float32),
                                 np.zeros((20, nfft // 2 + 1), np.float32) if mel else None)
    with pytest.raises(VttsError) as ei:
        call([lo - 1])
    assert ei.value.code == -1 and "at least %d samples" % lo in str(ei.value)
    assert list(call([lo])[0]) == [1]
    if name == "mel1024h512":          # pad (256) < L (300) < hop (512): one frame, read before the clip, without the check
        with pytest.raises(VttsError) as ei:
            call([600, 300])
        assert ei.value.code == -1


# ---------------------------------------------------------------------------------------------------- decoder tail
def _tail_parts(ent):
    e, cfg, blob, man = ent
    sb = cfg["subbands"]
    basis = _blob_tensor(blob, man, "dec.istft").reshape(18, 16)
    bank = _blob_tensor(blob, man, "dec.pqmf").reshape(sb, 63)
    try:
        w2 = _blob_tensor(blob, man, "dec.w2")
    except KeyError:
        w2 = None
    hop_total = C.hop_total(cfg)
    return sb, basis, bank, w2, hop_total // (4 * sb), hop_total


def run_tail(ent, lens, kind, first=0, seed=0):
    e = ent[0]
    sb, basis, bank, w2, up, hop_total = _tail_parts(ent)
    rng = np.random.default_rng(seed)
    prow, wav0, rows, n = S.tail_layout(lens, up, hop_total, first)
    post = np.full((rows + 3, sb * 18), np.nan, np.float32)       # poison in the gap rows
    P = []
    for b, T in enumerate(lens):
        p = S.post_values(kind, up * T + 1, sb * 18, rng)
        post[prow[b]:prow[b] + len(p)] = p
        P.append(p)
    wav = np.full(n + 11, SENT, np.float32)
    out = e.debug_istft(lens, post, wav, first=first)
    out2 = e.debug_istft(lens, post, wav, first=first)
    assert np.array_equal(out.view(np.uint32), out2.view(np.uint32)), "two launches differ"
    inside = np.zeros(out.size, bool)
    worst = 0.0
    res = []
    for b, T in enumerate(lens):
        seg = slice(wav0[b], wav0[b] + T * hop_total)
        inside[seg] = True
        ref, bound = S.tail(P[b], basis, bank, 4, w2=w2)
        got = out[seg].astype(np.float64)
        assert np.isfinite(got).all()
        r = float((np.abs(got - ref) / bound).max())
        assert r <= 1.0, "utterance %d (Ty=%d, %s): error %.3g x the bound at sample %d" % (
            b, T, kind, r, int(np.argmax(np.abs(got - ref) / bound)))
        worst = max(worst, r)
        res.append(out[seg].copy())
    assert np.all(out[~inside].view(np.uint32) == SENT.view(np.uint32)), "samples outside the utterances written"
    _note("istft_pqmf_kernel", worst)
    return res


@pytest.mark.parametrize("dec", TAILS)
@pytest.mark.parametrize("kind", ["normal", "logmag", "phase"])
def test_tail_every_length_alone(engines, dec, kind):
    ent = engines(dec)
    for T in S.TAIL_TY:
        run_tail(ent, [T], kind, seed=T)


@pytest.mark.parametrize("dec", TAILS)
def test_tail_ragged_batch_matches_alone(engines, dec):
    ent = engines(dec)
    rng = np.random.default_rng(1)
    lens = [int(t) for t in rng.choice(S.TAIL_TY[:-1] + [33, 150], 64)]
    lens[5] = 1000
    batch = run_tail(ent, lens, "normal", seed=2)
    # the same rows alone give the same bits: rerun each distinct utterance alone with the same rows
    sb, _, _, _, up, hop_total = _tail_parts(ent)
    rs = np.random.default_rng(2)
    Ps = [S.post_values("normal", up * T + 1, sb * 18, rs) for T in lens]
    for b in (0, 5, 17, 63):
        post = Ps[b]
        wav = ent[0].debug_istft([lens[b]], post, np.zeros(lens[b] * hop_total, np.float32))
        assert np.array_equal(wav.view(np.uint32), batch[b].view(np.uint32)), "utterance %d differs alone" % b


@pytest.mark.parametrize("dec", ["mb_istft", "quickvc"])
@pytest.mark.parametrize("first", [1, 24, 77])
def test_tail_chunk_addressing(engines, dec, first):
    """vtts_decode_chunk's rows start at offs[0] = lo > 0."""
    run_tail(engines(dec), [17], "normal", first=first, seed=first)
    run_tail(engines(dec), [5, 64], "phase", first=first, seed=first + 1)


# ---------------------------------------------------------------------------------------------------- MRF mean
# (channels, rmul) of each upsample stage: the VITS2 default decoder (512, [4, 4]) and QuickVC's (512, [5, 4])
MRF_STAGES = [(256, 4, False), (128, 16, True), (256, 5, False), (128, 20, True)]


@pytest.mark.parametrize("ch,rmul,last", MRF_STAGES)
@pytest.mark.parametrize("n", [1, 2, 3])
def test_mrf_mean(engines, ch, rmul, last, n):
    e = engines("mb_istft")[0]
    rng = np.random.default_rng(ch + rmul + n)
    lens = [1, 3, 17, 64, 5]
    offs = S.offsets(lens)
    rows = offs[-1] * rmul + 7
    x = (rng.standard_normal((n, rows, ch)) * rng.choice([1e-3, 1.0, 30.0], (n, rows, 1))).astype(np.float32)
    ref = S.mrf_mean(list(x))
    # FFMA: the whole buffer
    out0 = np.full((rows, ch), SENT, np.float32)
    a = e.debug_mrf_mean(lens, rmul, x, out=out0)[0]
    assert np.array_equal(a.view(np.uint32), e.debug_mrf_mean(lens, rmul, x, out=out0)[0].view(np.uint32))
    assert np.array_equal(a.view(np.uint32), ref.view(np.uint32)), "mrf_mean_kernel is not ((a + b) + c) / n"
    # tensor cores: planes of lrelu(mean) at the utterances' rows (and the reflect row), fp32 mean in out
    prow = offs[-1] * rmul + len(lens) + 5
    hs = np.full((prow, ch), 0xBEEF, np.uint16)
    for with_out in (False, True):
        o, hi, lo = e.debug_mrf_mean(lens, rmul, x, out=out0 if with_out else None, hi=hs, lo=hs, use_tc=True, last=last)
        o2, hi2, lo2 = e.debug_mrf_mean(lens, rmul, x, out=out0 if with_out else None, hi=hs, lo=hs, use_tc=True, last=last)
        assert np.array_equal(hi, hi2) and np.array_equal(lo, lo2)
        eh, el = np.full_like(hs, 0xBEEF), np.full_like(hs, 0xBEEF)
        eo = out0.copy()
        slope = 0.01 if last else 0.1
        for b, T in enumerate(lens):
            base, L = offs[b] * rmul, T * rmul
            q = S.lrelu32(ref[base:base + L], slope)
            h, l = S.split_bf16(q)
            r0 = base + (b if last else 0)
            if last:          # ReflectionPad1d((1, 0)): row 0 is row 1's planes, then the rows shifted by one
                eh[r0], el[r0] = h[1], l[1]
                eh[r0 + 1:r0 + 1 + L], el[r0 + 1:r0 + 1 + L] = h, l
            else:
                eh[r0:r0 + L], el[r0:r0 + L] = h, l
            eo[base:base + L] = ref[base:base + L]
        assert np.array_equal(hi, eh) and np.array_equal(lo, el), "planes differ (or rows outside the utterances written)"
        if with_out:
            assert np.array_equal(o.view(np.uint32), eo.view(np.uint32)) and np.array_equal(o, o2)
        else:
            assert o is None
