"""GPU (-m gpu): the CUDA path, called through the C ABI (libvtts.so via ctypes), against
 (1) fixtures produced by the unmodified reference (tests/golden), (2) the oracle on fresh seeded inputs,
 (3) size-independent properties at BASELINE.json's full sizes.
Tolerances: waveform max-abs <= 1e-3 (north_star, fp32); durations / alignment indices bit-exact."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden

pytestmark = pytest.mark.gpu
WAV_TOL = 1e-3      # north_star tolerance
WAV_TIGHT = 8e-5    # what the engine achieves on a +-0.9 waveform (fp32 FFMA ~2e-6, split-bf16 tensor path ~2.5e-5)


def _case(g, u):
    p = "u%d_" % u
    return dict(tok=g[p + "tokens"], sid=int(g[p + "sid"]), eps_dp=g[p + "eps_dp"], eps_z=g[p + "eps_z"],
                w_ceil=g[p + "w_ceil"], idx=g[p + "idx"], Ty=int(g[p + "y_length"]), wav=g[p + "wav"], z=g[p + "z"],
                z_p=g[p + "z_p"])


@pytest.mark.parametrize("name", [c for c in GOLDEN_CASES if c != "ragged3"])
def test_golden_single_utterance(engine, name):
    g = load_golden(name)
    c = _case(g, 0)
    T = len(c["tok"])
    engine.debug_flags(1)
    ylen, dur = engine.durations(c["tok"][None], [T], [c["sid"]], g["scales"], c["eps_dp"][None], want_durations=True)
    assert int(ylen[0]) == c["Ty"]
    assert np.array_equal(dur[0], c["w_ceil"]), "durations (w_ceil) must be bit-exact"
    wav, idx = engine.synthesize(ylen, c["eps_z"][None], want_alignment=True)
    assert np.array_equal(idx[0, : c["Ty"]], c["idx"]), "alignment indices must be bit-exact"
    z_p = engine.debug_read("z_p").reshape(c["Ty"], -1)
    z = engine.debug_read("z").reshape(c["Ty"], -1)
    assert np.abs(z_p - c["z_p"].T).max() < 3e-4      # |z_p| ~ 10-16: 2e-5 relative (split-bf16 encoder in mode 2)
    assert np.abs(z - c["z"].T).max() < 3e-4
    err = np.abs(wav[0, : c["Ty"] * 256] - c["wav"]).max()
    assert err < WAV_TOL
    assert err < WAV_TIGHT, "fp32 path drifted: %g" % err
    engine.debug_flags(0)


def test_golden_ragged_batch_in_one_call(engine):
    """Three utterances of different length in ONE call must each equal the reference's B=1 result
    (per-utterance zero halos in the unmasked decoder, SURVEY.md section 7 'ragged batches')."""
    g = load_golden("ragged3")
    n = int(g["n"])
    cs = [_case(g, u) for u in range(n)]
    Tm = max(len(c["tok"]) for c in cs)
    ids = np.full((n, Tm), 61, np.int64)          # garbage beyond the lengths must be ignored
    eps_dp = np.full((n, 2, Tm), 9.0, np.float32)
    for u, c in enumerate(cs):
        ids[u, : len(c["tok"])] = c["tok"]
        eps_dp[u, :, : len(c["tok"])] = c["eps_dp"]
    lens = [len(c["tok"]) for c in cs]
    ylen, dur = engine.durations(ids, lens, [c["sid"] for c in cs], g["scales"], eps_dp, want_durations=True)
    assert [int(v) for v in ylen] == [c["Ty"] for c in cs]
    eps_z = np.full((n, 192, int(ylen.max())), 7.0, np.float32)
    for u, c in enumerate(cs):
        assert np.array_equal(dur[u, : lens[u]], c["w_ceil"])
        eps_z[u, :, : c["Ty"]] = c["eps_z"]
    wav, idx = engine.synthesize(ylen, eps_z, want_alignment=True)
    for u, c in enumerate(cs):
        assert np.array_equal(idx[u, : c["Ty"]], c["idx"])
        assert np.abs(wav[u, : c["Ty"] * 256] - c["wav"]).max() < WAV_TIGHT
        assert not wav[u, c["Ty"] * 256:].any()


def _rel_margin(logw, length_scale):
    """Smallest distance of a duration w = exp(logw) * length_scale to an integer, relative to w: ceil(w) of an implementation
    with relative error eps on w can differ from the oracle's only if this is below eps (FFMA path ~2e-6, split-bf16 ~2e-5)."""
    w = (torch.exp(logw) * length_scale).double().numpy().reshape(-1)
    return float((np.abs(w - np.round(w)) / np.maximum(w, 1e-9)).min())


def _check_durations(dur, logw, length_scale, w_ceil, precision):
    """ceil(w) may differ from the oracle's only where the oracle's own w = exp(logw) * length_scale lies close to an integer:
    within 1e-4 (relative) for the fp32 FFMA text encoder (modes 0, 1; its error on w is ~2e-6, the slack covers the
    ill-conditioned spline), within 2e-3 for the tensor-core text encoders (modes 2, 3: measured flip rates 12 and 9 per
    1000 utterances against 3, profiles/r2_parity_sweep.json).  Returns True when every duration is equal."""
    ref = np.asarray(w_ceil).astype(np.int32).reshape(-1)
    dur = np.asarray(dur).reshape(-1)[: ref.size]
    w = (torch.exp(logw) * length_scale).double().numpy().reshape(-1)[: ref.size]
    rel = np.abs(w - np.round(w)) / np.maximum(w, 1e-9)
    mism = dur != ref
    thr = 1e-4 if precision < 2 else 2e-3
    assert not (mism & (rel >= thr)).any(), "duration flipped away from an integer boundary: rel. margins %s" % rel[mism]
    assert (np.abs(dur - ref)[mism] <= 1).all()
    return not mism.any()


def _oracle_case(cfg, folded, T, seed, sid, scales, min_margin=1e-4):
    """Seeded inputs whose durations all keep a relative distance >= min_margin from an integer (the first seed at or after
    `seed` that does: a deterministic choice, so the comparison below never has to be skipped)."""
    from oracle import vits_oracle as vo
    for s in range(seed, seed + 50):
        g = torch.Generator().manual_seed(s)
        tok = torch.randint(0, cfg["n_vocab"], (1, T), generator=g)
        eps_dp = torch.randn(1, 2, T, generator=g)
        with torch.no_grad():
            o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([sid]), scales, eps_dp, lambda shp: torch.zeros(shp), return_all=True, decode=False)
        if _rel_margin(o["logw"], scales[1]) >= min_margin:
            Ty = int(o["y_lengths"][0])
            eps_z = torch.randn(1, cfg["inter_channels"], Ty, generator=g)
            return tok, eps_dp, eps_z, Ty
    raise AssertionError("no seed with the required duration margin")


@pytest.mark.parametrize("T,seed,sid,scales", [(64, 11, 0, (0.8, 1.0, 0.8)), (200, 12, 4, (0.667, 0.9, 0.8)),
                                               (256, 13, 150, (1.0, 1.1, 1.0))])
def test_fresh_inputs_vs_oracle(engine, folded, cfg, T, seed, sid, scales):
    from oracle import vits_oracle as vo
    tok, eps_dp, eps_z, Ty = _oracle_case(cfg, folded, T, seed, sid, scales)
    with torch.no_grad():
        o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([sid]), scales, eps_dp, eps_z, return_all=True)
    assert Ty == int(o["y_lengths"][0])
    ylen, dur = engine.durations(tok.numpy(), [T], [sid], scales, eps_dp.numpy(), want_durations=True)
    same = _check_durations(dur[0], o["logw"], scales[1], o["w_ceil"][0, 0].numpy(), engine.precision)
    if not same:
        assert engine.precision >= 2
        engine.synthesize(ylen, None)
        return
    wav = engine.synthesize(ylen, eps_z.numpy())
    assert np.abs(wav[0, : Ty * 256] - o["o"][0, 0].numpy()).max() < WAV_TIGHT


def _rand_batch(cfg, B, lo, hi, seed):
    rng = np.random.RandomState(seed)
    lens = rng.randint(lo, hi + 1, size=B)
    ids = rng.randint(0, cfg["n_vocab"], size=(B, int(lens.max()))).astype(np.int64)
    sid = rng.randint(0, 5, size=B).astype(np.int64)
    return ids, lens, sid


def test_full_size_batch_invariance_and_determinism(engine, cfg):
    """BASELINE.json configs[2] shape (batch 64, 64-256 phonemes): an utterance's samples do not depend on what
    else is in the batch (to summation-order noise: the split-K decomposition of a conv is chosen from the size of
    the launch), and the Philox path is deterministic in its seed (bit-exact run to run)."""
    ids, lens, sid = _rand_batch(cfg, 64, 64, 256, 1)
    scales = (0.8, 1.0, 0.8)
    wav, ylen = engine.infer(ids, lens, sid, scales, seed=42)
    wav2, ylen2 = engine.infer(ids, lens, sid, scales, seed=42)
    assert np.array_equal(ylen, ylen2) and np.array_equal(wav, wav2)
    assert np.isfinite(wav).all() and 0.05 < np.abs(wav).max() < 20
    for b in (0, 17, 63):
        Ty = int(ylen[b])
        assert 64 <= Ty
        assert not wav[b, Ty * 256:].any()
    wav3, ylen3 = engine.infer(ids, lens, sid, scales, seed=43)
    assert not np.array_equal(wav3[:, :1024], wav[:, :1024])
    # noise-free: (noise scales 0) -> independent of the seed, and batch-invariant
    wa, ya = engine.infer(ids, lens, sid, (0.0, 1.0, 0.0), seed=1)
    for b in (3, 40):
        wb, yb = engine.infer(ids[b:b + 1, : lens[b]], lens[b:b + 1], sid[b:b + 1], (0.0, 1.0, 0.0), seed=99)
        assert int(yb[0]) == int(ya[b])
        assert np.abs(wb[0] - wa[b, : int(yb[0]) * 256]).max() < 2e-5


def test_length_scale_scales_durations(engine, cfg):
    ids, lens, sid = _rand_batch(cfg, 4, 100, 128, 5)
    _, d1 = engine.durations(ids, lens, sid, (0.0, 1.0, 0.0), want_durations=True)
    _, d2 = engine.durations(ids, lens, sid, (0.0, 2.0, 0.0), want_durations=True)
    assert (d2 >= d1).all() and (d2 <= 2 * d1).all() and d2.sum() > 1.5 * d1.sum()


def test_long_utterance_2000_phonemes_vs_oracle(engine, folded, cfg):
    """BASELINE.json configs[4] length, monolithic, against the oracle on the same inputs: all 2000 durations and the
    frame->token alignment bit-exact, the latent z after the flow (whose attention spans all ~2500 frames: the long-sequence
    path of the attention kernels) and the first and the last two seconds of audio (the decoder is local -- +-24 frames --
    so the oracle vocodes just those slices of its own z)."""
    from oracle import vits_oracle as vo
    T, sid, scales = 2000, 2, (0.8, 1.0, 0.8)
    tok, eps_dp, eps_z, Ty = _oracle_case(cfg, folded, T, 9, sid, scales)
    with torch.no_grad():
        o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([sid]), scales, eps_dp, eps_z, decode=False)
    engine.debug_flags(1)
    ylen, dur = engine.durations(tok.numpy(), [T], [sid], scales, eps_dp.numpy(), want_durations=True)
    same = _check_durations(dur[0], o["logw"], scales[1], o["w_ceil"][0, 0].numpy(), engine.precision)
    if not same:      # (tensor-core text encoders only, see _check_durations: a flipped ceil shifts every later frame)
        assert engine.precision >= 2
        engine.synthesize(ylen, None)
        engine.debug_flags(0)
        return
    assert int(ylen[0]) == Ty
    wav, idx = engine.synthesize(ylen, eps_z.numpy(), want_alignment=True)
    assert np.array_equal(idx[0, :Ty], o["idx"][0].numpy().astype(np.int32))
    z = engine.debug_read("z").reshape(Ty, -1)
    engine.debug_flags(0)
    assert np.abs(z - o["z"][0].numpy().T).max() < 3e-4
    assert wav.shape[1] == Ty * 256 and np.isfinite(wav).all()
    n2s, halo = 173, 24                                   # 173 frames = 2.0 s
    zz = o["z"] * o["y_mask"]
    with torch.no_grad():
        head, _ = vo.decoder_mb_istft(zz[:, :, : n2s + halo], folded, cfg)
        tail, _ = vo.decoder_mb_istft(zz[:, :, Ty - n2s - halo:], folded, cfg)
    assert np.abs(wav[0, : n2s * 256] - head[0, 0, : n2s * 256].numpy()).max() < WAV_TIGHT
    assert np.abs(wav[0, (Ty - n2s) * 256:] - tail[0, 0, halo * 256:].numpy()).max() < WAV_TIGHT


def test_batch64_utterances_vs_oracle(engine, folded, cfg):
    """BASELINE.json configs[2] shape (64 utterances of 64..256 phonemes in ONE ragged call, caller-supplied noise): every one of
    the 64 utterances' durations is checked against the oracle's B=1 run (rule: _check_durations), and the first eight whose
    durations all agree are compared sample by sample with the oracle's waveform."""
    from oracle import vits_oracle as vo
    B, scales = 64, (0.8, 1.0, 0.8)
    ids, lens, sid = _rand_batch(cfg, B, 64, 256, 1)
    g = torch.Generator().manual_seed(64)
    eps_dp = torch.randn(B, 2, ids.shape[1], generator=g)
    ylen, dur = engine.durations(ids, lens, sid, scales, eps_dp.numpy(), want_durations=True)
    eps_z = torch.randn(B, 192, int(ylen.max()), generator=g)
    wav = engine.synthesize(ylen, eps_z.numpy())
    compared = 0
    for b in range(B):
        T = int(lens[b])
        tok = torch.as_tensor(ids[b:b + 1, :T])
        with torch.no_grad():
            od = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([int(sid[b])]), scales, eps_dp[b:b + 1, :, :T],
                          lambda shp: torch.zeros(shp), return_all=True, decode=False)
        margin_ok = _check_durations(dur[b, :T], od["logw"], scales[1], od["w_ceil"][0, 0].numpy(), engine.precision)
        if margin_ok and compared < 8:
            Ty = int(od["y_lengths"][0])
            assert Ty == int(ylen[b])
            with torch.no_grad():
                o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([int(sid[b])]), scales, eps_dp[b:b + 1, :, :T], eps_z[b:b + 1, :, :Ty])
            assert np.abs(wav[b, : Ty * 256] - o["o"][0, 0].numpy()).max() < WAV_TIGHT, "utterance %d" % b
            assert not wav[b, Ty * 256:].any()
            compared += 1
    assert compared == 8


def test_chunked_vocoder_equals_monolithic(engine, cfg):
    """BASELINE.json configs[4] mechanism: flow once, vocode 64-frame chunks with a 24-frame halo that is discarded;
    the concatenation equals the monolithic waveform (the halo covers the decoder's receptive field, SURVEY.md section 5)."""
    rng = np.random.RandomState(4)
    ids = rng.randint(0, cfg["n_vocab"], size=(1, 300)).astype(np.int64)
    mono, yl = engine.infer(ids, [300], [2], (0.8, 1.0, 0.8), seed=9)
    chunks = list(engine.synthesize_stream(ids, 2, (0.8, 1.0, 0.8), chunk_frames=64, seed=9))
    wav = np.concatenate(chunks)
    assert len(chunks) == -(-int(yl[0]) // 64) and wav.size == mono.shape[1]
    tol = 2e-6 if engine.precision == 0 else 5e-5
    assert np.abs(wav - mono[0]).max() < tol


def test_error_paths(engine, cfg):
    from vosk_tts_b200.engine import VttsError
    ids, lens, sid = _rand_batch(cfg, 2, 8, 16, 2)
    with pytest.raises(VttsError) as e:
        engine.synthesize(np.array([4, 4]))
    assert e.value.code == -5
    with pytest.raises(VttsError) as e:
        engine.durations(ids, [0, 5], sid, (0.8, 1, 0.8))
    assert e.value.code == -1
    ylen = engine.durations(ids, lens, sid, (0.8, 1, 0.8))
    with pytest.raises(VttsError) as e:
        engine.synthesize(ylen, np.zeros((2, 192, 1), np.float32))      # too few noise columns
    assert e.value.code == -4


def test_graph_replay_equals_eager(engine, cfg):
    """The same call three times: eager, graph capture, graph replay -- bit-identical waveforms."""
    ids, lens, sid = _rand_batch(cfg, 2, 40, 60, 21)
    engine.set_graphs(False)
    ref, yl = engine.infer(ids, lens, sid, (0.8, 1.0, 0.8), seed=5)
    engine.set_graphs(True)
    n0 = engine.graph_replays()
    for _ in range(3):
        w, y2 = engine.infer(ids, lens, sid, (0.8, 1.0, 0.8), seed=5)
        assert np.array_equal(y2, yl) and np.array_equal(w, ref)
    assert engine.graph_replays() > n0


def test_one_handle_called_from_several_threads(engine, cfg):
    """The gRPC server of the reference calls ONE shared session from a thread pool (server/tts_server.py:35,57).  Both the
    one-shot call (vtts_infer) and the two-phase pair (vtts_durations -> vtts_synthesize, which keeps state in the handle
    between the calls) must give every thread its own utterance's result."""
    import threading
    g = torch.Generator().manual_seed(5)
    jobs = []
    for i in range(6):
        T = int(torch.randint(20, 90, (1,), generator=g))
        jobs.append([torch.randint(0, cfg["n_vocab"], (1, T), generator=g).numpy(), T, i % 5,
                     torch.randn(1, 2, T, generator=g).numpy(), None])
    serial = []
    for job in jobs:
        tok, T, sid, e1, _ = job
        yl = engine.durations(tok, [T], [sid], (0.8, 1.0, 0.8), e1)
        job[4] = torch.randn(1, 192, int(yl[0]), generator=g).numpy()       # (the frame count is data dependent)
        serial.append(engine.synthesize(yl, job[4]).copy())
    out, errs = [None] * len(jobs), []

    def work(k, two_phase):
        try:
            for rep in range(4):
                tok, T, sid, e1, e2 = jobs[k]
                if two_phase:
                    yl = engine.lib_durations_threadsafe(tok, [T], [sid], (0.8, 1.0, 0.8), e1)
                    w = engine.lib_synthesize_threadsafe(1, yl, e2[:, :, : int(yl[0])])
                else:
                    w, yl = engine.infer(tok, [T], [sid], (0.8, 1.0, 0.8), e1, e2[:, :, : serial[k].shape[1] // 256], frames_hint=serial[k].shape[1] // 256)
                out[k] = np.array(w)
        except Exception as ex:      # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=work, args=(k, k % 2 == 0)) for k in range(len(jobs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for k in range(len(jobs)):
        # (not bit-identical: a one-shot call may run its second phase for a larger predicted length bucket, whose launches
        #  split their k-loops differently -- same arithmetic, another summation order; other utterances differ by ~0.1)
        assert out[k].shape == serial[k].shape and np.abs(out[k] - serial[k]).max() < 2e-5, "thread %d got another utterance's result" % k


@pytest.mark.parametrize("margin", [None, "0.45"], ids=["default-margin", "forced-mispredictions"])
def test_speculative_second_phase_hits_and_misses(packed, cfg, margin):
    """Single-utterance infer calls enqueue phase 2 for a PREDICTED length bucket before the durations are known (the
    device-side lengths are clamped to that bucket, so an under-prediction cannot overrun the bucket-sized buffers) and
    repeat it with the true shape when the prediction was too small.  Whatever the prediction, the result must equal the
    two-phase API's.  With VTTS_SPEC_MARGIN=0.45 the predictor asks for less than half of what it has seen: every call
    whose frame count does not fit the under-sized bucket takes the repeat path."""
    import os
    from vosk_tts_b200.engine import Engine
    env = {"VTTS_SPEC": "1"}                       # (speculation is opt-in: see vtts_engine::use_spec)
    if margin is not None:
        env["VTTS_SPEC_MARGIN"] = margin
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        engine = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    g = torch.Generator().manual_seed(91)
    plan = [(100, 1.0), (90, 1.0), (110, 1.1), (100, 0.25), (96, 1.0), (100, 2.0), (64, 1.0), (128, 1.0), (128, 1.0)]
    for T, ls in plan:
        tok = torch.randint(0, cfg["n_vocab"], (1, T), generator=g).numpy()
        eps_dp = torch.randn(1, 2, T, generator=g).numpy()
        scales = (0.8, ls, 0.8)
        yl = engine.durations(tok, [T], [1], scales, eps_dp)
        Ty = int(yl[0])
        eps_z = torch.randn(1, 192, Ty, generator=g).numpy()
        ref = engine.synthesize(yl, eps_z)
        for rep in range(2):
            wav, yl2 = engine.infer(tok, [T], [1], scales, eps_dp, eps_z, frames_hint=Ty + 40)
            assert int(yl2[0]) == Ty
            assert np.abs(wav[:, : Ty * 256] - ref[:, : Ty * 256]).max() < 2e-5      # (another bucket => another summation order)
    hits, misses = engine.speculation_stats()
    if margin is None:
        assert hits >= 12, (hits, misses)
    else:
        assert misses >= 8, (hits, misses)
    engine.close()


def test_bucketed_graphs_serve_unseen_utterances(engine, cfg):
    """Graphs are captured per LENGTH BUCKET: utterances that were never seen before (other tokens, other lengths inside the
    bucket, other noise) must replay a captured graph and give exactly what eager launches give -- including a short
    utterance right after a longer one of the same bucket (rows behind the utterance's end hold the previous call's data
    until zero_tails_kernel clears them)."""
    g = torch.Generator().manual_seed(77)
    cases = []
    for T in (128, 121, 113, 126, 115, 128, 119):                       # one token bucket (113..128)
        tok = torch.randint(0, cfg["n_vocab"], (1, T), generator=g).numpy()
        eps_dp = torch.randn(1, 2, T, generator=g).numpy()
        eps_z = torch.randn(1, 192, 12 * T, generator=g).numpy()
        cases.append((tok, T, eps_dp, eps_z))
    engine.set_graphs(False)
    refs = []
    for tok, T, eps_dp, eps_z in cases:
        yl = engine.durations(tok, [T], [3], (0.8, 1.0, 0.8), eps_dp)
        refs.append((int(yl[0]), engine.synthesize(yl, eps_z[:, :, : int(yl[0])]).copy()))
    engine.set_graphs(True)
    n0 = engine.graph_replays()
    for rep in range(3):
        for (tok, T, eps_dp, eps_z), (Ty, ref) in zip(cases, refs):
            yl = engine.durations(tok, [T], [3], (0.8, 1.0, 0.8), eps_dp)
            assert int(yl[0]) == Ty
            wav = engine.synthesize(yl, eps_z[:, :, :Ty])
            assert np.array_equal(wav, ref), "graph replay differs from eager launches (rep %d, T=%d)" % (rep, T)
    # after the buckets have been seen twice everything replays: 7 utterances x 2 phases in the last repetition alone
    assert engine.graph_replays() - n0 >= 14


@pytest.mark.parametrize("env", [{"VTTS_TC_BN": "128"}, {"VTTS_TC_TALL": "1"}, {"VTTS_PDL": "0"}, {"VTTS_CONV_MAXS": "1", "VTTS_CONV_MAXG": "4"},
                                 {"VTTS_ATTN_ROWS": "4"}, {"VTTS_TC_MULTICAST": "1"}, {"VTTS_TC_SPLIT": "1"}, {"VTTS_TC_SPLIT": "2"},
                                 {"VTTS_TC_MINSTEPS": "1"}, {"VTTS_TC_BN": "128", "VTTS_TC_MINSTEPS": "1"}, {"VTTS_TC_BN": "64"}, {"VTTS_ATTN_SPLIT": "0"},
                                 {"VTTS_CONV_AUTOG": "0"}, {"VTTS_MRF_BRANCH": "1"}, {"VTTS_BUCKETS": "0"}, {"VTTS_ATTN_TC": "0"},
                                 {"VTTS_TC_PERSIST": "2", "VTTS_TC_SPLIT": "1"}, {"VTTS_TC_PERSIST": "2", "VTTS_TC_SPLIT": "1", "VTTS_TC_TALL": "-1"},
                                 {"VTTS_TC_PERSIST": "2", "VTTS_TC_SPLIT": "1", "VTTS_TC_WMC": "1"},
                                 {"VTTS_TC_PERSIST": "2", "VTTS_TC_SPLIT": "1", "VTTS_TC_BN": "128"}, {"VTTS_TC_SPLIT": "1", "VTTS_TC_MULTICAST": "2"}],
                         ids=["tc-128-wide-tiles", "tc-tall-activation-tiles", "no-programmatic-dependent-launch", "ffma-no-cluster-4-groups",
                              "attention-4-rows-per-warp", "tc-tma-multicast-cluster", "tc-no-split-k", "tc-split-k-pairs",
                              "tc-split-k-8-ways", "tc-128-wide-split-k-8-ways", "tc-64-wide-only", "attention-without-split-kv",
                              "ffma-single-thread-group", "mrf-chains-on-separate-streams", "exact-sizes-no-length-buckets",
                              "ffma-attention-in-the-flow", "tc-persistent-tile-loop-tall", "tc-persistent-tile-loop-per-tap-tiles",
                              "tc-persistent-weight-multicast-pairs", "tc-persistent-tile-loop-128-wide", "tc-tma-multicast-pairs-no-split-k"])
def test_alternative_kernel_configurations_match_golden(packed, cfg, env, default_conv_shapes):
    """The tuning switches select different tilings / launch modes of the same kernels (128-wide tensor-core tiles are what
    batched calls use automatically); each must still reproduce the reference fixture.  A switch of the dense conv launches
    (VTTS_TC_* / VTTS_CONV_*) must also change the launch of at least one conv of these utterances -- otherwise the case
    would silently re-run the default configuration."""
    import os
    from vosk_tts_b200.engine import Engine
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    shapes = _golden_pair_conv_shapes(e)
    if any(k.startswith(("VTTS_TC_", "VTTS_CONV_")) for k in env):
        assert shapes != default_conv_shapes, "the switch changed no conv launch"
    e.close()


def _golden_pair_conv_shapes(e):
    """Runs t128_sid2 and t17_sid2 (eager, capture, replay) against their fixtures; returns the conv launch shapes in launch
    order (an ordered list: the same shape may be right for one conv and a change for another)."""
    e.conv_log(1)
    for name in ("t128_sid2", "t17_sid2"):
        g = load_golden(name)
        c = _case(g, 0)
        T = len(c["tok"])
        for rep in range(3):          # eager, capture, replay
            ylen, dur = e.durations(c["tok"][None], [T], [c["sid"]], g["scales"], c["eps_dp"][None], want_durations=True)
            assert np.array_equal(dur[0], c["w_ceil"])
            wav = e.synthesize(ylen, c["eps_z"][None])
            assert np.abs(wav[0, : c["Ty"] * 256] - c["wav"]).max() < WAV_TIGHT
    shapes = [tuple(sorted(r.items())) for r in e.conv_log(2)]
    e.conv_log(0)
    return shapes


@pytest.fixture(scope="module")
def default_conv_shapes(packed, cfg):
    from vosk_tts_b200.engine import Engine
    e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    shapes = _golden_pair_conv_shapes(e)
    e.close()
    return shapes


def test_reserved_workspace_keeps_bucket_graphs_valid(packed, cfg):
    """Engine.reserve sizes the workspace once; afterwards a longer request must not move buffers, i.e. the CUDA graphs captured
    for shorter requests keep replaying (without the reservation every growth invalidates all of them)."""
    from vosk_tts_b200.engine import Engine
    g = torch.Generator().manual_seed(11)
    short = torch.randint(0, cfg["n_vocab"], (1, 24), generator=g).numpy()
    longer = torch.randint(0, cfg["n_vocab"], (1, 90), generator=g).numpy()
    for reserve in (True, False):
        e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
        if reserve:
            assert e.reserve(96, 512) >= 512
        ref = None
        for _ in range(3):                                   # eager + capture, then replays
            w, yl = e.infer(short, [24], [1], (0.667, 1.0, 0.8), seed=5, frames_hint=256)
            ref = w if ref is None else ref
            assert np.array_equal(w, ref)
        r0 = e.graph_replays()
        e.infer(longer, [90], [1], (0.667, 1.0, 0.8), seed=6, frames_hint=1024)      # new, larger buckets
        r1 = e.graph_replays()
        w, yl = e.infer(short, [24], [1], (0.667, 1.0, 0.8), seed=5, frames_hint=256)
        assert np.array_equal(w, ref)
        if reserve:
            assert e.graph_replays() - r1 == 2, "the short request's two graphs were invalidated by a longer request"
        e.close()


def test_plain_hifigan_resblock2_variant_vs_oracle(cfg):
    """Config-driven variant: plain HiFi-GAN `Generator` tail (conv_post + tanh, speaker projection added to conv_pre,
    models.py:845-898) with ResBlock2 (modules.py:234-258), three upsampling stages 8x8x4.  The reference's own `infer`
    cannot drive this decoder (`o, o_mb = self.dec(...)` at models.py:1703 fails to unpack the single tensor it returns),
    so the engine is compared with the oracle restatement only (fp32 path)."""
    import copy
    from oracle import vits_oracle as vo
    from vosk_tts_b200 import synthetic, weights
    from vosk_tts_b200.engine import Engine
    c2 = copy.deepcopy(cfg)
    c2.update(decoder="hifigan", resblock="2", resblock_kernel_sizes=[3, 5, 7], resblock_dilation_sizes=[[1, 2], [2, 6], [3, 9]],
              upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8], upsample_initial_channel=256, n_layers=3)
    folded = weights.fold_weight_norm(synthetic.make_random_checkpoint(c2, 77))
    blob, man = weights.pack(folded, c2)
    e = Engine(c2, blob, man, device=0, precision=0)
    assert e.hop == 256
    g = torch.Generator().manual_seed(5)
    T = 40
    tok = torch.randint(0, 62, (1, T), generator=g)
    e1, e2 = torch.randn(1, 2, T, generator=g), torch.randn(1, 192, 24 * T, generator=g)
    with torch.no_grad():
        o = vo.infer(folded, c2, tok, torch.tensor([T]), torch.tensor([4]), (0.8, 1.0, 0.8), e1, e2)
    ylen, dur = e.durations(tok.numpy(), [T], [4], (0.8, 1.0, 0.8), e1.numpy(), want_durations=True)
    assert np.array_equal(dur[0], o["w_ceil"][0, 0].numpy().astype(np.int32))
    Ty = int(ylen[0])
    wav = e.synthesize(ylen, e2[:, :, :Ty].numpy())
    assert np.abs(wav[0, : Ty * 256] - o["o"][0, 0].numpy()).max() < 2e-5
    e.close()


def test_fused_infer_equals_two_phase_and_handles_capacity(engine, cfg):
    """vtts_infer (one ABI call) == vtts_durations + vtts_synthesize; a too-small capacity falls back cleanly."""
    ids, lens, sid = _rand_batch(cfg, 3, 20, 45, 31)
    ref, yl = engine.infer(ids, lens, sid, (0.8, 1.0, 0.8), seed=11)
    w1, y1 = engine.infer(ids, lens, sid, (0.8, 1.0, 0.8), seed=11, frames_hint=int(yl.max()) + 7)
    assert np.array_equal(y1, yl) and np.array_equal(w1[:, : ref.shape[1]], ref)
    w2, y2 = engine.infer(ids, lens, sid, (0.8, 1.0, 0.8), seed=11, frames_hint=max(1, int(yl.max()) // 2))   # CAPACITY path
    assert np.array_equal(y2, yl) and np.array_equal(w2, ref)


def test_session_run_matches_reference_call_shape(packed, cfg):
    from vosk_tts_b200.session import VitsSession
    s = VitsSession(cfg=cfg, packed=packed, device=0, seed=7, precision=1)
    ids = np.random.RandomState(0).randint(0, 62, size=(1, 40)).astype(np.int64)
    feeds = {"input": ids, "input_lengths": np.array([40], np.int64), "scales": np.array([0.8, 1.0, 0.8], np.float32),
             "sid": np.array([2], np.int64), "bert": None, "phone_duration_extra": None}
    out = s.run(None, feeds)[0]
    assert out.dtype == np.float32 and out.ndim == 4 and out.shape[:3] == (1, 1, 1)
    assert out.shape[3] == int(s.last_y_lengths[0]) * 256
    s.close()


@pytest.mark.parametrize("precision", [0, 1])
def test_plain_coupling_flow_variant_vs_reference_fixture(precision):
    """use_transformer_flows=False (plain ResidualCouplingLayer + Flip == ResidualCouplingBlock, models.py:765-810,
    vc/modules.py:300-345) against the fixture the unmodified reference produced with that flag."""
    import copy
    import json
    from vosk_tts_b200 import config as C, synthetic, weights
    from vosk_tts_b200.engine import Engine
    g = load_golden("plainflow_t40")
    cfg = copy.deepcopy(C.DEFAULT_CONFIG)
    cfg.update(json.loads(str(g["model_overrides"])))
    w = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, int(g["weight_seed"])))
    blob, man = weights.pack(w, cfg)
    eng = Engine(cfg, blob, man, device=0, precision=precision)
    try:
        c = _case(g, 0)
        T = len(c["tok"])
        eng.debug_flags(1)
        ylen, dur = eng.durations(c["tok"][None], [T], [c["sid"]], g["scales"], c["eps_dp"][None], want_durations=True)
        assert int(ylen[0]) == c["Ty"]
        assert np.array_equal(dur[0], c["w_ceil"])
        wav, idx = eng.synthesize(ylen, c["eps_z"][None], want_alignment=True)
        assert np.array_equal(idx[0, : c["Ty"]], c["idx"])
        z = eng.debug_read("z").reshape(c["Ty"], -1)
        assert np.abs(z - c["z"].T).max() < 3e-4
        assert np.abs(wav[0, : c["Ty"] * 256] - c["wav"]).max() < WAV_TIGHT
    finally:
        eng.close()


@pytest.mark.parametrize("decoder", ["ms_istft", "istft"])
@pytest.mark.parametrize("precision", [0, 1])
def test_istft_decoder_variants_vs_oracle(decoder, precision):
    """Multistream_iSTFT_Generator (learned 63-tap merge filter, conv_post with bias; models.py:1066-1169) and iSTFT_Generator
    (one band, no filter bank; models.py:901-971) at full width against the oracle (which tests/test_decoder_variants.py
    pins against the unmodified reference on CPU)."""
    import copy
    from oracle import vits_oracle as vo
    from vosk_tts_b200 import config as C, synthetic, weights
    from vosk_tts_b200.engine import Engine
    cfg = copy.deepcopy(C.DEFAULT_CONFIG)
    cfg["decoder"] = decoder
    if decoder == "istft":
        cfg["subbands"] = 1
    w = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 4321))
    blob, man = weights.pack(w, cfg)
    eng = Engine(cfg, blob, man, device=0, precision=precision)
    try:
        g = torch.Generator().manual_seed(8)
        for T in (21, 70):
            tok = torch.randint(0, cfg["n_vocab"], (1, T), generator=g)
            eps_dp = torch.randn(1, 2, T, generator=g)
            ylen, dur = eng.durations(tok.numpy(), [T], [4], (0.8, 1.0, 0.8), eps_dp.numpy(), want_durations=True)
            Ty = int(ylen[0])
            eps_z = torch.randn(1, 192, Ty, generator=g)
            with torch.no_grad():
                o = vo.infer(w, cfg, tok, torch.tensor([T]), torch.tensor([4]), (0.8, 1.0, 0.8), eps_dp, eps_z)
            assert Ty == int(o["y_lengths"][0]) and np.array_equal(dur[0], o["w_ceil"][0, 0].numpy().astype(np.int32))
            wav = eng.synthesize(ylen, eps_z.numpy())
            hop = C.hop_total(cfg)
            assert eng.hop == hop and o["o"].shape[-1] == Ty * hop
            ref = o["o"][0, 0].numpy()
            err = np.abs(wav[0, : Ty * hop] - ref).max()
            assert err < WAV_TOL * max(1.0, float(np.abs(ref).max())), (decoder, precision, T, err, float(np.abs(ref).max()))
    finally:
        eng.close()
