"""Forced alignment on the GPU (vtts_align / vtts_align_spec): the neg_cent kernel alone against a float64 restatement, the MAS
plumbing against mas_oracle, reuse of the TTS encoder and of the conversion's posterior side, the reference's stored
SynthesizerTrn.forward alignment (tests/golden/ref_alignment.npz), ragged batches, repeatability and refusals.

neg_cent error bound (neg_cent_kernel, csrc/mas.cuh).  Per cell the kernel sums, in fp32, I quadratic terms
t_d = (q_d * s'_d) * q_d with q_d = z_d - m_d and s'_d = -0.5 expf(-2 logs_d), then adds c = sum_d (-0.5 log 2pi - logs_d),
itself an fp32 sum of I terms.  With u = 2^-24: q_d carries a relative error <= u, s'_d <= 2 ulp of expf + u (<= 3u), the
product and the FMA <= 2u, so each t_d is within 6u |t_d| of its exact value; accumulating I terms adds <= I u sum|t_d|, the
c sum <= I u sum_d |0.5 log 2pi + logs_d|, the final add u (|c| + |acc|).  Hence
    |gpu - exact| <= (I + 8) * 2^-23 * S,   S = sum_d (|0.5 log 2pi + logs_d| + 0.5 (z_d - m_d)^2 exp(-2 logs_d)),
with z, m, logs the engine's own fp32 z_p and stats (read back), exact = the float64 restatement (align_oracle.neg_cent).
The kernel is fp32 FFMA in every precision mode; the large shapes (t_x 2048, t_y 4000) run in mode 1 only, the rest in all four.
"""
import copy
import ctypes as C

import numpy as np
import pytest

import align_inputs as AI
import golden_ref as GR
import vc_inputs as VI
from oracle import align_oracle as ao, mas_oracle
from vosk_tts_b200 import config as CF, synthetic, weights

pytestmark = pytest.mark.gpu

SEQ_GAP = 8
PRECISIONS = [0, 1, 2, 3]
_PACKED, _ENGINES = {}, {}
CASES = {c[0]: c for c in AI.CASES}


def _cfg(model):
    return CF.from_training_json(AI.training_json(model), n_vocab=AI.n_vocab(model))


def _packed(model):
    if model not in _PACKED:
        cfg = _cfg(model)
        sd = synthetic.make_random_checkpoint(cfg, AI.SEEDS[model], posterior=True)
        _PACKED[model] = (cfg,) + weights.pack(weights.fold_weight_norm(sd), cfg, posterior=True)
    return _PACKED[model]


def _engine(model, precision):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if precision > 0 and not weights.tc_supported(_cfg(model)):
        pytest.skip("tiny widths: no tensor-core path")
    from vosk_tts_b200.engine import Engine
    key = (model, precision)
    if key not in _ENGINES:
        cfg, blob, man = _packed(model)
        _ENGINES[key] = Engine(cfg, blob, man, device=0, precision=precision)
    return _ENGINES[key]


def teardown_module(module):
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(np.asarray(lens) + SEQ_GAP)])[:-1].astype(np.int64)


def _run(e, ids, lens, sid, x, xl=None, spec=False, **kw):
    """One alignment with the debug read-backs: returns the call's outputs plus neg_cent [B, max t_y, max t_x] (NaN outside
    the utterances), z_p rows [frames + gaps, I] and stats rows [tokens + gaps, 2I]."""
    I = e.cfg["inter_channels"]
    e.debug_flags(1)
    try:
        dur, fr, tof, score = (e.align_spec if spec else e.align)(ids, lens, sid, x, xl, **kw)
        B = len(fr)
        nc = e.debug_read("align_neg_cent").reshape(B, int(fr.max()), -1)
        zp = e.debug_read("vc_z_p").reshape(-1, I)
        st = e.debug_read("stats").reshape(-1, 2 * I)
    finally:
        e.debug_flags(0)
    return dict(dur=dur, frames=fr, tof=tof, score=score, nc=nc, zp=zp, stats=st)


def _operands(r, lens, b):
    I = r["zp"].shape[1]
    fo, to = _offsets(r["frames"]), _offsets(lens)
    t_y, t_x = int(r["frames"][b]), int(lens[b])
    z = r["zp"][fo[b]:fo[b] + t_y].T
    m = r["stats"][to[b]:to[b] + t_x, :I].T
    lg = r["stats"][to[b]:to[b] + t_x, I:].T
    return z, m, lg


def _bound(z, m, lg):
    z, m, lg = (np.asarray(a, np.float64) for a in (z, m, lg))
    S = np.abs(0.5 * np.log(2 * np.pi) + lg).sum(0)[None, :].repeat(z.shape[1], 0)
    s = np.exp(-2 * lg)
    for d in range(z.shape[0]):
        q = z[d][:, None] - m[d][None, :]
        S += 0.5 * q * q * s[d][None, :]
    return (z.shape[0] + 8) * 2.0 ** -23 * S


def _check_call(r, lens):
    """neg_cent within the bound of its float64 restatement on the engine's own operands, NaN (never written) outside the
    utterances; token_of_frame / durations / score equal mas_oracle on the read-back neg_cent, bit for bit; sentinels."""
    lens = np.asarray(lens)
    worst = 0.0
    for b in range(len(lens)):
        t_y, t_x = int(r["frames"][b]), int(lens[b])
        z, m, lg = _operands(r, lens, b)
        gpu = r["nc"][b, :t_y, :t_x].astype(np.float64)
        err = np.abs(gpu - ao.neg_cent(z, m, lg))
        bnd = _bound(z, m, lg)
        assert (err <= bnd).all(), (b, float((err / bnd).max()))
        worst = max(worst, float((err / bnd).max()))
        assert np.isnan(r["nc"][b, t_y:]).all() and np.isnan(r["nc"][b, :, t_x:]).all()
        nc32 = r["nc"][b:b + 1, :t_y, :t_x]
        path = mas_oracle.maximum_path_vectorised(nc32, [t_y], [t_x])[0]
        tof, dur = ao.path_of(path)
        assert np.array_equal(r["tof"][b, :t_y], tof) and np.array_equal(r["dur"][b, :t_x], dur)
        assert dur.min() >= 1 and dur.sum() == t_y
        s = np.float32(0)
        for y in range(t_y):
            s = np.float32(nc32[0, y, tof[y]] + s)
        assert r["score"][b] == s
        assert not r["dur"][b, t_x:].any() and (r["tof"][b, t_y:] == -1).all()
    return worst


def _seeded(e, shapes, seed):
    """ids [B, max t_x] and seeded features [B, spec_channels, max t_y] for (t_x, t_y) per utterance."""
    rng = np.random.RandomState(seed)
    B = len(shapes)
    tx = np.array([s[0] for s in shapes])
    ty = np.array([s[1] for s in shapes])
    ids = rng.randint(1, e.cfg["n_vocab"], size=(B, tx.max())).astype(np.int64)
    ids[:, 1::2] = 0
    spec = (rng.randn(B, e.cfg["spec_channels"], ty.max()) * 2 - 4).astype(np.float32)
    return ids, tx, spec, ty


SHAPES = {
    "tx1": [(1, 1)], "tx2": [(2, 2)], "tx2_long": [(2, 37)], "tx63": [(63, 63)], "tx64": [(64, 200)], "tx65": [(65, 1000)],
    "tx200": [(200, 700)], "ragged5": [(1, 40), (63, 64), (64, 300), (65, 65), (200, 777)],
}
LARGE = {"tx200_4000": [(200, 4000)], "tx2048": [(2048, 2048)], "tx2048_4000": [(2048, 4000)]}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_neg_cent_and_mas_plumbing(name, precision):
    e = _engine("mel", precision)
    ids, tx, spec, ty = _seeded(e, SHAPES[name], 7)
    r = _run(e, ids, tx, np.arange(len(tx)) % 10, spec, ty, spec=True, seed=3)
    print("%s precision %d: max err / bound %.3f" % (name, precision, _check_call(r, tx)))


@pytest.mark.parametrize("name", list(LARGE))
def test_neg_cent_large(name):
    e = _engine("mel", 1)
    ids, tx, spec, ty = _seeded(e, LARGE[name], 8)
    r = _run(e, ids, tx, [4], spec, ty, spec=True, seed=3)
    print("%s: max err / bound %.3f" % (name, _check_call(r, tx)))


def test_neg_cent_batch64():
    e = _engine("mel", 1)
    rng = np.random.RandomState(9)
    tx = rng.randint(1, 201, size=64)
    shapes = [(int(t), int(t + rng.randint(0, 400))) for t in tx]
    ids, tx, spec, ty = _seeded(e, shapes, 10)
    r = _run(e, ids, tx, np.arange(64) % 200, spec, ty, spec=True, seed=3)
    print("batch 64: max err / bound %.3f" % _check_call(r, tx))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("B", [1, 3])
def test_stats_equal_tts_phase1_bitwise(B, precision):
    e = _engine("mel", precision)
    ids, tx, spec, ty = _seeded(e, [(45, 112), (17, 30), (80, 90)][:B], 11)
    sid = np.array([3, 9, 0][:B])
    e.debug_flags(1)
    try:
        e.durations(ids, tx, sid, (0.667, 1.0, 0.8), np.zeros((B, 2, ids.shape[1]), np.float32))
        tts = e.debug_read("stats")
        e.align_spec(ids, tx, sid, spec, ty)
        al = e.debug_read("stats")
    finally:
        e.debug_flags(0)
    I = e.cfg["inter_channels"]
    for b, o in enumerate(_offsets(tx)):
        rows = slice(int(o) * 2 * I, (int(o) + int(tx[b])) * 2 * I)
        assert np.array_equal(tts[rows], al[rows])


@pytest.mark.parametrize("precision", PRECISIONS)
def test_z_p_equals_conversion_bitwise(precision):
    e = _engine("mel", precision)
    wav = VI.wav_float(VI.speech()["b"])
    I = e.cfg["inter_channels"]
    eps = VI.eps_q("c1", I, len(wav) // 256).numpy()
    e.debug_flags(1)
    try:
        e.convert(wav, 5, 7, noise=eps)
        zc = e.debug_read("vc_z_p")
        e.align(AI.ids("a1"), 45, 5, wav, noise=eps)
        za = e.debug_read("vc_z_p")
    finally:
        e.debug_flags(0)
    assert np.array_equal(zc, za)


def _ref():
    return GR.load("ref_alignment.npz")


def _against_reference(r, case, t_x):
    """delta = max |GPU neg_cent - float64 neg_cent of the reference's z_p / m_p / logs_p| plus the fp32 accumulation bound of
    MAS per step; the GPU path's float64 score (on the reference's neg_cent) is within 2 t_y delta of the reference path's,
    and where the reference's 2-best margin exceeds that, path and durations are the reference's."""
    ref = _ref()
    p = case + "/"
    t_y = int(r["frames"][0])
    nc_ref = ao.neg_cent(ref[p + "z_p"], ref[p + "m_p"], ref[p + "logs_p"])
    gpu = r["nc"][0, :t_y, :t_x].astype(np.float64)
    delta = float(np.abs(gpu - nc_ref).max()) + t_y * 2.0 ** -24 * float(np.abs(gpu).max())
    s_gpu, s_ref = ao.path_score(nc_ref, r["tof"][0, :t_y]), ao.path_score(nc_ref, ref[p + "token_of_frame"])
    assert s_gpu >= s_ref - 2 * t_y * delta and s_gpu <= s_ref + 1e-9 * abs(s_ref) + 2 * t_y * delta
    margin = float(ref[p + "margin"])
    same = margin > 2 * t_y * delta
    if same:
        assert np.array_equal(r["tof"][0, :t_y], ref[p + "token_of_frame"]) and np.array_equal(r["dur"][0, :t_x], ref[p + "w"])
    return delta, margin, same


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("from_spec", [True, False])
@pytest.mark.parametrize("case", list(CASES))
def test_matches_reference(case, from_spec, precision):
    _, clip, model, sid, _ = CASES[case]
    e = _engine(model, precision)
    ref = _ref()
    ids = AI.ids(case)
    I = e.cfg["inter_channels"]
    t_y = AI.frames(clip)
    eps = AI.eps_q(case, I, t_y).numpy()
    x = AI.ref_spec(case)[None] if from_spec else VI.wav_float(VI.speech()[clip])[None]
    r = _run(e, ids[None], [len(ids)], sid, x, spec=from_spec, noise=eps)
    assert int(r["frames"][0]) == t_y
    zp = r["zp"][:t_y].T
    err = float(np.abs(zp - ref[case + "/z_p"]).max())
    _check_call(r, [len(ids)])
    delta, margin, same = _against_reference(r, case, len(ids))
    print("%s spec=%d precision %d: z_p err %.2e delta %.3e margin %.3f identical-path required %s"
          % (case, from_spec, precision, err, delta, margin, same))
    assert err <= 2e-3 * max(1.0, float(np.abs(ref[case + "/z_p"]).max())), err


@pytest.mark.parametrize("precision", PRECISIONS)
def test_ragged_batch_vs_single_clips(precision):
    e = _engine("mel", precision)
    cases = ["a0", "a1", "a2"]
    sp = VI.speech()
    clips = [VI.wav_float(sp[CASES[c][1]]) for c in cases]
    I = e.cfg["inter_channels"]
    L = max(len(c) for c in clips)
    wav = np.zeros((3, L + 100), np.float32)
    for i, c in enumerate(clips):
        wav[i, :len(c)] = c
    wl = np.array([len(c) for c in clips])
    idl = [AI.ids(c) for c in cases]
    tx = np.array([len(i) for i in idl])
    ids = np.zeros((3, tx.max()), np.int64)
    for i, v in enumerate(idl):
        ids[i, :len(v)] = v
    sid = np.array([CASES[c][3] for c in cases])
    eps = np.random.RandomState(4).randn(3, I, L // 256 + 3).astype(np.float32)
    rb = _run(e, ids, tx, sid, wav, wl, noise=eps)
    _check_call(rb, tx)
    for i in range(3):
        t_y = int(rb["frames"][i])
        r1 = _run(e, idl[i][None], [tx[i]], sid[i], clips[i][None], noise=eps[i:i + 1, :, :t_y])
        nb, n1 = rb["nc"][i, :t_y, :tx[i]].astype(np.float64), r1["nc"][0, :t_y, :tx[i]].astype(np.float64)
        delta = float(np.abs(nb - n1).max()) + t_y * 2.0 ** -24 * float(np.abs(n1).max())
        s_b, s_1 = ao.path_score(n1, rb["tof"][i, :t_y]), ao.path_score(n1, r1["tof"][0, :t_y])
        assert abs(s_b - s_1) <= 2 * t_y * delta
        best, second = ao.two_best(n1, t_y, int(tx[i]))
        if best - second > 2 * t_y * delta:
            assert np.array_equal(rb["tof"][i, :t_y], r1["tof"][0, :t_y])
            assert np.array_equal(rb["dur"][i, :tx[i]], r1["dur"][0, :tx[i]])


def test_graph_replay_equals_eager_bitwise():
    e = _engine("mel", 1)
    wav = VI.wav_float(VI.speech()["b"])
    ids = AI.ids("a1")
    e.set_graphs(False)
    eager = e.align(ids, 45, 5, wav, seed=11)
    e.set_graphs(True)
    r0 = e.graph_replays()
    first = e.align(ids, 45, 5, wav, seed=11)                     # eager run + capture
    second = e.align(ids, 45, 5, wav, seed=11)                    # replay
    assert e.graph_replays() > r0
    for a, b, c in zip(eager, first, second):
        assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_seeds(precision):
    e = _engine("mel", precision)
    wav = VI.wav_float(VI.speech()["a"])
    ids = AI.ids("a1")
    a = e.align(ids, 45, 3, wav, seed=5)
    b = e.align(ids, 45, 3, wav, seed=5)
    c = e.align(ids, 45, 3, wav, seed=6)
    d = e.align(ids, 45, 3, wav, seed=6, noise_scale=0.0)
    f = e.align(ids, 45, 3, wav, seed=7, noise_scale=0.0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert a[3][0] != c[3][0]
    assert all(np.array_equal(x, y) for x, y in zip(d, f))


def _code(fn):
    from vosk_tts_b200.engine import VttsError
    with pytest.raises(VttsError) as ei:
        fn()
    return ei.value.code, str(ei.value)


def test_refusals():
    e = _engine("mel", 0)
    wav = VI.wav_float(VI.speech()["b"])                           # 112 frames
    ids = AI.ids("a1")
    bad = ids.copy()
    bad[3] = 62
    assert _code(lambda: e.align(bad, 45, 5, wav))[0] == -1                       # id out of [0, n_vocab)
    assert _code(lambda: e.align(ids, 45, 200, wav))[0] == -1                     # speaker out of range
    assert _code(lambda: e.align(ids, 45, -1, wav))[0] == -1
    assert _code(lambda: e.align(ids[:1], 1, 5, wav[:384]))[0] == -1              # reflect padding needs > 384 samples
    dur, fr, tof, score = e.align(ids[:1], 1, 5, wav[:385])
    assert int(fr[0]) == 1 and int(dur[0, 0]) == 1 and tof.tolist() == [[0]]
    assert _code(lambda: e.align(ids, 0, 5, wav))[0] == -1                        # t_x < 1
    long_ids = np.tile(ids, 3)[:113]
    code, msg = _code(lambda: e.align(long_ids, 113, 5, wav))                     # t_x > t_y
    assert code == -1 and "frames" in msg
    e.align(long_ids[:112], 112, 5, wav)                                          # t_x == t_y: the forced path
    big = np.tile(ids, 50)[:2049]
    code, msg = _code(lambda: e.align(big, 2049, 5, np.zeros(2100 * 256, np.float32)))
    assert code == -1 and "2048" in msg
    # capacities
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    ids2 = np.ascontiguousarray(ids[None])
    il, wl, s = np.array([45], np.int64), np.array([len(wav)], np.int64), np.array([5], np.int64)
    dur, tof, fr = np.zeros((1, 45), np.int32), np.zeros(200, np.int32), np.zeros(1, np.int64)
    assert e.lib.vtts_align(e.h, P(ids2), P(il), 45, P(s), P(wav), P(wl), 1, len(wav), 1.0, None, 0, 0, P(dur), P(tof), 100, None,
                            P(fr)) == -4
    eps = np.zeros((1, e.cfg["inter_channels"], 100), np.float32)
    assert e.lib.vtts_align(e.h, P(ids2), P(il), 45, P(s), P(wav), P(wl), 1, len(wav), 1.0, P(eps), 100, 0, P(dur), None, 0, None,
                            P(fr)) == -4


def test_refused_models():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200 import onnx_weights
    from vosk_tts_b200.engine import Engine
    import os
    wav = VI.wav_float(VI.speech()["b"])
    ids = AI.ids("a3")
    cfg = _cfg("lin")
    sd = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, AI.SEEDS["lin"], posterior=True))
    blob, man = weights.pack(sd, cfg)                                             # TTS blob: no enc_q
    e = Engine(cfg, blob, man, precision=0)
    code, msg = _code(lambda: e.align(ids, len(ids), 1, wav))
    assert code == -1 and "posterior=True" in msg
    e.close()
    path = os.path.join(GR.GOLDEN, "tiny_model.onnx")
    ocfg = onnx_weights.config_from_onnx(path)
    oblob, oman = weights.pack(onnx_weights.state_dict_from_onnx(path), ocfg)
    e = Engine(ocfg, oblob, oman, precision=0)
    code, msg = _code(lambda: e.align(ids % ocfg["n_vocab"], len(ids), 0, wav))
    assert code == -1 and "enc_q" in msg
    e.close()
    c3 = copy.deepcopy(cfg)
    c3["flow_n_flows"] = 3
    b3, m3 = weights.pack(weights.fold_weight_norm(synthetic.make_random_checkpoint(c3, 3)), c3)
    e = Engine(c3, b3, m3, precision=0)
    code, msg = _code(lambda: e.align(ids, len(ids), 1, wav))
    assert code == -1 and "flow_n_flows" in msg
    e.close()
    # the single-speaker model aligns, and voice conversion still refuses it
    e = _engine("single", 0)
    dur, fr, _, _ = e.align(AI.ids("a4"), 41, None, wav)
    assert int(dur.sum()) == int(fr[0]) == 112
    assert _code(lambda: e.convert(wav, 0, 0))[0] == -1
