"""GPU (-m gpu): the normalisation kernels and the passes beside them, one launch at a time through the engine's own launch
helpers, against the float64 references and error bounds of tests/norm_ref.py:
  vtts_debug_add_ln       add_ln_kernel (add_ln: VITS text encoder, FFMA and tensor-core, and the transformer flows)
  vtts_debug_ln           cv_ln_kernel (ln_rows: ContentVec, HuBERT, BERT and StableTTS text encoder layers)
  vtts_debug_bert_embed   bert_embed_kernel (bt_embed)
  vtts_debug_dit_norm     dit_norm_kernel / dit_norm_planes_kernel (dit_norm: the StableTTS blocks)
  vtts_debug_act          cv_gelu_kernel (gelu_rows), dit_silu_kernel / dit_silu_planes_kernel (silu_rows)
  vtts_debug_gate         dit_gate_kernel / dit_gate_planes_kernel (gate_rows)
  vtts_debug_groupnorm    cv_stage, then the three cv_gn_kernel passes (cv_layer0) with a ContentVec engine's weights
Every case runs twice and must give the same bits, and each utterance must give the same bits alone and in its batch.  Input
rows outside the utterances are NaN, so a stray read shows; output rows and planes outside them hold a sentinel that must
survive.  Planes must be the device split of the fp32 value the kernel wrote, bit for bit, and a *_planes kernel must write
the fp32 rows of its plain twin bit for bit."""
import json

import numpy as np
import pytest
import torch

import contentvec_inputs as CI
import norm_ref as N
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from vosk_tts_b200 import weights
from vosk_tts_b200.engine import Engine, VttsError

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
PSENT = np.uint16(0x7777)
WORST = {}                                 # largest error / bound seen per kernel
RAGGED = [1, 3, 4, 5, 8, 9, 17, 37]        # lengths around 4 (add_ln) and 8 (the others) rows per CTA
LONG = [2000, 1, 513]
B64 = list(np.random.default_rng(64).integers(1, 70, 64))
BATCHES = {"ragged": RAGGED, "long": LONG, "b64": B64}


def _note(kernel, r):
    WORST[kernel] = max(WORST.get(kernel, 0.0), float(r))


@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cfg = dict(QI.config())
    cfg["contentvec"] = CI.cv()
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    e = Engine(cfg, blob, man, device=0, precision=0)
    yield e
    e.close()
    print("\nnormalisation kernels error / bound, largest per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


# ---------------------------------------------------------------------------------------------------- row layout
def _layout(lens):
    off = N.offsets(lens)
    valid = np.zeros(off[-1], bool)
    for b, n in enumerate(lens):
        valid[off[b]:off[b] + n] = True
    return off, valid


def _inputs(lens, C_, seed, width=None):
    """Mixed-kind rows [rows, width or C_] (kinds cycle per row), NaN outside the utterances and in columns >= C_."""
    off, valid = _layout(lens)
    x = N.mixed_rows(off[-1], width or C_, np.random.default_rng(seed))
    x[~valid] = np.nan
    x[:, C_:] = np.nan
    return x


def _sent(rows, C_):
    return np.full((rows, C_), SENT, np.float32)


def _psent(rows, C_):
    return np.full((rows, C_), PSENT, np.uint16)


def _check_outside(valid, *arrays, cols=None):
    for a in arrays:
        if a is None:
            continue
        s = PSENT if a.dtype == np.uint16 else SENT
        assert np.all(a[~valid] == s), "a row outside the utterances was written"
        if cols is not None:
            assert np.all(a[:, cols:] == s), "a column past C was written"


def _check_planes(out, valid, hi, lo, mid=None, C_=None):
    """Planes == the device split of the fp32 rows the kernel wrote (columns < C_), bit for bit."""
    if hi is None:
        return
    o = out[valid][:, :C_]
    if mid is None:
        h, l_ = N.split_bf16(o)
        assert np.array_equal(hi[valid][:, :C_], h) and np.array_equal(lo[valid][:, :C_], l_)
    else:
        h, m, l_ = N.split_bf16_3(o)
        assert np.array_equal(hi[valid][:, :C_], h) and np.array_equal(mid[valid][:, :C_], m) and np.array_equal(lo[valid][:, :C_], l_)
        val = lambda p: (p.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
        assert np.array_equal(val(hi[valid][:, :C_]) + val(mid[valid][:, :C_]) + val(lo[valid][:, :C_]), o.astype(np.float64))


def _same(a, b, what="two runs differ"):
    for x, y in zip(a, b):
        if x is not None:
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what


def _per_row(lens):
    """Each valid row's utterance index."""
    return np.concatenate([np.full(n, b) for b, n in enumerate(lens)])


# ---------------------------------------------------------------------------------------------------- add_ln_kernel
ADD_LN_OPTS = [(c, v, p) for c in (0, 1) for v in (0, 1) for p in (0, 2, 3)]


@pytest.mark.parametrize("C_", [32, 96, 192, 256])
@pytest.mark.parametrize("cadd,vec,planes", ADD_LN_OPTS)
def test_add_ln(eng, C_, cadd, vec, planes):
    rng = np.random.default_rng(C_ * 10 + cadd * 4 + vec * 2 + planes)
    g, beta = N.affine(C_, rng)
    for name, lens in BATCHES.items():
        off, valid = _layout(lens)
        rows, B = off[-1], len(lens)
        a, b = _inputs(lens, C_, 1 + C_), _inputs(lens, C_, 2 + C_)
        ca = _inputs(lens, C_, 3 + C_) if cadd else None
        vv = rng.standard_normal((B, C_ + 8)).astype(np.float32) if vec else None

        def run(lens_, s, vrow):
            n = s.stop - s.start
            pl = [_psent(n, C_) if planes else None, _psent(n, C_) if planes == 3 else None, _psent(n, C_) if planes else None]
            return eng.debug_add_ln(lens_, a[s], g, beta, _sent(n, C_), b=b[s], cadd=ca[s] if cadd else None,
                                    vec=vv[vrow] if vec else None, hi=pl[0], mid=pl[1], lo=pl[2])

        res = run(lens, slice(0, rows), slice(0, B))
        _same(res, run(lens, slice(0, rows), slice(0, B)))
        out, hi, mid, lo = res
        _check_outside(valid, out, hi, mid, lo)
        _check_planes(out, valid, hi, lo, mid, C_)
        utt = _per_row(lens)
        ref, bound = N.add_ln(a[valid], b[valid], g, beta, ca[valid] if cadd else None, vv[utt, :C_] if vec else None)
        r = N.within(out[valid], ref, bound)
        _note("add_ln_kernel", r)
        assert r <= 1, (name, r)
        for u in (0, B - 1):
            s = slice(off[u], off[u] + lens[u])
            for x_, y_ in zip(res, run([lens[u]], s, slice(u, u + 1))):
                if x_ is not None:
                    assert np.array_equal(x_[s].view(np.uint8), y_.view(np.uint8)), "alone != batched"


def test_add_ln_refusals(eng):
    for C_ in (48, 288, 16):
        x = np.zeros((4, C_), np.float32)
        with pytest.raises(VttsError, match="multiple of 32"):
            eng.debug_add_ln([4], x, np.ones(C_), np.zeros(C_), x.copy())


# ---------------------------------------------------------------------------------------------------- cv_ln_kernel
@pytest.mark.parametrize("C_", [48, 144, 512, 768, 1008, 1024])
@pytest.mark.parametrize("with_y", [False, True])
@pytest.mark.parametrize("eps", [1e-5, 1e-12])
@pytest.mark.parametrize("planes", [False, True])
def test_cv_ln(eng, C_, with_y, eps, planes):
    rng = np.random.default_rng(C_ + 7 * with_y + planes)
    g, beta = N.affine(C_, rng)
    for name, lens in BATCHES.items():
        if name == "b64" and (planes or eps == 1e-12):
            continue
        off, valid = _layout(lens)
        a = _inputs(lens, C_, 5 + C_)
        const = np.flatnonzero(valid) % len(N.ROW_KINDS) == N.ROW_KINDS.index("constant")
        y = np.clip(_inputs(lens, C_, 6 + C_), -30, 30) if with_y else None
        if with_y:                  # gelu(0) = 0: the constant rows of a stay constant, with a sum that is exact
            y[np.flatnonzero(valid)[const]] = 0
        # output rows: the utterances in reverse order, 3 rows apart, after 5 leading rows
        B = len(lens)
        oo = np.zeros(B, np.int32)
        pos = 5
        for b in reversed(range(B)):
            oo[b] = pos
            pos += lens[b] + 3
        ovalid = np.zeros(pos, bool)
        for b in range(B):
            ovalid[oo[b]:oo[b] + lens[b]] = True

        def run(lens_, aa, yy, oo_, rows):
            return eng.debug_ln(lens_, aa, g, beta, eps, oo_, _sent(rows, C_), y=yy, hi=_psent(rows, C_) if planes else None,
                                lo=_psent(rows, C_) if planes else None)

        out, hi, lo = run(lens, a, y, oo, pos)
        _same((out, hi, lo), run(lens, a, y, oo, pos))
        _check_outside(ovalid, out, hi, lo)
        _check_planes(out, ovalid, hi, lo, None, C_)
        order = np.concatenate([np.arange(oo[b], oo[b] + lens[b]) for b in range(B)])
        ref, bound = N.cv_ln(a[valid], y[valid] if with_y else None, g, beta, eps)
        r = N.within(out[order], ref, bound)
        _note("cv_ln_kernel", r)
        assert r <= 1, (name, r)
        # the constant rows: variance 0, so the output is beta exactly (with eps 1e-12 the bound cannot cover them: a mean
        # error of one rounding would be 10^6 sigma); every other row has a finite bound
        assert np.all(np.isfinite(bound[~const])), "a row the bound does not cover"
        assert np.array_equal(out[order][const], np.broadcast_to(beta, (const.sum(), C_))), "a constant row is not beta"
        for b in (0, B - 1):
            s = slice(off[b], off[b] + lens[b])
            o1, h1, l1 = run([lens[b]], a[s], y[s] if with_y else None, [0], lens[b])
            assert np.array_equal(o1.view(np.uint8), out[oo[b]:oo[b] + lens[b]].view(np.uint8)), "alone != batched"


def test_cv_ln_refusals(eng):
    x = np.zeros((2, 1040), np.float32)
    with pytest.raises(VttsError, match="1024"):
        eng.debug_ln([2], x, np.ones(1040), np.zeros(1040), 1e-5, [0], x.copy())


# ---------------------------------------------------------------------------------------------------- bert_embed_kernel
@pytest.mark.parametrize("C_", [48, 144, 512, 768, 1008, 1024])
@pytest.mark.parametrize("planes", [False, True])
def test_bert_embed(eng, C_, planes):
    P = 40
    word, pos, type0, (g, beta) = N.bert_tables(C_, P, C_)
    V = word.shape[0]
    for lens in ([P, 1, 7, 8, 9, 33], B64 if not planes else [3, 40]):
        lens = [min(int(n), P) for n in lens]
        off, valid = _layout(lens)
        rows = off[-1]
        ids = np.random.default_rng(C_ + len(lens)).integers(0, V, rows).astype(np.int32)
        ids[0], ids[off[1]] = 0, V - 1
        ids[~valid] = -1            # not a piece: the kernel must not read these

        def run(lens_, ids_):
            n = len(ids_)
            return eng.debug_bert_embed(lens_, np.where(ids_ < 0, 0, ids_), word, pos, type0, g, beta, 1e-12, _sent(n, C_),
                                        hi=_psent(n, C_) if planes else None, lo=_psent(n, C_) if planes else None)

        out, hi, lo = run(lens, ids)
        _same((out, hi, lo), run(lens, ids))
        _check_outside(valid, out, hi, lo)
        _check_planes(out, valid, hi, lo, None, C_)
        t, rws = N.bert_positions(lens)
        ref, bound = N.bert_embed(ids[rws], t, word, pos, type0, g, beta, 1e-12)
        r = N.within(out[rws], ref, bound)
        _note("bert_embed_kernel", r)
        assert r <= 1, r
        # sentence 1 starts with piece V - 1 at position 0: a row of variance 0, whose output is beta exactly
        assert np.array_equal(out[off[1]], beta), "a row of variance 0 is not beta"
        for b in (0, len(lens) - 1):
            o1, _, _ = run([lens[b]], ids[off[b]:off[b] + lens[b]])
            assert np.array_equal(o1.view(np.uint8), out[off[b]:off[b] + lens[b]].view(np.uint8)), "alone != batched"


def test_bert_embed_refusals(eng):
    word, pos, type0, (g, beta) = N.bert_tables(48, 4, 1)
    out = _sent(5, 48)
    with pytest.raises(VttsError, match="outside the table"):
        eng.debug_bert_embed([5], np.array([0, 1, 60, 2, 3], np.int32), word, np.pad(pos, ((0, 1), (0, 0))), type0, g, beta, 1e-12, out)
    with pytest.raises(VttsError, match="position table"):
        eng.debug_bert_embed([5], np.zeros(5, np.int32), word, pos, type0, g, beta, 1e-12, out)
    w = np.zeros((3, 1056), np.float32)
    with pytest.raises(VttsError, match="1024"):
        eng.debug_bert_embed([1], np.zeros(1, np.int32), w, w, w[0], w[0], w[0], 1e-12, np.zeros((1, 1056), np.float32))


# ---------------------------------------------------------------------------------------------------- dit_norm(_planes)_kernel
DIT_OPTS = [(True, False), (False, True), (False, False)]     # (FiLM, y): the decoder's first norm, the second, a text block


@pytest.mark.parametrize("C_", [48, 192, 208, 512])
@pytest.mark.parametrize("film_on,y_on", DIT_OPTS)
@pytest.mark.parametrize("pad", [0, 16])
def test_dit_norm(eng, C_, film_on, y_on, pad):
    rng = np.random.default_rng(C_ + 3 * film_on + 5 * y_on + pad)
    film = np.concatenate(N.affine(C_, rng)) if film_on else None
    gate_off, shift_off, scale_off = (2 * C_, 3 * C_, 4 * C_) if y_on else (2 * C_, 0, C_)
    for name, lens in BATCHES.items():
        off, valid = _layout(lens)
        rows, B = off[-1], len(lens)
        a = _inputs(lens, C_, 8 + C_, C_ + pad)
        y = _inputs(lens, C_, 9 + C_) if y_on else None
        if y is not None:
            y = np.clip(y, -1e3, 1e3)
        ada = (0.5 * np.random.default_rng(10 + C_).standard_normal((B, 6 * C_ + 8))).astype(np.float32)

        def run(lens_, aa, yy, ad, planes):
            n = aa.shape[0]
            return eng.debug_dit_norm(lens_, aa, C_, ad, shift_off, scale_off, _sent(n, C_), _sent(n, C_), film=film, y=yy,
                                      gate_off=gate_off, hi=_psent(n, C_) if planes else None, lo=_psent(n, C_) if planes else None)

        plain = run(lens, a, y, ada, False)
        withp = run(lens, a, y, ada, True)
        _same(plain, run(lens, a, y, ada, False))
        _same(withp, run(lens, a, y, ada, True))
        _same(plain[:2], withp[:2], "dit_norm_planes_kernel's fp32 rows differ from its twin's")
        xo, no, hi, lo = withp
        _check_outside(valid, xo, no, hi, lo)
        _check_planes(no, valid, hi, lo, None, C_)
        utt = _per_row(lens)
        rw = lambda o: ada[utt, o:o + C_]
        v, dv, ref, bound = N.dit_norm(a[valid][:, :C_], film, y[valid] if y_on else None, rw(gate_off), rw(shift_off), rw(scale_off))
        r0, r1 = N.within(xo[valid], v, dv), N.within(no[valid], ref, bound)
        _note("dit_norm_kernel", max(r0, r1))
        assert r0 <= 1 and r1 <= 1, (name, r0, r1)
        for b in (0, B - 1):
            s = slice(off[b], off[b] + lens[b])
            one = run([lens[b]], a[s], y[s] if y_on else None, ada[b:b + 1], True)
            for x_, y_ in zip(withp, one):
                assert np.array_equal(x_[s].view(np.uint8), y_.view(np.uint8)), "alone != batched"


def test_dit_norm_refusals(eng):
    a = np.zeros((2, 528), np.float32)
    with pytest.raises(VttsError, match="512"):
        eng.debug_dit_norm([2], a, 528, np.zeros((1, 6 * 528), np.float32), 0, 528, _sent(2, 528), _sent(2, 528))
    with pytest.raises(VttsError, match="lda"):
        eng.debug_dit_norm([2], a[:, :40], 48, np.zeros((1, 6 * 48), np.float32), 0, 48, _sent(2, 48), _sent(2, 48))


# ---------------------------------------------------------------------------------------------------- the passes
@pytest.mark.parametrize("C_", [48, 144, 192, 208, 512, 768, 1008, 1024])
@pytest.mark.parametrize("act", ["gelu", "silu"])
def test_activation_passes(eng, C_, act):
    f, ferr = (N.gelu, N.gelu_err) if act == "gelu" else (N.silu, N.silu_err)
    for name, lens in BATCHES.items():
        off, valid = _layout(lens)
        rows = off[-1]
        y = np.clip(_inputs(lens, C_, 11 + C_), -50, 50)
        y[~valid] = SENT              # rows outside the utterances are the sentinel, which in place must survive
        out, _, _ = eng.debug_act(act, lens, y)
        _same((out,), (eng.debug_act(act, lens, y)[0],))
        _check_outside(valid, out)
        r = N.within(out[valid], f(y[valid]), ferr(y[valid]))
        _note({"gelu": "cv_gelu_kernel", "silu": "dit_silu_kernel"}[act], r)
        assert r <= 1, (name, r)
        y2, hi, lo = eng.debug_act(act, lens, y, hi=_psent(rows, C_), lo=_psent(rows, C_))
        _check_outside(valid, hi, lo)
        _check_planes(out, valid, hi, lo, None, C_)    # the planes split the fp32 value the in-place pass writes
        if act == "gelu":
            assert np.array_equal(y2.view(np.uint8), y.view(np.uint8)), "the GELU planes pass wrote its input"
        else:
            assert np.array_equal(y2.view(np.uint8), out.view(np.uint8)), "dit_silu_planes_kernel's fp32 rows differ from its twin's"
        for b in (0, len(lens) - 1):
            s = slice(off[b], off[b] + lens[b])
            o1, _, _ = eng.debug_act(act, [lens[b]], y[s])
            assert np.array_equal(o1.view(np.uint8), out[s].view(np.uint8)), "alone != batched"


@pytest.mark.parametrize("C_", [48, 192, 208, 512])
@pytest.mark.parametrize("pad", [0, 40])
def test_gate(eng, C_, pad):
    ldo = C_ + pad
    for name, lens in BATCHES.items():
        off, valid = _layout(lens)
        rows, B = off[-1], len(lens)
        x, y = _inputs(lens, C_, 12 + C_), _inputs(lens, C_, 13 + C_)
        ada = (0.5 * np.random.default_rng(14 + C_).standard_normal((B, 6 * C_))).astype(np.float32)
        out, _, _ = eng.debug_gate(lens, x, y, ada, 5 * C_, _sent(rows, ldo))
        _same((out,), (eng.debug_gate(lens, x, y, ada, 5 * C_, _sent(rows, ldo))[0],))
        o2, hi, lo = eng.debug_gate(lens, x, y, ada, 5 * C_, _sent(rows, ldo), hi=_psent(rows, ldo), lo=_psent(rows, ldo))
        assert np.array_equal(o2.view(np.uint8), out.view(np.uint8)), "dit_gate_planes_kernel's fp32 rows differ from its twin's"
        _check_outside(valid, out, hi, lo, cols=C_)
        _check_planes(out, valid, hi, lo, None, C_)
        utt = _per_row(lens)
        ref, bound = N.gate(x[valid], y[valid], ada[utt, 5 * C_:6 * C_])
        r = N.within(out[valid][:, :C_], ref, bound)
        _note("dit_gate_kernel", r)
        assert r <= 1, (name, r)
        for b in (0, B - 1):
            s = slice(off[b], off[b] + lens[b])
            o1, _, _ = eng.debug_gate([lens[b]], x[s], y[s], ada[b:b + 1], 5 * C_, _sent(lens[b], ldo))
            assert np.array_equal(o1.view(np.uint8), out[s].view(np.uint8)), "alone != batched"


# ---------------------------------------------------------------------------------------------------- GroupNorm
K0, S0 = 10, 5


def _samples(rows):
    return (rows - 1) * S0 + K0


def _clip(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "speech":
        return CI.speech(n, seed)
    if kind == "sine":
        return np.sin(2 * np.pi * 441.0 * np.arange(n) / 16000 + 0.3).astype(np.float32)
    if kind == "dc":
        return (0.5 + 1e-3 * rng.standard_normal(n)).astype(np.float32)
    if kind == "silence":
        return np.zeros(n, np.float32)
    if kind == "click":
        x = np.zeros(n, np.float32)
        x[n // 3] = 1.0
        return x
    raise ValueError(kind)


GN_KINDS = ["speech", "sine", "dc", "silence", "click"]
# the shortest clip, layer-0 row counts around one and two chunks, 1 s, 10 s, 30 s (+ 3 samples: a partial last window)
GN_LENGTHS = [400, _samples(255), _samples(256), _samples(257), _samples(511), _samples(512), _samples(513), 16000, 16003,
              160000, 480000, 400, 2000, _samples(256) + 4, 16000, 7000]


def _gn_weights():
    sd = CI.model()
    fe = "feature_extractor.conv_layers.0."
    return (np.asarray(sd[fe + "conv.weight"], np.float32)[:, 0, :], np.asarray(sd[fe + "layer_norm.weight"], np.float32),
            np.asarray(sd[fe + "layer_norm.bias"], np.float32))


def _gn_run(eng, clips):
    B = len(clips)
    ld = max(len(c) for c in clips)
    wav = np.full((B, ld), np.nan, np.float32)
    for b, c in enumerate(clips):
        wav[b, :len(c)] = c
    rows0 = sum(N.layer0_rows(len(c), K0, S0) + 1700 for c in clips)
    rows = (rows0 + 65535) // 65536 * 65536 + 65536
    Cc = CI.cv()["cv_conv_dim"]
    return eng.debug_groupnorm(wav, [len(c) for c in clips], _sent(rows, Cc))


def test_groupnorm(eng):
    w0, g, beta = _gn_weights()
    eps = CI.cv()["cv_gn_eps"]
    clips = [_clip(GN_KINDS[i % len(GN_KINDS)], n, 100 + i) for i, n in enumerate(GN_LENGTHS)]
    out, len0, off0 = _gn_run(eng, clips)
    again, _, _ = _gn_run(eng, clips)
    assert np.array_equal(out.view(np.uint8), again.view(np.uint8)), "two runs differ"
    valid = np.zeros(out.shape[0], bool)
    for b, c in enumerate(clips):
        assert len0[b] == N.layer0_rows(len(c), K0, S0)
        valid[off0[b]:off0[b] + len0[b]] = True
    _check_outside(valid, out)
    for b, c in enumerate(clips):
        ref, bound = N.groupnorm_clip(c, w0, g, beta, eps, K0, S0)
        r = N.within(out[off0[b]:off0[b] + len0[b]], ref, bound)
        _note("cv_gn_kernel", r)
        assert r <= 1, (b, len(c), GN_KINDS[b % len(GN_KINDS)], r)
    for b in (0, 2, 3, 10):
        o1, l1, f1 = _gn_run(eng, [clips[b]])
        assert np.array_equal(o1[f1[0]:f1[0] + l1[0]].view(np.uint8), out[off0[b]:off0[b] + len0[b]].view(np.uint8)), "alone != batched"


def test_groupnorm_refusals(eng):
    with pytest.raises(VttsError, match="too short"):
        _gn_run(eng, [np.zeros(399, np.float32)])
