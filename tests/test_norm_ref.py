"""CPU: the float64 references of tests/norm_ref.py pinned to torch and to the oracles' modules, and the sharpness of every
bound: each plausible kernel mistake must break its bound on an input the GPU tests (test_gpu_norm.py) run."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import contentvec_inputs as CI
import norm_ref as N
from oracle import bert_oracle, contentvec_oracle, stabletts_cfm_oracle as so, vits_oracle as vo
from vosk_tts_b200 import config as C, synthetic


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


# ---------------------------------------------------------------------------------------------------- pinned to torch
@pytest.mark.parametrize("C_", [32, 48, 208, 1024])
@pytest.mark.parametrize("eps", [1e-5, 1e-12])
def test_normalize_is_torch_layer_norm(C_, eps):
    x = N.mixed_rows(24, C_, np.random.default_rng(C_))
    ref = F.layer_norm(_t(x), (C_,), eps=float(np.float32(eps))).numpy()
    assert np.allclose(N.normalize(N.f64(x), float(np.float32(eps))), ref, rtol=1e-10, atol=1e-9)


def test_add_ln_is_torch_layer_norm_then_adds():
    rng = np.random.default_rng(1)
    a, b, cadd, vec = (rng.standard_normal((9, 96)).astype(np.float32) for _ in range(4))
    g, beta = N.affine(96, rng)
    out, bound = N.add_ln(a, b, g, beta, cadd, vec)
    ref = F.layer_norm(_t(a) + _t(b), (96,), _t(g), _t(beta), eps=float(np.float32(1e-5))) + _t(cadd) + _t(vec)
    assert np.allclose(out, ref.numpy(), rtol=1e-12, atol=1e-12) and np.all(bound > 0)


def test_cv_ln_is_torch_layer_norm_of_a_plus_gelu():
    rng = np.random.default_rng(2)
    a, y = (rng.standard_normal((7, 144)).astype(np.float32) for _ in range(2))
    g, beta = N.affine(144, rng)
    out, _ = N.cv_ln(a, y, g, beta, 1e-5)
    ref = F.layer_norm(_t(a) + F.gelu(_t(y), approximate="none"), (144,), _t(g), _t(beta), eps=float(np.float32(1e-5)))
    assert np.allclose(out, ref.numpy(), rtol=1e-12, atol=1e-12)


def test_activations_are_torch():
    x = np.linspace(-12, 12, 4001)
    assert np.allclose(N.gelu(x), F.gelu(_t(x), approximate="none").numpy(), rtol=1e-13, atol=1e-15)
    assert np.allclose(N.silu(x), F.silu(_t(x)).numpy(), rtol=1e-13, atol=1e-15)
    assert np.all(N.gelu_err(x) > 0) and np.all(N.silu_err(x) > 0)


def test_groupnorm_is_torch_group_norm_of_the_conv():
    rng = np.random.default_rng(3)
    w0 = rng.standard_normal((64, 10)).astype(np.float32)
    g, beta = N.affine(64, rng)
    x = CI.speech(4000, 5)
    out, _ = N.groupnorm_clip(x, w0, g, beta, 1e-5, 10, 5, block=24)
    y = F.conv1d(_t(x)[None, None], _t(w0)[:, None, :], stride=5)
    ref = F.gelu(F.group_norm(y, 64, _t(g), _t(beta), eps=float(np.float32(1e-5))))[0].T.numpy()
    assert out.shape == (N.layer0_rows(4000, 10, 5), 64) and np.allclose(out, ref, rtol=1e-9, atol=1e-10)


# ---------------------------------------------------------------------------------------------------- pinned to the oracles
def test_add_ln_is_the_vits_layer_norm():
    rng = np.random.default_rng(4)
    a, b = (rng.standard_normal((2, 192, 11)).astype(np.float32) for _ in range(2))
    g, beta = N.affine(192, rng)
    ref = vo.layer_norm_c(_t(a) + _t(b), _t(g), _t(beta)).numpy()        # [B, C, T]
    for i in range(2):
        out, _ = N.add_ln(a[i].T, b[i].T, g, beta)
        assert np.allclose(out, ref[i].T, rtol=1e-10, atol=1e-10)


def test_bert_embed_is_the_oracles_embeddings():
    bt = C.bert_config({"hidden_size": 128, "num_attention_heads": 4, "intermediate_size": 512, "num_hidden_layers": 3,
                        "vocab_size": 300})
    sd = synthetic.make_random_bert(bt, 7)
    ids = np.random.default_rng(5).integers(0, bt["bt_vocab"], 37)
    ref = bert_oracle.bert_features(sd, dict(bt, cv_layers=0), ids).numpy()
    e = "embeddings."
    t, _ = N.bert_positions([37])
    out, _ = N.bert_embed(ids, t, sd[e + "word_embeddings.weight"], sd[e + "position_embeddings.weight"],
                          sd[e + "token_type_embeddings.weight"][0], sd[e + "LayerNorm.weight"], sd[e + "LayerNorm.bias"], bt["cv_ln_eps"])
    assert np.allclose(out, ref, rtol=1e-10, atol=1e-10)


def test_dit_norm_is_the_cfm_oracles_norm1():
    cfg = C.stabletts_cfm_config()
    sd = synthetic.make_random_stabletts_cfm(cfg, 11)
    H, T, dt = cfg["hidden_channels"], 13, torch.float64
    x = torch.as_tensor(np.random.default_rng(6).standard_normal((H, T)).astype(np.float32)).to(dt)
    temb = so.time_embedding(sd, cfg, 0.3, dt)
    ada = so.ada_rows(sd, cfg, torch.as_tensor(sd["spk_emb.weight"][0]).to(dt), 0, dt)
    taps = {}
    so.block(sd, cfg, 0, x, temb, ada, so.rope_table(T, H // cfg["n_heads"] // 2, dt), dt, taps)
    film = torch.cat(so.film_rows(sd, cfg, temb, 0, dt)).numpy()
    rows = lambda k: np.repeat(ada[k].numpy()[None], T, 0)
    _, _, no, _ = N.dit_norm(x.numpy().T, film, None, rows(2), rows(0), rows(1))
    # (the reference reads the FiLM and adaLN rows as the fp32 values the kernel is given; the oracle keeps them in float64)
    assert np.allclose(no, taps["norm1"].numpy().T, rtol=1e-6, atol=1e-6)


def test_groupnorm_is_contentvecs_feature_extractor():
    cv = dict(CI.cv(), cv_conv_kernel=[10], cv_conv_stride=[5])          # the feature encoder cut after layer 0
    sd = CI.folded()
    x = CI.speech(1600, 9)
    st = {}
    contentvec_oracle.contentvec_units(sd, cv, x, stages=st)
    fe = "feature_extractor.conv_layers.0."
    out, _ = N.groupnorm_clip(x, np.asarray(sd[fe + "conv.weight"])[:, 0, :], sd[fe + "layer_norm.weight"],
                              sd[fe + "layer_norm.bias"], cv["cv_gn_eps"], 10, 5)
    assert np.allclose(out, st["feat"].numpy(), rtol=1e-9, atol=1e-10)


# ---------------------------------------------------------------------------------------------------- the bounds
def test_bound_grows_with_the_mean_against_the_spread():
    rng = np.random.default_rng(8)
    x = N.rows_of("random", 1, 256, rng)
    en0 = N.normalize_bound(N.f64(x), np.zeros((1, 256)), 1e-5, N.warp_depth(256)).max()
    en1 = N.normalize_bound(N.f64(x) + 1e3, np.zeros((1, 256)), 1e-5, N.warp_depth(256)).max()
    assert en1 > 100 * en0


def _warp_sum(t, fma_sq=False):
    """cv_ln_kernel's row sum in fp32: lane l adds t[l + 32 i] in order (fmaf(t, t, q) when fma_sq), then the xor butterfly."""
    f = np.float32
    C = t.size
    lanes = np.zeros(32, f)
    for i in range(0, C, 32):
        u = t[i:i + 32].astype(np.float64)
        k = u.size
        lanes[:k] = ((lanes[:k] + u * u) if fma_sq else (lanes[:k] + u)).astype(f)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[np.arange(32) ^ o]).astype(f)
    return lanes[0]


def test_kernel_arithmetic_in_fp32_meets_the_bound():
    """A float32 restatement of cv_ln_kernel's own arithmetic (its summation tree, two-pass variance) is within the bound,
    with the largest ratio on the rows of large mean: the bound is sharp enough to be met by less than 100x."""
    rng = np.random.default_rng(9)
    f = np.float32
    worst = 0.0
    for C_ in (48, 1008, 1024):
        a = N.mixed_rows(60, C_, rng)
        g, beta = N.affine(C_, rng)
        out = np.empty_like(a)
        for i, v in enumerate(a):
            m = f(_warp_sum(v) / f(C_))
            d = (v - m).astype(f)
            r = f(1 / np.sqrt(np.float64(f(f(_warp_sum(d, True) / f(C_)) + f(1e-5)))))
            out[i] = ((d * r).astype(f).astype(np.float64) * g + beta).astype(f)
        ref, bound = N.cv_ln(a, None, g, beta, 1e-5)
        worst = max(worst, N.within(out, ref, bound))
    assert 0.01 < worst <= 1, worst


# ---------------------------------------------------------------------------------------------------- mutations
def _ln_case(C_, seed):
    rng = np.random.default_rng(seed)
    return N.mixed_rows(120, C_, rng), *N.affine(C_, rng)


@pytest.mark.parametrize("mutate", ["one_pass", "unbiased", "eps_outside"])
@pytest.mark.parametrize("C_", [32, 256])
def test_add_ln_mistakes_break_the_bound(mutate, C_):
    a, g, beta = _ln_case(C_, C_)
    b = N.mixed_rows(120, C_, np.random.default_rng(C_ + 1))
    ref, bound = N.add_ln(a, b, g, beta)
    bad, _ = N.add_ln(a, b, g, beta, mutate=mutate)
    assert N.within(bad, ref, bound) > 1


@pytest.mark.parametrize("mutate", ["cadd_before", "vec_before"])
def test_add_ln_adds_after_the_norm(mutate):
    a, g, beta = _ln_case(96, 12)
    rng = np.random.default_rng(13)
    cadd, vec = rng.standard_normal((120, 96)).astype(np.float32), np.repeat(rng.standard_normal((1, 96)), 120, 0).astype(np.float32)
    ref, bound = N.add_ln(a, None, g, beta, cadd, vec)
    bad, _ = N.add_ln(a, None, g, beta, cadd, vec, mutate=mutate)
    assert N.within(bad, ref, bound) > 1


@pytest.mark.parametrize("mutate", ["one_pass", "unbiased", "eps_outside", "tanh"])
@pytest.mark.parametrize("C_", [48, 1024])
def test_cv_ln_mistakes_break_the_bound(mutate, C_):
    a, g, beta = _ln_case(C_, C_ + 2)
    y = N.mixed_rows(120, C_, np.random.default_rng(C_ + 3)) if mutate == "tanh" else None
    if y is not None:
        y = np.clip(y, -4, 4)
    ref, bound = N.cv_ln(a, y, g, beta, 1e-5)
    bad, _ = N.cv_ln(a, y, g, beta, 1e-5, mutate=mutate)
    assert N.within(bad, ref, bound) > 1


def test_tanh_gelu_breaks_the_pass_bound():
    y = N.mixed_rows(60, 144, np.random.default_rng(14))
    assert N.within(N.gelu_tanh(N.f64(y)), N.gelu(N.f64(y)), N.gelu_err(N.f64(y))) > 1


@pytest.mark.parametrize("mistake", ["eps_1e-5", "batch_pos", "one_pass"])
def test_bert_embed_mistakes_break_the_bound(mistake):
    lens = [5, 9, 17]
    word, pos, type0, (g, beta) = N.bert_tables(144, max(lens), 15)
    ids = np.random.default_rng(16).integers(0, word.shape[0], N.offsets(lens)[-1]).astype(np.int32)
    t, rows = N.bert_positions(lens)
    ref, bound = N.bert_embed(ids[rows], t, word, pos, type0, g, beta, 1e-12)
    if mistake == "eps_1e-5":
        bad, _ = N.bert_embed(ids[rows], t, word, pos, type0, g, beta, 1e-5)
    elif mistake == "batch_pos":
        tb, _ = N.bert_positions(lens, mutate="batch_pos")
        bad, _ = N.bert_embed(ids[rows], tb, word, np.pad(pos, ((0, N.offsets(lens)[-1]), (0, 0))), type0, g, beta, 1e-12)
    else:
        bad, _ = N.bert_embed(ids[rows], t, word, pos, type0, g, beta, 1e-12, mutate=mistake)
    assert N.within(bad, ref, bound) > 1


def dit_case(C_, n, seed):
    """The GPU test's dit_norm data: a rows of pitch lda = C + 16, FiLM rows, y, and one adaLN row of 6 C."""
    rng = np.random.default_rng(seed)
    a = N.mixed_rows(n, C_ + 16, rng)
    film = np.concatenate(N.affine(C_, rng))
    y = rng.standard_normal((n, C_)).astype(np.float32)
    ada = (0.5 * rng.standard_normal(6 * C_)).astype(np.float32)
    return a, film, y, ada


@pytest.mark.parametrize("mistake", ["one_pass", "unbiased", "eps_outside", "film_swap", "scale", "gate_at_shift", "pitch"])
def test_dit_norm_mistakes_break_the_bound(mistake):
    C_, n = 192, 120
    a, film, y, ada = dit_case(C_, n, 16)
    rows = lambda k: np.repeat(ada[None, k * C_:(k + 1) * C_], n, 0)
    if mistake in ("one_pass", "eps_outside"):
        film = y = None          # a text encoder block's first norm: the residual alone, whose offset / tiny rows they meet
    ref = N.dit_norm(a[:, :C_], film, y, rows(2), rows(3), rows(4))
    if mistake == "pitch":
        bad = N.dit_norm(a.reshape(-1)[:n * C_].reshape(n, C_), film, y, rows(2), rows(3), rows(4))
    else:
        bad = N.dit_norm(a[:, :C_], film, y, rows(2), rows(3), rows(4), mutate=mistake)
    assert max(N.within(bad[0], ref[0], ref[1]), N.within(bad[2], ref[2], ref[3])) > 1


def test_groupnorm_statistics_per_chunk_break_the_bound():
    sd = CI.model()
    fe = "feature_extractor.conv_layers.0."
    w0 = np.asarray(sd[fe + "conv.weight"])[:64, 0, :]
    g, beta = np.asarray(sd[fe + "layer_norm.weight"])[:64], np.asarray(sd[fe + "layer_norm.bias"])[:64]
    x = CI.speech(16000, 17)
    ref, bound = N.groupnorm_clip(x, w0, g, beta, 1e-5, 10, 5)
    for mistake in ("chunk", "tanh", "unbiased"):
        bad, _ = N.groupnorm_clip(x, w0, g, beta, 1e-5, 10, 5, mutate=mistake)
        assert N.within(bad, ref, bound) > 1, mistake


def test_gate_reference():
    rng = np.random.default_rng(18)
    x, y, g = (rng.standard_normal((5, 48)).astype(np.float32) for _ in range(3))
    out, bound = N.gate(x, y, g)
    assert np.allclose(out, N.f64(x) + N.f64(g) * N.f64(y), rtol=0, atol=0) and np.all(bound >= 0)
