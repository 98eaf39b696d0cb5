"""GPU (-m gpu): the relative-position attention kernels in isolation against a plain PyTorch reference of the same
op (attentions.py:165-196 restated on q, k, v directly; float64 so that both kernels' errors are visible).

  tensor-core kernel (csrc/attn_tc.cuh: wgmma QK^T / PV with split-bf16 operands, P in registers, online softmax)
  fp32 FFMA kernels (csrc/kernels.cuh attn_kernel / attn_split_kernel)

Tolerances: fp32 FFMA <= 2e-5, tensor-core <= 2e-4 max-abs on outputs of magnitude ~1 (the split-bf16 operands carry
~2^-18 relative error per factor; the waveform budget of the whole path is 1e-3)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def ref_attention(qkv, relk, relv, n_heads, window):
    """qkv [T, 3H] float64; relk / relv [2W+1, dk].  Returns [T, H]."""
    T, H3 = qkv.shape
    H = H3 // 3
    dk = H // n_heads
    out = torch.zeros(T, H, dtype=torch.float64)
    i = torch.arange(T)
    d = i[None, :] - i[:, None]                      # j - i
    inband = d.abs() <= window
    slot = (d + window).clamp(0, 2 * window)
    for h in range(n_heads):
        q = qkv[:, h * dk:(h + 1) * dk] / (dk ** 0.5)
        k = qkv[:, H + h * dk:H + (h + 1) * dk]
        v = qkv[:, 2 * H + h * dk:2 * H + (h + 1) * dk]
        s = q @ k.T
        rl = q @ relk.T                              # [T, 2W+1]
        s = s + torch.where(inband, torch.gather(rl, 1, slot), torch.zeros_like(s))
        p = torch.softmax(s, dim=1)
        o = p @ v
        pb = torch.where(inband, p, torch.zeros_like(p))            # band probabilities scattered to their relative slot
        rel_w = torch.zeros(T, 2 * window + 1, dtype=torch.float64)
        rel_w.scatter_add_(1, slot, pb)
        # (slots outside the band received zeros only, except the clamped ends which got exact zeros too)
        o = o + rel_w @ relv
        out[:, h * dk:(h + 1) * dk] = o
    return out


@pytest.fixture(scope="module")
def eng1(packed, cfg):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    yield e
    e.close()


def _inputs(T, H, seed, kind):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, 3 * H, generator=g, dtype=torch.float64)
    if kind == "peaky":          # wide score distribution
        x[:, : 2 * H] *= 2.0
    elif kind == "growing":      # later keys score much higher than earlier ones: the running max must be refreshed
        ramp = torch.linspace(0.2, 3.0, T, dtype=torch.float64)[:, None]
        x[:, H:2 * H] *= ramp
        x[:, :H] = x[:, :H].abs()                     # q . k grows with the key index for every query
        x[:, H:2 * H] = x[:, H:2 * H].abs()
    return x.float().double()                         # exactly representable in fp32


@pytest.mark.parametrize("T,kind", [(1, "plain"), (5, "plain"), (64, "plain"), (65, "peaky"), (128, "plain"), (129, "peaky"),
                                    (162, "plain"), (300, "growing"), (1000, "peaky"), (1000, "growing"), (4765, "plain")])
@pytest.mark.parametrize("use_tc", [1, 0], ids=["tcgen05", "ffma"])
def test_attention_kernel_vs_torch(eng1, folded, cfg, T, kind, use_tc):
    H, W = cfg["hidden_channels"], cfg["window_size"]
    heads = cfg.get("flow_n_heads", 2)
    a = "flow.flows.0.pre_transformer.attn_layers.0"
    relk, relv = folded[a + ".emb_rel_k"][0].double(), folded[a + ".emb_rel_v"][0].double()
    qkv = _inputs(T, H, 100 + T, kind)
    ref = ref_attention(qkv, relk, relv, heads, W).numpy()
    out, _ = eng1.debug_attention("flow.0.tr", qkv.float().numpy(), use_tc)
    err = np.abs(out - ref).max()
    assert np.isfinite(out).all()
    assert err < (2e-4 if use_tc else 2e-5), "T=%d %s: max-abs error %.3e" % (T, kind, err)
