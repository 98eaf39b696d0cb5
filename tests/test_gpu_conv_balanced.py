"""GPU (-m gpu): grouped tensor-core conv launches whose problems are split-K reduced over different numbers of CTAs
inside one cluster size (mixed splits, csrc/conv_tc.cuh), through the engine's own launch code (vtts_debug_conv) and
against the float64 reference and fp32 accumulation bound of tests/conv_ref.py.  Each case asserts the per-problem splits
the engine reports, that rows outside the utterances keep their sentinel, that output planes are split(lrelu(y)) bit for
bit, and that two launches are bit-identical (the reduce sums the partials of a tile in a fixed rank order)."""
import zlib

import pytest
import torch

import conv_ref as cr
from test_gpu_conv import _ov, _prob, run_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(packed, cfg):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    e = Engine(cfg, packed[0], packed[1], device=0, precision=1)
    yield e
    e.close()


# engine defaults (split-K on, 64-wide tiles unless the plan picks 128, no forced persistent / tall path)
AUTO = dict(tc_bn=0, tc_split=0, tc_persist=1, tc_tall=0, tc_mc=0, tc_wmc=0, tc_min_steps=2)


def mrf_group(C, dil_index, second, planes=False):
    """The decoder's grouped MRF launch of one dilation step: resblocks k = 11, 7, 3 (largest first, as the engine orders
    them); the first conv of the pair is dilated, the second adds the residual."""
    probs = []
    for j, k in enumerate((11, 7, 3)):
        d = 1 if second else (1, 3, 5)[dil_index]
        probs.append(_prob(Cin=C, Cout=C, k=k, dil=d, pad=d * (k - 1) // 2, ldy=3 * C, yoff=j * C,
                           res=1 if second else 0, ldr=3 * C, roff=j * C,
                           planes_on=1 if planes else 0, ldp=3 * C, poff=j * C, pl_slope=0.1))
    return probs


def check_report(rep, n):
    assert len(rep["psplit"]) == n
    assert all(rep["split"] % s == 0 for s in rep["psplit"]), rep
    if len(set(rep["psplit"])) > 1:
        assert rep["grid_x"] == 1 and rep["grid_y"] == 1 and rep["grid_z"] % rep["split"] == 0, rep
    else:
        assert rep["psplit"] == [rep["split"]] * n, rep


# The bench utterance (162 frames; its 192-frame length bucket gets the same plans) on an H100 (co-resident clusters of
# 2/4/8 conv CTAs: 66/30/15): stage 1 (648 rows x 256 channels) takes 128-wide tiles in clusters of 4 with splits 4/4/2 (longest k-loop 11 k-steps, was 22); stage 2 (2592 x 128)
# clusters of 2 with splits 2/2/1 (11 k-steps, was 22 on the persistent path).
BENCH = {4: dict(bn=128, split=4, psplit=[4, 4, 2], persist=0, image=0), 16: dict(bn=128, split=2, psplit=[2, 2, 1], persist=0, image=0)}


@pytest.mark.parametrize("L", [1, 33, 162, 256, 1000])
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("second", [False, True])
def test_mrf_groups_auto(eng, L, stage, second):
    C, rmul = (256, 4) if stage == 1 else (128, 16)
    probs = mrf_group(C, 1, second, planes=not second)
    expect = BENCH[rmul] if L == 162 else {}
    rep = run_case(eng, "tc", [L], rmul, probs, expect, ov=AUTO, seed=zlib.crc32(b"mrf%d%d%d" % (L, stage, second)))
    check_report(rep, 3)
    if L in (33, 162, 256) or (L == 1 and stage == 2):
        assert len(set(rep["psplit"])) > 1, rep      # single-wave launches with unequal k-loops get unequal splits


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("dil_index", [0, 2])
def test_mrf_groups_pinned_tile_width(eng, bn, dil_index):
    """Both tile widths under mixed splits, the widest halo (dilation 5 at k = 11) included."""
    probs = mrf_group(256, dil_index, False, planes=True)
    ov = dict(AUTO, tc_bn=bn)
    rep = run_case(eng, "tc", [162], 4, probs, dict(bn=bn), ov=ov, seed=bn + dil_index)
    check_report(rep, 3)
    assert len(set(rep["psplit"])) > 1, rep


@pytest.mark.parametrize("rmul", [4, 16])
def test_mrf_groups_ragged(eng, rmul):
    """Ragged batches: clusters covering tiles of several utterances, some of them idle."""
    C = 256 if rmul == 4 else 128
    lens = [1, 40, 3, 17] if rmul == 4 else [9, 1, 5]
    for second in (False, True):
        rep = run_case(eng, "tc", lens, rmul, mrf_group(C, 2, second), {}, ov=AUTO, seed=rmul + second)
        check_report(rep, 3)
        assert len(set(rep["psplit"])) > 1, rep


@pytest.mark.parametrize("second", [False, True])
def test_mrf_groups_machine_filling_batch(eng, second):
    """A batch whose tiles fill the machine keeps the persistent path with one factor (no split) under the defaults."""
    lens = [60 + 4 * i for i in range(16)]
    rep = run_case(eng, "tc", lens, 4, mrf_group(256, 1, second), dict(persist=1, split=1, psplit=[1, 1, 1], image=2),
                   ov=AUTO, seed=30 + second)
    check_report(rep, 3)


@pytest.mark.parametrize("stage", [1, 2])
def test_ups_polyphase_groups(eng, stage):
    """The upsampling ConvTranspose1d as four polyphase problems of equal k-loops: one split for all of them."""
    Cin, rmul = (512, 1) if stage == 1 else (256, 4)
    probs = [_prob(Cin=Cin, Cout=Cin // 2, k=4, pad=p, out_mul=4, out_add=r, ldy=Cin // 2, planes_on=1, ldp=Cin // 2, pl_slope=0.1)
             for r, p in enumerate([2, 2, 1, 1])]
    for L in (1, 162):
        rep = run_case(eng, "tc", [L], rmul, probs, dict(persist=0), ov=AUTO, seed=stage * 10 + L)
        check_report(rep, 4)
        assert len(set(rep["psplit"])) == 1, rep


def test_wn_residual_skip_pair(eng):
    """The flow's WaveNet {rsx, rss} pair (k = 1): too few k-steps for split-K."""
    probs = [_prob(Cin=192, Cout=192, ldy=384, yoff=0, res=2, ldr=384, roff=0, planes_on=1, ldp=192),
             _prob(Cin=192, Cout=192, ldy=384, yoff=192, res=2, ldr=384, roff=192)]
    rep = run_case(eng, "tc", [162], 1, probs, dict(split=1, psplit=[1, 1], persist=0), ov=AUTO, seed=5)
    check_report(rep, 2)
    # with the minimum k-steps per CTA lowered, a 3-step k-loop splits: one factor for both problems
    rep = run_case(eng, "tc", [162], 1, probs, {}, ov=dict(AUTO, tc_min_steps=1), seed=6)
    check_report(rep, 2)
    assert rep["split"] > 1 and len(set(rep["psplit"])) == 1, rep
