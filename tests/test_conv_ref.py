"""CPU: the conv reference of tests/conv_ref.py and its tolerance.  The splits restate the device functions, the operand-exact
emulation agrees with the exact conv within the split's analytic bound, a float32 restatement with another summation order
passes the comparison -- and every deliberately corrupted output is rejected, so the GPU tests built on it
(test_gpu_conv.py) would fail if a kernel were subtly wrong."""
import numpy as np
import pytest

import conv_ref as cr
from vosk_tts_b200 import weights


def test_split_bf16_restates_device_rounding():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(20000).astype(np.float32) * 10.0 ** rng.integers(-6, 6, 20000),
                        np.array([0.0, -0.0, 1.0, -1.0, 3.0e38, 1e-30], np.float32)]).astype(np.float32)   # (normal range:
    # a remainder below 2^-126 would lose bits to subnormal rounding)
    hi, lo = cr.split_bf16(x)
    # hi rounds half away from zero: |x - hi| <= half an ulp of hi's 8-bit significand
    h = cr.bf16_value(hi)
    assert np.all(np.abs(x - h) <= np.abs(h) * 2.0 ** -8 + 1e-45)
    s = h + cr.bf16_value(lo)
    assert np.all(np.abs(s - x) <= np.abs(x) * 2.0 ** -16)
    # a tie (x exactly halfway between two bf16 values) goes away from zero, where the host packer's RNE goes to even
    tie = np.array([1.0 + 2.0 ** -8, -(1.0 + 2.0 ** -8)], np.float32)
    assert cr.bf16_value(cr.split_bf16(tie)[0]).tolist() == [1.0 + 2.0 ** -7, -(1.0 + 2.0 ** -7)]
    assert cr.bf16_value(weights.to_bf16_bits(tie)).tolist() == [1.0, -1.0]
    h3, m3, l3 = cr.split_bf16_3(x)
    assert np.array_equal((cr.bf16_value(h3) + cr.bf16_value(m3) + cr.bf16_value(l3)).astype(np.float32), x)
    assert np.array_equal(cr.bf16_value(h3) + cr.bf16_value(m3) + cr.bf16_value(l3), x.astype(np.float64))


def test_weight_packers_keep_the_conv_layouts():
    rng = np.random.default_rng(1)
    w = rng.standard_normal((65, 32, 3)).astype(np.float32)
    b = rng.standard_normal(65).astype(np.float32)
    wp, bp = weights.conv_ffma_layout(w, b)
    assert wp.shape == (3, 32, 68) and np.array_equal(wp[:, :, :65], w.transpose(2, 1, 0)) and not wp[:, :, 65:].any()
    assert np.array_equal(bp[:65], b) and not bp[65:].any()
    hi, lo = weights.conv_tc_planes(w)
    assert hi.shape == (3, 65, 32)
    assert np.all(np.abs(cr.bf16_value(hi) + cr.bf16_value(lo) - w.transpose(2, 0, 1)) <= np.abs(w.transpose(2, 0, 1)) * 2.0 ** -16)
    h3, m3, l3 = weights.conv_tc3_planes(w)
    assert np.array_equal(cr.bf16_value(h3) + cr.bf16_value(m3) + cr.bf16_value(l3), w.transpose(2, 0, 1).astype(np.float64))


def _setup(n_planes=2, Cin=128, Cout=128, k=3, dil=2, pad=2, lens=(1, 3, 40), epi=cr.EPI_GATE, seed=3):
    rng = np.random.default_rng(seed)
    offs = cr.offsets(lens)
    x = rng.standard_normal((offs[-1], Cin)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k)) / np.sqrt(Cin * k)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    cond = rng.standard_normal((len(lens), Cout)).astype(np.float32)
    planes = cr.split_planes(x, n_planes)
    wpl = np.stack([cr.bf16_value(p).transpose(1, 2, 0)
                    for p in (weights.conv_tc_planes(w) if n_planes == 2 else weights.conv_tc3_planes(w))])
    q = dict(Cin=Cin, Cout=Cout, k=k, dil=dil, pad=pad, epi=epi)
    ins = cr.tc_inputs(planes, list(lens), 1, 0)
    return q, w, bias, cond, ins, wpl, list(lens), x


def _flat(res):
    return np.concatenate([v.reshape(-1) for _, _, v, _ in res]), np.concatenate([d.reshape(-1) for _, _, _, d in res])


@pytest.mark.parametrize("n_planes", [2, 3])
def test_emulation_matches_exact_conv_within_the_split_bound(n_planes):
    q, w, bias, cond, ins, wpl, lens, _ = _setup(n_planes, epi=0)
    emu = cr.reference("tc", q, w, bias, lens, 1, ins, n_planes, wpl)
    ex = cr.reference("tc", q, w, bias, lens, 1, ins, n_planes, wpl, exact=True)
    for (_, _, ve, _), (_, _, vx, _), X in zip(emu, ex, ins):
        xs = X.sum(axis=0)
        mag = cr.conv_taps(np.abs(xs), np.abs(w.astype(np.float64)), q["dil"], q["pad"])     # sum |x w| per output
        err = np.abs(ve - vx)
        if n_planes == 2:
            assert np.all(err <= 3 * 2.0 ** -16 * mag)                       # ~2^-16 relative per product
            assert err.max() > 2.0 ** -24 * mag.max()                        # (and the split error is really there)
        else:
            assert np.all(err <= 2.01 * 2.0 ** -24 * mag)                    # below one fp32 rounding per product
            n_terms = 6 * q["Cin"] * q["k"]
            assert np.all(err <= (n_terms + 8) * cr.U23 * mag)              # i.e. under the accumulation bound


def _float32_restatement(ins, wpl, n_planes, q, bias, cond, lens):
    """The same launch computed in float32 with another summation order (taps reversed, planes summed last)."""
    out = []
    for b, X in enumerate(ins):
        X32, W32 = X.astype(np.float32), wpl.astype(np.float32)
        L = X.shape[1]
        acc = np.zeros((L, q["Cout"]), np.float32)
        for ia, iw in reversed(cr.PAIRS[n_planes]):
            part = np.zeros((L, q["Cout"]), np.float32)
            for j in reversed(range(q["k"])):
                d = j * q["dil"] - q["pad"]
                t0, t1 = max(0, -d), min(L, L - d)
                if t1 > t0:
                    part[t0:t1] += X32[ia][t0 + d:t1 + d] @ W32[iw][:, :, j].T
            acc = acc + part
        a = acc + (bias + cond[b])[None, :].astype(np.float32)
        out.append(np.tanh(a[:, 0::2]) / (np.float32(1) + np.exp(-a[:, 1::2])))
    return np.concatenate([o.reshape(-1) for o in out])


def test_tolerance_passes_a_correct_float32_result_and_rejects_corrupted_ones():
    n_planes = 2
    q, w, bias, cond, ins, wpl, lens, _ = _setup(n_planes)
    ref, bnd = _flat(cr.reference("tc", q, w, bias, lens, 1, ins, n_planes, wpl, cond=cond))
    good = _float32_restatement(ins, wpl, n_planes, q, bias, cond, lens)
    assert not np.array_equal(good, ref.astype(np.float32))          # it really rounds differently ...
    assert cr.within(good, ref, bnd)                                  # ... and still passes
    corruptions = {
        "one MMA term dropped (lo*hi)": dict(drop_pair=(1, 0)),
        "tap 1 shifted by one row": dict(shift=(1, 1)),
        "last 64-channel K chunk dropped": dict(drop_chunk=True),
        "left halo read from the previous utterance": dict(halo_from_prev=True),
        "cond row of utterance b-1": dict(cond_prev=True),
        "gate pairs swapped": dict(gate_swap=True),
    }
    for name, c in corruptions.items():
        bad, _ = _flat(cr.reference("tc", q, w, bias, lens, 1, ins, n_planes, wpl, cond=cond, corrupt=c))
        assert not cr.within(bad, ref, bnd), name
    # the last output column of every 64-wide tile missing (left at what the buffer held)
    res = cr.reference("tc", q, w, bias, lens, 1, ins, n_planes, wpl, cond=cond)
    for _, cols, v, _ in res:
        v[:, cols % 64 == 63] = 0.0
    bad, _ = _flat(res)
    assert not cr.within(bad, ref, bnd), "missing tile column"


def test_ffma_tolerance_rejects_a_shifted_tap():
    rng = np.random.default_rng(5)
    lens, Cin, Cout, k = [7, 30], 32, 24, 5
    offs = cr.offsets(lens)
    x = rng.standard_normal((offs[-1], Cin)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k)) / np.sqrt(Cin * k)).astype(np.float32)
    bias = np.zeros(Cout, np.float32)
    q = dict(Cin=Cin, Cout=Cout, k=k, dil=1, pad=2, ldx=Cin)
    ins = cr.ffma_inputs(x, lens, 1, q)
    ref, bnd = _flat(cr.reference("ffma", q, w, bias, lens, 1, ins))
    # float32 conv in another order passes
    f32 = np.concatenate([cr.conv_taps(X.astype(np.float32), w.astype(np.float32), 1, 2).astype(np.float32).reshape(-1) for X in ins])
    assert cr.within(f32, ref, bnd)
    bad, _ = _flat(cr.reference("ffma", q, w, bias, lens, 1, ins, corrupt=dict(shift=(4, -1))))
    assert not cr.within(bad, ref, bnd)
