"""The split-K plan of grouped tensor-core conv launches (tc_split_plan in csrc/engine.cu), on the host alone through
vtts_tc_split_plan: the plans of the bench utterance's decoder launches on an H100, and the old one-factor rule wherever the
problems of a launch have equal k-loops."""
import itertools

import pytest

from vosk_tts_b200.engine import VttsError, tc_split_plan

H100_SM = 132
H100_CAP = [66, 30, 15, 66, 30, 15]     # co-resident conv_tc clusters of 2/4/8 CTAs at BN 64, BN 128 (H100 SXM, 227 KB)


def mrf(C):
    return [dict(Cin=C, Cout=C, k=k) for k in (11, 7, 3)]


# The 162-frame bench utterance runs in the 192-frame length bucket; the plan must be the same for both.
@pytest.mark.parametrize("frames", [162, 192])
def test_bench_decoder_plans(frames):
    # MRF stage 1 (x4 rows, 256 channels): 128-wide tiles, clusters of 4, longest k-loop 44/4 = 11 k-steps (was 22)
    assert tc_split_plan(mrf(256), [frames], 4, H100_SM, H100_CAP) == (128, 4, [4, 4, 2])
    # MRF stage 2 (x16 rows, 128 channels): clusters of 2, 22/2 = 11 k-steps (was 22 on the persistent path)
    assert tc_split_plan(mrf(128), [frames], 16, H100_SM, H100_CAP) == (128, 2, [2, 2, 1])
    # the polyphase upsampling groups: equal k-loops, one factor
    ups1 = [dict(Cin=512, Cout=256, k=4)] * 4
    ups2 = [dict(Cin=256, Cout=128, k=4)] * 4
    assert tc_split_plan(ups1, [frames], 1, H100_SM, H100_CAP) == (128, 4, [4, 4, 4, 4])
    assert tc_split_plan(ups2, [frames], 4, H100_SM, H100_CAP) == (128, 4, [4, 4, 4, 4])
    # the flow's WaveNet {rsx, rss} pair: 3 k-steps, no split
    assert tc_split_plan([dict(Cin=192, Cout=192, k=1)] * 2, [frames], 1, H100_SM, H100_CAP) == (64, 1, [1, 1])


def test_machine_filling_batch_is_not_split():
    """64 utterances: far more tiles than SMs, no split (the launch takes the persistent path)."""
    lens = [100 + 3 * i for i in range(64)]
    for probs, rmul in ((mrf(256), 4), (mrf(128), 16), ([dict(Cin=192, Cout=192, k=5)], 1)):
        bn, split, ps = tc_split_plan(probs, lens, rmul, H100_SM, H100_CAP)
        assert split == 1 and ps == [1] * len(probs)


def old_rule(probs, lens, rmul, bn, max_split, min_steps, n_sm, cap):
    """The one-factor rule the plan generalises: the widest split whose clusters are all co-resident and that leaves
    min_steps k-steps to every CTA; 128-wide tiles when they allow a wider split than 64-wide ones."""
    minsteps = min(q["Cin"] // 64 * q["k"] for q in probs)
    wide = all(q["Cout"] >= 128 for q in probs)
    active = [sum((n * rmul + q.get("in_extra", 0) + 127) // 128 * ((q["Cout"] + w - 1) // w) for q in probs for n in lens)
              for w in (64, 128)]

    def best(wi):
        for S, si in ((8, 2), (4, 1), (2, 0)):
            if S <= max_split and minsteps >= min_steps * S and active[wi] <= cap[3 * wi + si]:
                return S
        return 1
    if bn:
        return bn, best(bn == 128)
    s64, s128 = best(0), (best(1) if wide else 1)
    return (128, s128) if s128 > s64 else (64, s64)


@pytest.mark.parametrize("n", [1, 2, 4])
def test_equal_k_loops_reduce_to_the_one_factor_rule(n):
    cases = 0
    for Cin, Cout, k, lens, rmul, bn, max_split, min_steps in itertools.product(
            (64, 192, 256, 512), (64, 96, 192, 256), (1, 3, 5, 11), ([1], [33], [162], [300], [1000], [3, 17, 40]),
            (1, 4), (0, 64, 128), (8, 2), (2, 1)):
        probs = [dict(Cin=Cin, Cout=Cout, k=k)] * n
        ctas128 = sum((m * rmul + 127) // 128 * ((Cout + 127) // 128) for m in lens) * n
        if bn == 0 and Cout >= 128 and ctas128 >= 2 * H100_SM:
            continue                  # (launch_tc takes 128-wide tiles without split-K before any plan is made)
        want_bn, want_s = old_rule(probs, lens, rmul, bn, max_split, min_steps, H100_SM, H100_CAP)
        got = tc_split_plan(probs, lens, rmul, H100_SM, H100_CAP, bn=bn, max_split=max_split, min_steps=min_steps)
        assert got == (want_bn, want_s, [want_s] * n), (probs, lens, rmul, bn, max_split, min_steps, got)
        cases += 1
    assert cases > 1000


def test_invalid_arguments_are_refused():
    with pytest.raises(VttsError):
        tc_split_plan([dict(Cin=100, Cout=64, k=3)], [10], 1, H100_SM, H100_CAP)
    with pytest.raises(VttsError):
        tc_split_plan([dict(Cin=64, Cout=64, k=3)] * 5, [10], 1, H100_SM, H100_CAP)
    with pytest.raises(VttsError):
        tc_split_plan([dict(Cin=64, Cout=64, k=3)], [10], 1, H100_SM, H100_CAP, bn=96)
