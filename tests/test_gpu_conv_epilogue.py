"""GPU (-m gpu): the tensor-core conv epilogue at the flow's WN in-conv shape, through the harness of test_gpu_conv.py.

The flow's WN in-conv (Cin 192 -> 2 x 192, k = 5, gated, with cond) split 8 ways at BN 64: each CTA of a cluster finishes
W = 8 columns, one column pair per consumer thread in each of its two rows.  That pair's loads are the ones issued before
the cluster barriers, and no later pair's loads follow them."""
import pytest

import conv_ref as cr
from test_gpu_conv import _ov, _prob, eng, run_case  # noqa: F401  (eng: the engine fixture of that module)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lens", [[162], [1], [129]])
def test_tc_split8_bn64_wn_in_gated(eng, lens):  # noqa: F811
    run_case(eng, "tc", lens, 1, [_prob(Cin=192, Cout=384, k=5, pad=2, epi=cr.EPI_GATE, cond=True)],
             dict(bn=64, split=8, image=0, grid_y=6, grid_z=8), ov=_ov(tc_split=8, tc_min_steps=1), seed=sum(lens) + 80)
