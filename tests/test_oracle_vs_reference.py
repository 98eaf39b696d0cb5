"""CPU: pins the oracle restatement and the weight packer's helpers against what the unmodified reference modules
computed on the same seeded inputs (tests/golden/ref_pins.npz, written by oracle/make_golden_ref.py)."""
import numpy as np
import pytest
import torch

import golden_ref as GR
from oracle import vits_oracle as vo


@pytest.fixture(scope="module")
def pins():
    return GR.load("ref_pins.npz")


def test_fold_equals_remove_weight_norm(pins, folded):
    keys = {k[3:] for k in pins.files if k.startswith("sd/")}
    for k, v in folded.items():
        assert k in keys, k
        flat = v.reshape(-1).numpy()
        assert np.abs(flat[GR.sample_index(flat.size, k, GR.SD_SAMPLE)] - pins["sd/" + k]).max() <= 1e-6, k


def test_istft_basis_and_pqmf_match_reference(pins):
    from vosk_tts_b200 import weights
    assert np.abs(weights.istft_inverse_basis(16, 4) - pins["basis"]).max() < 1e-7
    assert np.abs(weights.pqmf_synthesis_filter(4) - pins["pqmf"]).max() < 1e-7


def test_spline_inverse_matches_reference_transforms(pins):
    x, uw, uh, ud = GR.spline_inputs()
    got = vo.rq_spline_inverse(x.clone(), uw.clone(), uh.clone(), ud.clone(), bound=5.0)
    assert np.array_equal(pins["spline"], got.numpy())


@pytest.mark.parametrize("T,seed", GR.INFER_CASES)
def test_oracle_equals_reference_infer(pins, folded, cfg, T, seed):
    tok, eps_dp, eps_z, scales = GR.infer_inputs(T, seed)
    with torch.no_grad():
        o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([3]), scales, eps_dp, eps_z, return_all=True)
    ro = pins["infer%d/o" % T]
    assert ro.shape == tuple(o["o"].shape)
    assert np.array_equal(pins["infer%d/attn" % T], o["attn"].numpy().astype(np.uint8))
    assert np.abs(ro - o["o"].numpy()).max() < 1e-5
    assert tuple(pins["infer%d/z_shape" % T]) == tuple(o["z"].shape)
    z = o["z"].reshape(-1).numpy()
    assert np.abs(pins["infer%d/z" % T] - z[GR.sample_index(z.size, "z%d" % T)]).max() < 5e-5
