"""SURVEY.md section 8f rank 3: the other inverse-STFT decoders of the reference (Multistream_iSTFT_Generator,
iSTFT_Generator).  The oracle restatement and the weight packing are pinned against what the UNMODIFIED reference
computed on CPU (tests/golden/ref_decoder_variants.npz, written by oracle/make_golden_ref.py); the CUDA engine's parity run
for them is tests/test_gpu_parity.py::test_istft_decoder_variants_vs_oracle."""
import numpy as np
import pytest
import torch

import golden_ref as GR
from oracle import vits_oracle as vo
from vosk_tts_b200 import config as C, synthetic, weights

N_VOCAB = GR.N_VOCAB
_training_json = GR.training_json


@pytest.mark.parametrize("flag,kind", GR.DECODER_VARIANTS)
def test_oracle_matches_reference_for_decoder_variant(flag, kind):
    ref = GR.load("ref_decoder_variants.npz")
    tj = _training_json(flag)
    cfg = C.from_training_json(tj, n_vocab=N_VOCAB)
    assert cfg["decoder"] == kind and C.hop_total(cfg) == (64 if kind == "istft" else 256)
    folded = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 11))
    tok, eps_dp, eps_z, scales = GR.variant_inputs(cfg)
    T = tok.shape[1]
    torch.set_num_threads(1)
    with torch.no_grad():
        o = vo.infer(folded, cfg, tok, torch.tensor([T]), torch.tensor([2]), scales, eps_dp, eps_z, return_all=True)
    assert np.array_equal(o["w_ceil"][0, 0].numpy().astype(np.int32), ref[flag + "/w"])
    assert np.array_equal(o["idx"][0].numpy(), ref[flag + "/idx"])
    shape = tuple(ref[flag + "/o_shape"])
    assert tuple(o["o"].shape) == shape and shape[-1] == int(o["y_lengths"][0]) * C.hop_total(cfg)
    flat = o["o"].reshape(-1).numpy()
    assert float(np.abs(flat[GR.sample_index(flat.size, flag)] - ref[flag + "/o"]).max()) < 1e-5


@pytest.mark.parametrize("flag", ["ms_istft_vits", "istft_vits"])
def test_packed_tail_filter_is_what_the_decoder_applies(flag):
    """pack() hands the CUDA tail kernel one 63-tap filter per band: the learned multistream filter, or a unit impulse."""
    tj = _training_json(flag)
    cfg = C.from_training_json(tj, n_vocab=N_VOCAB)
    folded = weights.fold_weight_norm(synthetic.make_random_checkpoint(cfg, 11))
    blob, man = weights.pack(folded, cfg, tc=False)
    ent = {}
    for line in man.strip().splitlines():
        parts = line.split()
        ent[parts[0]] = [int(x) for x in parts[1:]]
    off, n = ent["dec.pqmf"][0], ent["dec.pqmf"][1]
    bank = blob[off:off + n].reshape(-1, 63)
    if flag == "ms_istft_vits":
        assert np.array_equal(bank, folded["dec.multistream_conv_post.weight"][0].numpy())
        assert "dec.post.b" in ent            # models.py:1095: this conv_post has a bias
    else:
        assert bank.shape == (1, 63) and bank[0, 31] == 1.0 and np.count_nonzero(bank) == 1


def test_engine_config_accepts_every_istft_decoder():
    """All three inverse-STFT decoders map onto the same engine decoder type (the tail kernel takes the filter bank from
    the blob); the GPU parity runs are tests/test_gpu_parity.py::test_istft_decoder_variants_vs_oracle."""
    from vosk_tts_b200 import engine
    for flag in ("ms_istft_vits", "istft_vits", "mb_istft_vits"):
        cfg = C.from_training_json(_training_json(flag), n_vocab=N_VOCAB)
        cc = engine.make_c_config(cfg)
        assert cc.decoder_type == 0 and cc.subbands == (1 if flag == "istft_vits" else 4)
