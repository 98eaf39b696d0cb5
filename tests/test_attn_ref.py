"""CPU: the float64 attention restatement and error bound of tests/attn_ref.py.  The restatement is pinned against the
oracle's rel_attention (itself pinned to the reference by test_oracle_vs_reference.py) on packed ragged batches; float32
restatements with other summation orders and with the tensor-core kernel's lazily refreshed running max must pass the
bound, and each deliberately corrupted output must fail it."""
import numpy as np
import pytest
import torch

import attn_ref as ar
from oracle import vits_oracle as vo

W, HEADS = 4, 2
LAYER, SRC = "enc.0", "enc_p.encoder.attn_layers.0"


@pytest.fixture(scope="module")
def tables(packed, cfg):
    return ar.layer_tables(packed[0], packed[1], LAYER, cfg["hidden_channels"] // HEADS)


def packed_qkv(lens, H, seed, kind="plain", tail=12):
    """qkv [rows, 3H] of a packed batch: utterance rows drawn by `kind`, gap and tail rows finite garbage."""
    rng = np.random.default_rng(seed)
    offs = ar.offsets(lens)
    x = rng.uniform(-30.0, 30.0, (offs[-1] + tail, 3 * H)).astype(np.float32)
    for b, n in enumerate(lens):
        u = rng.standard_normal((n, 3 * H))
        if kind == "peaky":
            u[:, :2 * H] *= 2.5
        elif kind == "growing":      # later keys score higher for every query: the running max is refreshed
            u[:, :H] = np.abs(u[:, :H])
            u[:, H:2 * H] = np.abs(u[:, H:2 * H]) * np.linspace(0.2, 4.0, n)[:, None]
        x[offs[b]:offs[b] + n] = u
    return x


def test_blob_tables_are_the_checkpoint_tables(tables, folded):
    ek = folded[SRC + ".emb_rel_k"][0].numpy()
    ev = folded[SRC + ".emb_rel_v"][0].numpy()
    assert np.array_equal(tables["relk"], ek) and np.array_equal(tables["relv"], ev)
    for nm, t in (("rk", ek), ("rv", ev)):
        hi, lo = tables[nm]
        assert np.all(np.abs(hi + lo - t) <= 2.0 ** -16 * np.abs(t))


@pytest.mark.parametrize("lens", [[3], [1, 4, 2], [37, 5, 70], [129]], ids=["T<W", "ragged-short", "ragged", "single"])
def test_restatement_matches_oracle(tables, cfg, lens):
    """rel_attention with 1x1 projections q, k, v = Wq x, Wk x, Wv x of an H-channel input (the oracle derives dk from the
    input width, so the selection is done by the projections) and conv_o = identity, on a masked batch."""
    H = cfg["hidden_channels"]
    rng = np.random.default_rng(len(lens) * 100 + lens[0])
    B, T = len(lens), max(lens)
    x = torch.tensor(rng.standard_normal((B, H, T)))
    mask = (torch.arange(T)[None, :] < torch.tensor(lens)[:, None]).double()
    w = {SRC + ".emb_rel_k": torch.tensor(tables["relk"], dtype=torch.float64)[None],
         SRC + ".emb_rel_v": torch.tensor(tables["relv"], dtype=torch.float64)[None]}
    proj = {}
    for nm in ("q", "k", "v"):
        proj[nm] = torch.tensor(rng.standard_normal((H, H)) / np.sqrt(H))
        w[SRC + ".conv_%s.weight" % nm], w[SRC + ".conv_%s.bias" % nm] = proj[nm][:, :, None], torch.zeros(H, dtype=torch.float64)
    w[SRC + ".conv_o.weight"], w[SRC + ".conv_o.bias"] = torch.eye(H, dtype=torch.float64)[:, :, None], torch.zeros(H, dtype=torch.float64)
    with torch.no_grad():
        ref = vo.rel_attention(x * mask[:, None], mask[:, None, :, None] * mask[:, None, None, :], w, SRC, HEADS, W).numpy()
    offs = ar.offsets(lens)
    qkv = np.full((offs[-1] + 4, 3 * H), 1e3, np.float32)
    for b, n in enumerate(lens):
        xb = x[b, :, :n].numpy()
        qkv[offs[b]:offs[b] + n] = np.concatenate([(proj[nm].numpy() @ xb).T for nm in ("q", "k", "v")], 1)
    for kind in ("ffma", "tc"):
        for b, (rows, out, bnd) in enumerate(ar.reference(qkv, lens, HEADS, W, tables, kind)):
            assert np.abs(out - ref[b, :, :lens[b]].T).max() < (1e-5 if kind == "ffma" else 2e-3), kind


@pytest.mark.parametrize("kind", ["plain", "peaky", "growing"])
def test_float32_restatements_within_bound(tables, cfg, kind):
    H = cfg["hidden_channels"]
    lens = [150, 9, 200]
    qkv = packed_qkv(lens, H, 7, kind)
    res = ar.reference(qkv, lens, HEADS, W, tables, "ffma")
    plain, _ = ar.f32_attention(qkv, lens, HEADS, W, tables["relk"], tables["relv"])
    lazy, refreshes = ar.f32_attention(qkv, lens, HEADS, W, tables["relk"], tables["relv"], lazy=ar.LAZY)
    if kind == "growing":
        assert refreshes > 0
    for out in (plain, lazy):
        for rows, ref, bnd in res:
            assert ar.within(out[rows], ref, bnd), ar.worst(out, res)


def test_tc_emulation_close_to_exact(tables, cfg):
    """The operand-exact emulation differs from the exact attention of the fp32 operands by the split-bf16 operand error
    only (~2^-16 relative per factor): a sanity check of the emulation, not of a kernel."""
    H = cfg["hidden_channels"]
    lens = [70, 33]
    qkv = packed_qkv(lens, H, 3)
    for (rows, a, _), (_, b, _) in zip(ar.reference(qkv, lens, HEADS, W, tables, "tc"), ar.reference(qkv, lens, HEADS, W, tables, "ffma")):
        assert np.abs(a - b).max() < 1e-3


CORRUPTIONS = {
    "band-edge-slot-dropped": dict(drop_slot=0),
    "band-slot-shifted": dict(shift=1),
    "ev-dropped": dict(no_ev=True),
    "last-key-masked": dict(mask_last=True),
    "row-beyond-len-unmasked": dict(unmask_next=True),
    "rel-logits-scaled-twice": dict(rel_scale2=True),
    "head-channels-offset-32": dict(head_shift=True),
    "ql-kh-dropped": dict(drop_qlkh=True),
}


@pytest.mark.parametrize("name", list(CORRUPTIONS))
def test_bound_rejects_corrupted_output(tables, cfg, name):
    H = cfg["hidden_channels"]
    lens = [70, 9, 33]
    qkv = packed_qkv(lens, H, 11, "peaky")
    res = ar.reference(qkv, lens, HEADS, W, tables, "tc")
    bad = ar.reference(qkv, lens, HEADS, W, tables, "tc", corrupt=CORRUPTIONS[name])
    assert not all(ar.within(o, ref, bnd) for (_, o, _), (_, ref, bnd) in zip(bad, res)), name


def test_bound_rejects_refresh_without_rescale(tables, cfg):
    H = cfg["hidden_channels"]
    lens = [150, 9, 200]
    qkv = packed_qkv(lens, H, 7, "growing")
    bad, refreshes = ar.f32_attention(qkv, lens, HEADS, W, tables["relk"], tables["relv"], lazy=ar.LAZY, no_rescale=True)
    assert refreshes > 0
    for kind in ("ffma", "tc"):
        res = ar.reference(qkv, lens, HEADS, W, tables, kind)
        assert not all(ar.within(bad[rows], ref, bnd) for rows, ref, bnd in res), kind
