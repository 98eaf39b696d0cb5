"""GPU (-m gpu): the relative-position attention kernels in isolation -- attn_tc_kernel<dk> (csrc/attn_tc.cuh: wgmma with
split-bf16 operands, P in registers, lazily refreshed online softmax) and the fp32 FFMA attn_split_kernel<dk> /
attn_kernel<dk, R> (csrc/kernels.cuh) -- one launch at a time through the engine's own launch code
(vtts_debug_attention), on packed ragged batches, against the float64 reference and error bound of tests/attn_ref.py:
  tensor cores   operand-exact emulation of the products the kernel issues
  FFMA           exact attention of the kernels' fp32 operands
Every case pins the kernel and asserts the launch the engine reports (kernel, dk template, R, grid), so a change of the
selection heuristics cannot quietly move it onto another kernel.  Every case also checks that output rows outside the
utterances keep the sentinel written beforehand, that the output planes equal the device split of the fp32 output bit for
bit, that a second launch is bit-identical and, on batches, that other data in the gap and tail rows or in a neighbouring
utterance leaves every other utterance's output bit-identical.  Gap and tail rows of qkv hold finite garbage: the kernels'
masks (and, for the tensor-core input planes, the engine's zero_tails pass) must keep it out.

Head widths: the default model (dk 96 in the encoder and the flow) and synthetic checkpoints built here with hidden 128 /
4 heads (encoder dk 32, flow dk 64) and hidden 256 / 2 heads (dk 128); windows 1, 6 (the tensor-core band scratch exactly
full) and 7 (tensor cores refused).  All engines run precision mode 2, so the encoder layers have the tensor-core tables."""
import json

import numpy as np
import pytest
import torch

import attn_ref as ar
import conv_ref as cr
from vosk_tts_b200 import synthetic, weights
from vosk_tts_b200.engine import VttsError

pytestmark = pytest.mark.gpu
SENT = np.float32(777.25)
PSENT = np.uint16(0x7E7E)
LAYERS = ["enc.0", "flow.0.tr"]
KERNELS = ["tc", "split", "r1", "r4"]
KINDS = ["plain", "peaky", "growing", "lazy_under", "lazy_over", "dominant"]
VARIANTS = {"d96": {}, "d32": dict(hidden_channels=128, n_heads=4), "d128": dict(hidden_channels=256, n_heads=2),
            "w1": dict(window_size=1), "w6": dict(window_size=6), "w7": dict(window_size=7)}
WORST = {}                   # largest error / bound seen per kernel


@pytest.fixture(scope="module")
def engines(packed, cfg):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    made = {}

    def get(name):
        if name not in made:
            c = dict(cfg, **VARIANTS[name])
            blob, man = packed if name == "d96" else weights.pack(
                weights.fold_weight_norm(synthetic.make_random_checkpoint(c, 4321)), c)
            made[name] = (Engine(c, blob, man, device=0, precision=2), blob, man, {})
        return made[name]
    yield get
    for e, _, _, _ in made.values():
        e.close()
    print("\nattention error / bound, largest per kernel: " + json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


def _geom(e, layer):
    c = e.cfg
    H = c["hidden_channels"]
    heads = c["n_heads"] if layer.startswith("enc.") else c.get("flow_n_heads", 2)
    return H, heads, H // heads, c["window_size"]


def _utterance(rng, n, H, heads, kind):
    dk = H // heads
    u = rng.standard_normal((n, 3 * H))
    if kind == "peaky":                     # wide score distribution
        u[:, :2 * H] *= 2.5
    elif kind == "growing":                 # later keys score higher for every query: the running max is refreshed
        u[:, :H] = np.abs(u[:, :H])
        u[:, H:2 * H] = np.abs(u[:, H:2 * H]) * np.linspace(0.2, 3.0, n)[:, None]
    elif kind in ("lazy_under", "lazy_over"):
        # scores rise by just under / just over ATC_LAZY = 6 from one 64-key tile to the next: the lazily refreshed running
        # max is kept / refreshed at every tile
        step = 5.9 if kind == "lazy_under" else 6.1
        t = (np.arange(n) // ar.TC_KT)[:, None]
        u[:, :H] = 1.0 + 0.05 * u[:, :H]
        u[:, H:2 * H] = t * step / np.sqrt(dk) + 0.05 * u[:, H:2 * H]
    elif kind == "dominant":                # one row dominated by a single key
        i0, j0 = n // 3, n // 2
        u[j0, H:2 * H] = 4.0 * u[i0, :H]
    return u


def make_qkv(lens, H, heads, seed, kind, tail):
    rng = np.random.default_rng(seed)
    offs = cr.offsets(lens)
    x = rng.uniform(-1e3, 1e3, (offs[-1] + tail, 3 * H))       # finite garbage in gap and tail rows
    for b, n in enumerate(lens):
        x[offs[b]:offs[b] + n] = _utterance(rng, n, H, heads, kind)
    return x.astype(np.float32)


def expected_report(kernel, lens, launch, heads, dk):
    ml = max(launch or lens)
    rows = {"tc": 128, "split": 4, "r1": 8, "r4": 32}[kernel]
    return dict(kernel=kernel, dk=dk, R={"tc": 0, "split": 1, "r1": 1, "r4": 4}[kernel], grid_x=-(-ml // rows), grid_y=heads,
                grid_z=len(lens))


def tables(ent, layer, dk):
    e, blob, man, cache = ent
    if layer not in cache:
        cache[layer] = ar.layer_tables(blob, man, layer, dk)
    return cache[layer]


def run_case(ent, layer, kernel, lens, kind="plain", launch=None, tail=70, seed=0, p_planes=2):
    """One launch (and its repeats), checked against attn_ref.  Returns the launch report."""
    e = ent[0]
    H, heads, dk, W = _geom(e, layer)
    qkv = make_qkv(lens, H, heads, seed, kind, tail)
    rows = qkv.shape[0]
    out0 = np.full((rows, H), SENT, np.float32)
    pl0 = np.full((p_planes, rows * H), PSENT, np.uint16)
    runs = [e.debug_attention(layer, qkv, lens, kernel, launch, out=out0, planes=pl0) for _ in range(2)]
    (o, pl, rep, _), (o2, pl2, rep2, _) = runs
    assert rep == rep2
    if kernel in KERNELS:
        exp = expected_report(kernel, lens, launch, heads, dk)
        assert {k: rep[k] for k in exp} == exp, "launch %s, expected %s" % (rep, exp)
    assert rep["dk"] == dk
    assert np.array_equal(o.view(np.uint32), o2.view(np.uint32)) and np.array_equal(pl, pl2), "two launches differ"
    # ---- values within the bound
    res = ar.reference(qkv, lens, heads, W, tables(ent, layer, dk), "tc" if rep["kernel"] == "tc" else "ffma")
    assert np.isfinite(o).all()
    ratio = ar.worst(o, res)
    WORST[rep["kernel"]] = max(WORST.get(rep["kernel"], 0.0), ratio)
    assert ratio <= 1.0, "%s %s lens %s: error %.3g x the bound" % (layer, rep, lens[:8], ratio)
    # ---- rows outside the utterances untouched, output planes = the device split of the output
    inside = np.zeros(rows, bool)
    for r, _, _ in res:
        inside[r] = True
    assert np.all(o[~inside].view(np.uint32) == SENT.view(np.uint32)), "rows outside the utterances written"
    pl = pl.reshape(p_planes, rows, H)
    assert np.all(pl[:, ~inside] == PSENT), "plane rows outside the utterances written"
    assert np.array_equal(pl[:, inside], cr.split_planes(o[inside], p_planes)), "output planes != split(out)"
    if rep["kernel"] == "tc":
        # the production launch: planes only
        _, pq, rep3, _ = e.debug_attention(layer, qkv, lens, kernel, launch, out=False, planes=pl0)
        assert rep3 == rep
        assert np.array_equal(pq.reshape(p_planes, rows, H), pl), "planes-only launch differs"
        recon = cr.bf16_value(pl[0]) + cr.bf16_value(pl[1])
        for r, ref, bnd in res:
            assert ar.within(recon[r], ref, bnd * (1 + 2.0 ** -16) + 2.0 ** -16 * np.abs(ref))
    if len(lens) > 1:
        # other garbage in gap / tail rows and other data in utterance 0: every other utterance bit-identical
        rng = np.random.default_rng(seed + 1)
        q2 = qkv.copy()
        q2[~inside] = rng.uniform(-1e3, 1e3, q2[~inside].shape)
        offs = cr.offsets(lens)
        q2[offs[0]:offs[0] + lens[0]] = _utterance(rng, lens[0], H, heads, "plain")
        o3, _, _, _ = e.debug_attention(layer, q2, lens, kernel, launch, out=out0, planes=pl0)
        for b in range(1, len(lens)):
            r = slice(offs[b], offs[b] + lens[b])
            assert np.array_equal(o3[r].view(np.uint32), o[r].view(np.uint32)), "utterance %d depends on other rows" % b
    return rep


def _fits_split(lens, launch, heads, dk, W):
    """attn_split_fits restated: key tiles of the longest launch length resident in shared memory, CTAs in one wave."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    ll = launch or lens
    mt = -(-max(ll) // 32)
    nrel = 2 * W + 1
    floats = 2 * mt * 32 * (dk + 4) + 4 * (dk + 4) + 2 * nrel * (dk + 4) + 4 * nrel + 16 * 32 + 16 * (4 + dk)
    return mt <= 8 and sum(-(-n // 4) for n in ll) * heads <= n_sm and floats * 4 <= 227 * 1024


def _cases():
    cases = []
    singles = [1, 2, 4, 5, 31, 32, 33, 63, 64, 65, 127, 128, 129, 193, 255, 256, 257, 1000, 4765]
    batches = [([1, 129, 64, 300], None, 70), ([5, 1, 7], None, 70), ([5, 1, 7], [64, 64, 64], 70), ([33, 65], None, 0),
               ([5, 1, 7], None, 0), ([1, 129, 64, 300], [300] * 4, 70), ([100], [128], 70)]
    b64 = [int(v) for v in torch.randint(64, 257, (64,), generator=torch.Generator().manual_seed(1))]
    for layer in LAYERS:
        for kernel in KERNELS:
            for i, T in enumerate(singles):
                cases.append(("d96", layer, kernel, [T], None, KINDS[i % 3], 70))
            for kind in KINDS:
                cases.append(("d96", layer, kernel, [256 if kernel == "split" else 300], None, kind, 70))
            for lens, launch, tail in batches:
                cases.append(("d96", layer, kernel, lens, launch, "plain", tail))
            cases.append(("d96", layer, kernel, b64, None, "peaky", 70))
            for v, Ts in (("d32", [1, 33, 65, 129, 193, 256, 300]), ("d128", [1, 33, 65, 129, 192, 193, 256, 300]),
                          ("w1", [1, 2, 65, 300]), ("w6", [1, 6, 7, 65, 129, 300]), ("w7", [1, 7, 8, 65, 300])):
                for i, T in enumerate(Ts):
                    cases.append((v, layer, kernel, [T], None, KINDS[i % len(KINDS)], 70))
                for lens, launch, tail in batches[:3]:
                    cases.append((v, layer, kernel, lens, launch, "plain", 70))
    return cases


def _id(c):
    v, layer, kernel, lens, launch, kind, tail = c
    s = "%s-%s-%s-%s" % (v, layer, kernel, "x".join(map(str, lens)) if len(lens) <= 4 else "b%d" % len(lens))
    return s + ("-launch%d" % max(launch) if launch else "") + "-" + kind + ("-notail" if tail == 0 else "")


@pytest.mark.parametrize("case", _cases(), ids=_id)
def test_attention_kernel(engines, case):
    v, layer, kernel, lens, launch, kind, tail = case
    ent = engines(v)
    H, heads, dk, W = _geom(ent[0], layer)
    refused = (kernel == "tc" and 2 * W + 1 > 13) or (kernel == "split" and not _fits_split(lens, launch, heads, dk, W))
    if refused:
        with pytest.raises(VttsError, match="not available" if kernel == "tc" else "does not fit") as ei:
            ent[0].debug_attention(layer, make_qkv(lens, H, heads, 0, kind, tail), lens, kernel, launch)
        assert ei.value.code == -1          # VTTS_ERR_INVALID, before any launch
        return
    p_planes = 3 if (kernel in ("r1", "r4", "split") and kind == "plain") else 2
    run_case(ent, layer, kernel, lens, kind, launch, tail, seed=len(lens) * 1000 + lens[0], p_planes=p_planes)


@pytest.mark.parametrize("T", [193, 256])
@pytest.mark.parametrize("layer", LAYERS)
def test_split_kv_overflow_falls_back_dk128(engines, layer, T):
    """dk 128 at W 4: the split-KV kernel's key tiles need 258,800 B of shared memory at 7 tiles (T 193..224) and 292,592 B
    at 8 (T 225..256), more than the 227 KB a kernel may have.  The engine's own choice must not pick it: tensor cores where
    the layer has them, attn_kernel R=1 among the FFMA kernels."""
    ent = engines("d128")
    H, heads, dk, W = _geom(ent[0], layer)
    assert dk == 128 and not _fits_split([T], None, heads, dk, W)
    assert run_case(ent, layer, "auto", [T], "plain")["kernel"] == "tc"
    assert run_case(ent, layer, "ffma", [T], "plain")["kernel"] == "r1"


@pytest.mark.parametrize("layer", LAYERS)
def test_auto_selection_on_benchmark_shapes(engines, layer):
    """For the shipped configuration (dk 96, W 4) the shared-memory test changes nothing: at every length the split-KV kernel
    is eligible for it also fits.  The engine's choice on the benchmark's shapes stays: split-KV for a single utterance of
    162 frames, tensor cores for 4765 frames and for a 64-utterance batch (attn_kernel R=4 among the FFMA kernels)."""
    ent = engines("d96")
    H, heads, dk, W = _geom(ent[0], layer)
    assert all(_fits_split([T], None, heads, dk, W) for T in range(1, 257))
    b64 = [int(v) for v in torch.randint(64, 257, (64,), generator=torch.Generator().manual_seed(1))]
    assert run_case(ent, layer, "auto", [162])["kernel"] == "split"
    assert run_case(ent, layer, "ffma", [162])["kernel"] == "split"
    assert run_case(ent, layer, "auto", [4765])["kernel"] == "tc"
    assert run_case(ent, layer, "ffma", [4765])["kernel"] == "r4"
    assert run_case(ent, layer, "auto", b64)["kernel"] == "tc"
    assert run_case(ent, layer, "ffma", b64)["kernel"] == "r4"


def test_window7_auto_uses_ffma(engines):
    ent = engines("w7")
    for layer in LAYERS:
        assert run_case(ent, layer, "auto", [300])["kernel"] in ("r1", "r4", "split")
