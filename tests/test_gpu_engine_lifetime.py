"""Destroying an engine gives back every byte it allocated, device and pinned host alike, whatever the handle did: synthesis,
streaming, conversion and alignment workspaces, profiling, the timeline, the debug and tool entry points, QuickVC with
ContentVec, workspace growth, a second handle on the same device and a failed vtts_create.  The counters
(engine.live_bytes) belong to this process, so other work on the GPU does not move them: the checks are exact."""
import numpy as np
import pytest
import torch

import contentvec_inputs as CI
import quickvc_convert_inputs as QC
import quickvc_inputs as QI
from vosk_tts_b200 import engine as E
from vosk_tts_b200 import monotonic_align, synthetic, weights

pytestmark = pytest.mark.gpu

_PACKED = {}


@pytest.fixture(autouse=True)
def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _vits(cfg):
    if "vits" not in _PACKED:
        sd = synthetic.make_random_checkpoint(cfg, 7, posterior=True)
        _PACKED["vits"] = weights.pack(weights.fold_weight_norm(sd), cfg, posterior=True)
    return _PACKED["vits"]


def _grew(base):
    now = E.live_bytes()
    assert now[0] > base[0] and now[1] > base[1], (base, now)


def _ids(cfg, T, seed=0):
    return (np.arange(T, dtype=np.int64) * 7 + 1 + seed) % int(cfg["n_vocab"])


def _debug_calls(e, cfg, precision):
    e.timeline(1)
    e.infer(_ids(cfg, 20)[None], [20], [0], (0.667, 1.0, 0.8), seed=3)
    e.timeline(2)
    e.timeline(0)
    e.microbench("tc:64:64:3:1:128" if precision >= 1 else "ffma:64:64:3:1:128", iters=4)
    H = int(cfg["hidden_channels"])
    rng = np.random.default_rng(0)
    e.debug_attention("enc.0", rng.standard_normal((20, 3 * H)).astype(np.float32), iters=2)
    C_, k, rows = 16, 3, 20
    prob = dict(Cin=C_, Cout=C_, k=k, dil=1, pad=1, w=rng.standard_normal((k, C_, C_)).astype(np.float32),
                bias=np.zeros(C_, np.float32), y_on=1, ldy=C_, ldx=C_)
    e.debug_conv(False, [rows], 1, [prob], rng.standard_normal((rows, C_)).astype(np.float32), y=np.zeros(rows * C_, np.float32))


@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_vits2_engine_gives_back_everything(cfg, precision):
    blob, man = _vits(cfg)
    base = E.live_bytes()
    e = E.Engine(cfg, blob, man, device=0, precision=precision)
    e.reserve(max_tokens=32, max_frames=128)
    e.infer(_ids(cfg, 24)[None], [24], [1], (0.667, 1.0, 0.8), seed=1)
    chunks = list(e.synthesize_stream(_ids(cfg, 30), 2, (0.667, 1.0, 0.8), chunk_frames=16, seed=2))
    assert len(chunks) >= 2
    e.reserve_convert(max_frames=64)
    e.reserve_align(max_tokens=16, max_frames=64)
    e.profile(True)
    e.infer(_ids(cfg, 24)[None], [24], [1], (0.667, 1.0, 0.8), seed=1)
    e.profile(False)
    _debug_calls(e, cfg, precision)
    _grew(base)
    e.close()
    assert E.live_bytes() == base


def test_quickvc_with_contentvec_gives_back_everything():
    blob, man = weights.pack_quickvc(weights.fold_weight_norm(QC.model()), QI.config(), contentvec=CI.model())
    cfg = dict(QI.config(), contentvec=CI.cv())
    base = E.live_bytes()
    e = E.Engine(cfg, blob, man, device=0, precision=1)
    wav = CI.speech(16000, 5)
    g = e.speaker_embedding(wav)
    e.quickvc_convert(QC.units(37, 1), g)
    e.content_units(wav)
    e.quickvc_convert_wav(wav, g)
    _grew(base)
    e.close()
    assert E.live_bytes() == base


def test_workspace_growth_gives_back_everything(cfg):
    blob, man = _vits(cfg)
    base = E.live_bytes()
    e = E.Engine(cfg, blob, man, device=0, precision=1)
    e.reserve(max_tokens=16, max_frames=64)
    small = E.live_bytes()
    e.reserve(max_tokens=128, max_frames=1024, batch=2)
    assert E.live_bytes()[0] > small[0]
    e.close()
    assert E.live_bytes() == base


def test_two_handles_on_one_device(cfg):
    blob, man = _vits(cfg)
    base = E.live_bytes()
    a = E.Engine(cfg, blob, man, device=0, precision=1)
    a.reserve(max_tokens=32, max_frames=128)
    mid = E.live_bytes()
    b = E.Engine(cfg, blob, man, device=0, precision=0)
    b.reserve(max_tokens=64, max_frames=256)
    assert E.live_bytes()[0] > mid[0]
    b.close()
    assert E.live_bytes() == mid
    a.infer(_ids(cfg, 24)[None], [24], [1], (0.667, 1.0, 0.8), seed=1)
    a.close()
    assert E.live_bytes() == base


def test_failed_create_gives_back_everything(cfg):
    blob, man = _vits(cfg)
    lines = man.splitlines()
    drop = next(i for i, ln in enumerate(lines) if ln.split()[0] == "enc.emb")      # bound in every precision mode
    base = E.live_bytes()
    with pytest.raises(E.VttsError):
        E.Engine(cfg, blob, "\n".join(lines[:drop] + lines[drop + 1:]) + "\n", device=0, precision=1)
    assert E.live_bytes() == base


def test_maximum_path_gives_back_everything():
    base = E.live_bytes()
    rng = np.random.default_rng(1)
    path = monotonic_align.maximum_path_numpy(rng.standard_normal((2, 40, 12)).astype(np.float32), [40, 31], [12, 9])
    assert path[0].sum() == 40 and path[1].sum() == 31
    assert E.live_bytes() == base
