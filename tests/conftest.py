import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
GOLDEN_CASES = ["t17_sid2", "t128_sid2", "t50_slow", "t33_nonoise", "ragged3", "t1_single"]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def cfg():
    from vosk_tts_b200 import config
    return config.DEFAULT_CONFIG


@pytest.fixture(scope="session")
def checkpoint(cfg):
    from vosk_tts_b200 import synthetic
    return synthetic.make_random_checkpoint(cfg, 1234)


@pytest.fixture(scope="session")
def folded(checkpoint):
    from vosk_tts_b200 import weights
    return weights.fold_weight_norm(checkpoint)


@pytest.fixture(scope="session")
def packed(folded, cfg):
    from vosk_tts_b200 import weights
    return weights.pack(folded, cfg)


@pytest.fixture(scope="session", params=[0, 1, 2, 3], ids=["fp32-ffma", "tcgen05-flow-decoder", "tcgen05-all", "tcgen05-all-exact-encoder"])
def engine(request, packed, cfg):
    """precision 0: fp32 FFMA kernels everywhere; 1: flow + decoder convs (and batched attention) on wgmma (split-bf16, 3 MMAs
    per K16 slice); 2: text encoder too; 3: text encoder on wgmma with the exact 3-way split (6 MMAs per K16 slice).
    (The ids keep the names the tensor-core modes were first given; they select precision modes, not an instruction set.)"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.engine import Engine
    e = Engine(cfg, packed[0], packed[1], device=0, precision=request.param)
    e.precision = request.param
    yield e
    e.close()


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))
