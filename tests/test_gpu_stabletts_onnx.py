"""A multistream voice loaded from its exported model.onnx (StableTTS.from_onnx, Model over a deployed directory) on the GPU:
durations, mel and waveform against what the reference's own synthesise and vocoder give for the modules the graph was exported
from (tests/golden/ref_stabletts_onnx.npz, oracle/make_golden_stabletts_onnx.py), in modes 0 and 1; a ragged batch against the
single calls; the step-count refusal; Synth and the CLI end to end."""
import os
import subprocess
import sys
import wave

import numpy as np
import pytest

import stabletts_onnx_inputs as SI
from test_stabletts_onnx_host import GOLDEN, _deployed_dir
from vosk_tts_b200.model import Model
from vosk_tts_b200.stabletts import StableTTS
from vosk_tts_b200.synth import Synth

pytestmark = pytest.mark.gpu
# what the checkpoint path meets: max |mel - reference| on the normalised mel, and max |wav - reference| per precision mode
# (measured on an H100 80GB HBM3 at 700 W: 3.6e-6; 5.5e-7 in mode 0 and 6.0e-6 in mode 1)
MEL_BUDGET = 2.6e-5
WAV_BUDGET = {0: 1.2e-6, 1: 1.2e-5}
N_UTT = 4


@pytest.fixture(scope="module")
def fix():
    return dict(np.load(os.path.join(GOLDEN, "ref_stabletts_onnx.npz")))


@pytest.fixture(scope="module")
def graph_path(tmp_path_factory, fix):
    return SI.write_graph(tmp_path_factory.mktemp("stabletts_onnx"), fix)


@pytest.fixture(scope="module", params=[0, 1], ids=["fp32", "mode1"])
def tts(request, graph_path):
    t = StableTTS.from_onnx(graph_path, device=0, precision=request.param)
    t.precision = request.param
    yield t
    t.close()


def _utterances(fix):
    return [tuple(fix["u%d.%s" % (i, k)] for k in ("ids", "bert", "pause", "sid", "noise")) for i in range(N_UTT)]


def _run(tts, fix, us):
    return tts.synthesise([u[0] for u in us], [u[1] for u in us], [int(u[3]) for u in us], [u[2] for u in us],
                          n_timesteps=tts.n_timesteps, temperature=float(fix["temperature"]), length_scale=float(fix["length_scale"]),
                          noise=[u[4] for u in us], return_wav=True)


def test_matches_the_reference(tts, fix):
    std = float(tts.mel_std)
    for i, u in enumerate(_utterances(fix)):
        r = _run(tts, fix, [u])
        ref_w, ref_mel, ref_wav = (fix["u%d.%s" % (i, k)] for k in ("w_round", "mel", "wav"))
        assert np.array_equal(r["durations"][0], ref_w.astype(r["durations"][0].dtype)), i
        mel, wav = r["mel"][0], r["wav"][0]
        assert mel.shape == ref_mel.shape and wav.shape == ref_wav.shape
        e_mel, e_wav = float(np.abs(mel - ref_mel).max()) / std, float(np.abs(wav - ref_wav).max())
        print("u%d mode %d: |mel - ref| / mel_std %.2e  |wav - ref| %.2e" % (i, tts.precision, e_mel, e_wav))
        assert e_mel < MEL_BUDGET and e_wav < WAV_BUDGET[tts.precision], (i, e_mel, e_wav)


def test_ragged_batch_equals_single_calls(tts, fix):
    us = _utterances(fix)
    batch = _run(tts, fix, us)
    for i, u in enumerate(us):
        one = _run(tts, fix, [u])
        assert np.array_equal(batch["durations"][i], one["durations"][0])
        for k in ("mel", "wav"):
            diff = float(np.abs(batch[k][i] - one[k][0]).max())
            if tts.precision == 0:
                assert diff == 0.0, (i, k)
            else:              # the tensor-core split-K plans follow the batch shape (DESIGN.md 4.n)
                assert diff < 2e-4, (i, k, diff)


def test_prior_is_refused(tts, fix):
    u = _utterances(fix)[0]
    with pytest.raises(RuntimeError, match="no mel encoder"):
        tts.synthesise(u[0], u[1], int(u[3]), n_timesteps=3, noise=u[4], return_prior=True)


def test_model_and_synth_from_the_deployed_directory(tmp_path):
    d = _deployed_dir(tmp_path)
    with pytest.raises(ValueError, match="unrolls 3 flow-matching steps"):
        Model(model_path=d, n_timesteps=4)
    model = Model(model_path=d, precision=0)
    try:
        assert model.onnx.n_timesteps == 3
        out = str(tmp_path / "out.wav")
        Synth(model).synth("Привет, мир! Ещё раз.", out, speaker_id=2)
        with wave.open(out, "rb") as w:
            assert (w.getnchannels(), w.getsampwidth(), w.getframerate()) == (1, 2, 22050)
            pcm = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)
        assert pcm.size > 0 and np.abs(pcm).max() > 0
    finally:
        model.onnx.close()
    out = tmp_path / "cli.wav"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "vosk_tts_b200.cli", "-m", str(d), "-i", "Привет, мир!", "-o", str(out)], cwd=root,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    with wave.open(str(out), "rb") as w:
        assert w.getframerate() == 22050 and w.getnframes() > 0
