"""BERT on the GPU (vtts_bert_features, StableTTS.bert_features) against the float64 oracle, which matches transformers'
BertModel as bert-export.py calls it (tests/test_bert_host.py), in precision modes 0 and 1.

Error budgets, max |engine - float64 oracle| over every row of a sentence (the rows are LayerNorm outputs of O(1)), stated
before the first run: 3e-5 in mode 0 (fp32 FFMA), 5e-4 in mode 1 (split-bf16 tensor cores).  ContentVec's transformer, the
same layers at the same shape, measured 4.6e-6 and 1.1e-4."""
import numpy as np
import pytest
import torch

import bert_inputs as BI
import stabletts_cfm_inputs as SI
from oracle import bert_oracle as O

pytestmark = pytest.mark.gpu

BUDGET = {0: 3e-5, 1: 5e-4}
_TTS = {}
_REF = {}


def _tts(shape, precision):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from vosk_tts_b200.stabletts import StableTTS
    key = (shape, precision)
    if key not in _TTS:
        bt = getattr(BI, shape)()
        _TTS[key] = StableTTS(None, SI.model(), precision=precision, bert=(BI.model(bt), bt))
    return _TTS[key]


def _ref(shape, ids):
    key = (shape, ids.tobytes())
    if key not in _REF:
        bt = getattr(BI, shape)()
        _REF[key] = O.bert_features(BI.model(bt), bt, ids).numpy()
    return _REF[key]


def teardown_module(module):
    for t in _TTS.values():
        t.close()
    _TTS.clear()


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("shape", ["tiny", "production"])
def test_features_match_oracle(shape, precision):
    tts = _tts(shape, precision)
    bt = getattr(BI, shape)()
    for L in BI.LENGTHS:
        ids = BI.sentence(bt, L)
        got = tts.bert_features(ids)
        assert got.shape == (L, bt["cv_hidden"])
        err = float(np.abs(got - _ref(shape, ids)).max())
        print("bert %s mode %d L=%d: max|gpu - float64| = %.2e (budget %.0e)" % (shape, precision, L, err, BUDGET[precision]))
        assert err <= BUDGET[precision], (L, err)


@pytest.mark.parametrize("precision", [0, 1])
def test_ragged_batch_equals_alone(precision):
    tts = _tts("production", precision)
    bt = BI.production()
    sents = BI.ragged(bt, 64)
    batch = tts.bert_features(sents)
    for i, ids in enumerate(sents):
        alone = tts.bert_features(ids)
        assert np.array_equal(batch[i], alone), i
    worst = 0.0
    for i in range(0, 64, 16):
        worst = max(worst, float(np.abs(batch[i] - _ref("production", sents[i])).max()))
    print("bert ragged 64 mode %d: bit-identical alone; max|gpu - float64| over 4 sentences = %.2e" % (precision, worst))
    assert worst <= BUDGET[precision]


@pytest.mark.parametrize("precision", [0, 1])
def test_graph_replay_equals_eager(precision):
    tts = _tts("tiny", precision)
    eng = tts.engine
    bt = BI.tiny()
    sents = [BI.sentence(bt, L, salt=9) for L in (5, 33, 17)]
    first = tts.bert_features(sents)
    r0 = eng.graph_replays()
    second = tts.bert_features(sents)
    assert eng.graph_replays() > r0
    for a, b in zip(first, second):
        assert np.array_equal(a, b)
    eng.set_graphs(False)
    try:
        eager = tts.bert_features(sents)
    finally:
        eng.set_graphs(True)
    for a, b in zip(first, eager):
        assert np.array_equal(a, b)


def test_refusals():
    from vosk_tts_b200.engine import VttsError
    from vosk_tts_b200.stabletts import StableTTS
    tts = _tts("tiny", 0)
    bt = BI.tiny()
    ok = BI.sentence(bt, 9)
    for bad, what in ((np.array([2, bt["bt_vocab"], 3]), "vocabulary"), (np.array([2, -1, 3]), "vocabulary"),
                      (BI.sentence(bt, bt["bt_max_pos"] + 1), "position table")):
        with pytest.raises(VttsError, match=what) as e:
            tts.bert_features(bad)
        assert e.value.code == -1
    with pytest.raises(ValueError, match="at least one sentence"):
        tts.bert_features([])
    assert np.array_equal(tts.bert_features(ok), tts.bert_features(ok))      # the engine still serves after a refusal
    plain = StableTTS(None, SI.model(), precision=0)
    try:
        with pytest.raises(VttsError, match="no BERT"):
            plain.bert_features(ok)
    finally:
        plain.close()
