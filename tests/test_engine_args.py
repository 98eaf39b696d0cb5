"""The Python side of the calls on recordings: batch-axis promotion, length defaults, ragged lists and the noise-shape
check.  The helpers are plain numpy; the entry points run on an Engine whose library only records what it is passed, so
no GPU is needed."""
import ctypes

import numpy as np
import pytest

from vosk_tts_b200 import config as Cf, engine as E

I, G = 192, 256


# ---- the helpers

@pytest.mark.parametrize("shape,ndim,t_axis,T", [((1000,), 2, -1, 1000), ((3, 1000), 2, -1, 1000), ((80, 50), 3, -1, 50),
                                                  ((2, 80, 50), 3, -1, 50), ((40, 768), 3, 1, 40), ((2, 40, 768), 3, 1, 40)])
def test_batch_axis_and_default_lengths(shape, ndim, t_axis, T):
    y, lengths = E._batch(np.ones(shape, np.float64), None, ndim, t_axis)
    B = shape[0] if len(shape) == ndim else 1
    assert y.dtype == np.float32 and y.flags.c_contiguous and y.ndim == ndim and y.shape[0] == B
    assert lengths.dtype == np.int64 and lengths.flags.c_contiguous and list(lengths) == [T] * B


def test_batch_given_lengths():
    x = np.zeros((3, 100), np.float32)[:, ::2]                # not contiguous
    y, lengths = E._batch(x, [10, 20, 30], 2)
    assert y.flags.c_contiguous and y.shape == (3, 50) and lengths.dtype == np.int64 and list(lengths) == [10, 20, 30]
    assert list(E._batch(x, 7, 2)[1]) == [7, 7, 7]            # one value for every item
    with pytest.raises(ValueError):
        E._batch(x, [1, 2], 2)


def test_batch_ragged():
    y, lengths = E._batch([np.ones(5, np.float32), 2 * np.ones((1, 9), np.float32)], None, 2, ragged=True)
    assert y.shape == (2, 9) and list(lengths) == [5, 9] and not y[0, 5:].any() and (y[1] == 2).all()
    y, lengths = E._batch([np.ones((4, 768)), np.ones((7, 768))], [1, 1], 3, t_axis=1, ragged=True)
    assert y.shape == (2, 7, 768) and list(lengths) == [4, 7] and not y[0, 4:].any()


@pytest.mark.parametrize("shape", [(2, I, 10), (2, I, 1)])
def test_noise_accepted(shape):
    n, ld = E._noise(np.zeros(shape, np.float64), 2, I)
    assert n.dtype == np.float32 and n.flags.c_contiguous and ld == shape[2]
    assert E._noise(None, 2, I) == (None, 0)


@pytest.mark.parametrize("shape", [(1, I, 10), (3, I, 10), (2, I - 1, 10), (2, I + 1, 10), (2, I), (2, I, 10, 1), (2, I, 0)])
def test_noise_refused(shape):
    with pytest.raises(ValueError, match="noise"):
        E._noise(np.zeros(shape, np.float32), 2, I)


def test_per_item():
    assert E._per_item(np.ones(G), 3, G).shape == (3, G)
    g = np.arange(2 * G, dtype=np.float64).reshape(2, G)
    assert np.array_equal(E._per_item(g, 2, G), g) and E._per_item(g, 2, G).dtype == np.float32


# ---- every entry point on recordings, through a recording library

class _Lib:
    """Stands in for libvtts: reads the batch size, row pitch and lengths each call is given, and reports success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*a):
            i = 5 if name in ("vtts_align", "vtts_align_spec") else 1       # (x, lengths, B, ld) start here
            B, ld = a[i + 2], a[i + 3]
            lengths = ctypes.cast(a[i + 1], ctypes.POINTER(ctypes.c_int64))
            self.calls.append((name, B, ld, [lengths[b] for b in range(B)]))
            return 0
        return call


@pytest.fixture
def eng():
    e = E.Engine.__new__(E.Engine)
    e.lib, e.h, e.hop = _Lib(), None, 256
    e.cfg = dict(Cf.DEFAULT_CONFIG, inter_channels=I, gin_channels=G, n_speakers=4, spec_channels=80)
    return e


def _wav(B, L=4000):
    return np.zeros((B, L), np.float32) if B else np.zeros(L, np.float32)


def _spec(B, T=20):
    return np.zeros((B, 80, T), np.float32) if B else np.zeros((80, T), np.float32)


def _units(B, T=20):
    return np.zeros((B, T, 768), np.float32) if B else np.zeros((T, 768), np.float32)


def _ids(x, ndim):
    return np.ones((len(x) if isinstance(x, list) or x.ndim == ndim else 1, 5), np.int64)


# name: (call, input maker, full length, keyword of the lengths)
CALLS = {
    "convert": (lambda e, x, **k: e.convert(x, 0, 1, **k), _wav, 4000, "lengths"),
    "convert_spec": (lambda e, x, **k: e.convert_spec(x, 0, 1, **k), _spec, 20, "lengths"),
    "speaker_embedding": (lambda e, x, **k: e.speaker_embedding(x, **k), _wav, 4000, "lengths"),
    "speaker_embedding_mel": (lambda e, x, **k: e.speaker_embedding_mel(x, **k), _spec, 20, "lengths"),
    "align": (lambda e, x, **k: e.align(_ids(x, 2), 5, 0, x, **k), _wav, 4000, "wav_lengths"),
    "align_spec": (lambda e, x, **k: e.align_spec(_ids(x, 3), 5, 0, x, **k), _spec, 20, "spec_lengths"),
    "content_units": (lambda e, x, **k: e.content_units(x, **k), _wav, 4000, "lengths"),
    "quickvc_convert": (lambda e, x, **k: e.quickvc_convert(x, np.zeros(G, np.float32), **k), _units, 20, "lengths"),
    "quickvc_convert_wav": (lambda e, x, **k: e.quickvc_convert_wav(x, np.zeros(G, np.float32), **k), _wav, 4000, "lengths"),
}
NOISE = ["convert", "convert_spec", "align", "align_spec", "quickvc_convert", "quickvc_convert_wav"]
RAGGED = ["content_units", "quickvc_convert", "quickvc_convert_wav"]


@pytest.mark.parametrize("name", sorted(CALLS))
@pytest.mark.parametrize("B", [0, 1, 3])
def test_entry_point_batch_and_lengths(eng, name, B):
    """One item without a batch axis is a batch of one; lengths default to the full rows; given lengths pass through."""
    call, make, full, kw = CALLS[name]
    call(eng, make(B))
    _, nb, ld, lengths = eng.lib.calls[-1]
    assert nb == max(B, 1) and ld == full and lengths == [full] * nb
    call(eng, make(B), **{kw: np.arange(full - nb + 1, full + 1)})
    assert eng.lib.calls[-1][3] == list(range(full - nb + 1, full + 1))


@pytest.mark.parametrize("name", RAGGED)
def test_entry_point_ragged_lists(eng, name):
    call, make, full, _ = CALLS[name]
    call(eng, [make(0)[: full // 2], make(0)])
    assert eng.lib.calls[-1][1:] == (2, full, [full // 2, full])


@pytest.mark.parametrize("name", sorted(set(CALLS) - set(RAGGED)))
def test_entry_point_ragged_lists_only_where_documented(eng, name):
    call, make, full, _ = CALLS[name]
    with pytest.raises(ValueError):
        call(eng, [make(0)[: full // 2], make(0)])


@pytest.mark.parametrize("name", NOISE)
@pytest.mark.parametrize("shape", [(1, I, 40), (3, I, 40), (2, I - 1, 40), (2, I + 1, 40), (2, I, 40, 1), (2, I)])
def test_entry_point_noise_shape(eng, name, shape):
    """Noise of the wrong batch, channel count or rank is refused before the library is called: the engine reads every
    [b, channel] row of a [B, inter_channels, noise_ld] array."""
    call, make, _, _ = CALLS[name]
    call(eng, make(2), noise=np.zeros((2, I, 40), np.float32))
    n = len(eng.lib.calls)
    with pytest.raises(ValueError, match="noise"):
        call(eng, make(2), noise=np.zeros(shape, np.float32))
    assert len(eng.lib.calls) == n
