"""CPU restatement of the QuickVC speaker encoder (SpeakerEncoder, vc/models.py:728-767) as plain float64 functions.

The target's log-mel is vc_oracle.mel_spectrogram (vc/mel_processing.py differs from the VITS2 module only in dead code).
"""
import numpy as np

SLICE, HOP = 128, 64        # embed_utterance(partial_frames=128, partial_hop=64)


def slices(T):
    """(start, length) of every sequence embed_utterance runs for a clip of T mel frames (models.py:739-760)."""
    if T <= SLICE:
        return [(0, T)]
    return [(s, SLICE) for s in range(0, T - SLICE, HOP)] + [(T - SLICE, SLICE)]


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_recurrence(xp, whh):
    """One LSTM layer from its projected inputs: xp [T][4G] = W_ih x_t + b_ih + b_hh, whh [4G][G] (gate order i, f, g, o).
    Returns h [T][G], float64, h_{-1} = c_{-1} = 0."""
    xp = np.asarray(xp, np.float64)
    whh = np.asarray(whh, np.float64)
    G = whh.shape[1]
    h, c = np.zeros(G), np.zeros(G)
    out = np.zeros((xp.shape[0], G))
    for t in range(xp.shape[0]):
        z = xp[t] + whh @ h
        i, f, g, o = _sigmoid(z[:G]), _sigmoid(z[G:2 * G]), np.tanh(z[2 * G:3 * G]), _sigmoid(z[3 * G:])
        c = f * c + i * g
        h = o * np.tanh(c)
        out[t] = h
    return out


def lstm_input(x, sd, layer):
    """Projected inputs W_ih x + b_ih + b_hh of one layer, float64 [T][4G]."""
    p = "enc_spk.lstm.%s_l%d"
    f = lambda n: np.asarray(sd[p % (n, layer)], np.float64)
    return np.asarray(x, np.float64) @ f("weight_ih").T + f("bias_ih") + f("bias_hh")


def embed(mel, sd, n_layers=3):
    """g of one clip from its log-mel [n_mel][T] (SpeakerEncoder.embed_utterance(mel.transpose(1, 2)), models.py:865)."""
    mel = np.asarray(mel, np.float64)
    W = np.asarray(sd["enc_spk.linear.weight"], np.float64)
    b = np.asarray(sd["enc_spk.linear.bias"], np.float64)
    es = []
    for s, L in slices(mel.shape[1]):
        x = mel[:, s:s + L].T
        for l in range(n_layers):
            x = lstm_recurrence(lstm_input(x, sd, l), np.asarray(sd["enc_spk.lstm.weight_hh_l%d" % l]))
        e = np.maximum(W @ x[-1] + b, 0.0)
        es.append(e / np.linalg.norm(e))
    return np.mean(es, axis=0)
