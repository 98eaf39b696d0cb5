"""Inputs of the QuickVC speaker-encoder tests: the configuration, the seeded speaker encoder and the target clips (int16
16 kHz slices of the reference tree's vc/test_data, stored in tests/golden/quickvc_targets.npz)."""
import os

import numpy as np

from vosk_tts_b200 import config as C, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 4321
# the published vc/configs/quickvc.json, minus the training-only blocks
QUICKVC_JSON = {
    "data": {"max_wav_value": 32768.0, "sampling_rate": 16000, "filter_length": 1280, "hop_length": 320, "win_length": 1280,
             "n_mel_channels": 80, "mel_fmin": 0.0, "mel_fmax": None, "add_blank": True, "n_speakers": 0},
    "model": {"ms_istft_vits": True, "mb_istft_vits": False, "istft_vits": False, "subbands": 4, "gen_istft_n_fft": 16,
              "gen_istft_hop_size": 4, "inter_channels": 192, "hidden_channels": 192, "filter_channels": 768, "n_heads": 2,
              "n_layers": 6, "kernel_size": 3, "p_dropout": 0.1, "resblock": "1", "resblock_kernel_sizes": [3, 7, 11],
              "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]], "upsample_rates": [5, 4],
              "upsample_initial_channel": 512, "upsample_kernel_sizes": [16, 16], "n_layers_q": 3, "use_spectral_norm": False,
              "gin_channels": 256, "use_sdp": False, "ssl_dim": 1024, "use_spk": False},
}
# (key, file, first sample, samples): under 128 mel frames, just over 128 (129 frames: two slices), about 8 s
TARGETS = [("short", "p225_001.wav", 0, 26007), ("t129", "p226_005.wav", 1600, 129 * 320 + 5),
           ("long", "4280-185518-0004.wav", 0, 8 * 16000 + 123)]


def config():
    return C.from_quickvc_json(QUICKVC_JSON)


def speaker_encoder():
    return synthetic.make_random_speaker_encoder(config(), SEED)


def targets():
    z = np.load(os.path.join(GOLDEN, "quickvc_targets.npz"))
    return {k: z[k] for k, _, _, _ in TARGETS}


def wav_float(x):
    return (np.asarray(x, np.float32) / 32768.0).astype(np.float32)
