"""StableTTS on the GPU, as far as it is built: the conditional-flow-matching decoder that turns the text encoder's output,
already expanded to frames, into a mel spectrogram (CFM.forward of training/stabletts/matcha/models/components/flow_matching.py,
called at matcha_tts.py:183).  The text encoder, the duration predictor and the vocoder are not part of this module: a caller
supplies mu_y (matcha_tts.py:170-171) and vocodes the mel itself."""
import numpy as np

from . import config as _config
from . import weights as _weights


class StableTTS:
    """A MatchaTTS (StableTTS) checkpoint's flow-matching decoder on one GPU."""

    def __init__(self, config, checkpoint, device=0, precision=1):
        """config: overrides of config.STABLETTS_CFM (n_spks, spk_emb_dim, ...) or None; checkpoint: a path (Lightning's
        `state_dict` entry is taken when present) or a state dict."""
        from .engine import Engine
        self.cfg = _config.stabletts_cfm_config(config)
        sd = _weights.load_checkpoint(checkpoint) if isinstance(checkpoint, str) else checkpoint
        sd = sd.get("state_dict", sd)
        blob, man = _weights.pack_stabletts_cfm(sd, self.cfg)
        self.engine = Engine(self.cfg, blob, man, device=device, precision=precision)

    def refine(self, mu_y, sid, n_timesteps=10, temperature=1.0, guidance_scale=0.5, noise=None, seed=0, denormalise=False):
        """mu_y: the aligned encoder output [cond_channels, T] of one utterance, or a list of them; sid: a speaker id for all, or
        one per utterance; noise: [noise_channels, T] per utterance standing in for torch.randn, or None for the engine's
        Philox(seed).  Returns the mel [noise_channels, T] of each utterance (a list for a list), normalised as the model
        produces it unless denormalise."""
        single = not isinstance(mu_y, (list, tuple))
        items = [mu_y] if single else list(mu_y)
        rows = [np.ascontiguousarray(np.asarray(m, np.float32).T) for m in items]
        nz = None
        if noise is not None:
            nz = [np.ascontiguousarray(np.asarray(n, np.float32).T) for n in ([noise] if single else list(noise))]
        mel, lengths = self.engine.cfm_decode(rows, sid, n_timesteps=n_timesteps, temperature=temperature,
                                              guidance_scale=guidance_scale, noise=nz, seed=seed, denormalise=denormalise)
        out = [np.ascontiguousarray(mel[b, :int(lengths[b])].T) for b in range(len(items))]
        return out[0] if single else out

    def close(self):
        self.engine.close()
