"""GPT-SoVITS on the GPU.  Text-to-semantic decoding: the reference's Text2SemanticDecoder.infer_panel
(training/gpt-sovits/ar/models/t2s_model.py:324-448) behind its own signature, and a ragged batch of sentences in one call (Text2Semantic).  The prompt's tokens of a reference
recording: HuBERT and SynthesizerTrn.extract_latent (SemanticEncoder)."""
import numpy as np

from . import config as _config
from . import weights as _weights
from .engine import Engine


class Text2Semantic:
    """checkpoint: a path (either layout weights.load_t2s reads) or (state dict, config.t2s_config).  precision 0 runs every
    kernel on the fp32 FFMA pipe; >= 1 the text prefill on the split-bf16 tensor cores (the decode steps stay fp32)."""

    def __init__(self, checkpoint, device=0, precision=1):
        sd, cfg = _weights.load_t2s(checkpoint) if isinstance(checkpoint, str) else checkpoint
        self.cfg = cfg
        blob, manifest = _weights.pack_t2s(sd, cfg, tc=precision >= 1)
        self.engine = Engine(cfg, blob, manifest, device=device, precision=precision)
        self.EOS = int(cfg["t2s_vocab"]) - 1

    def close(self):
        self.engine.close()

    def infer_panel(self, x, x_lens, prompts, bert_feature, top_k=-100, top_p=100, early_stop_num=-1, temperature=1.0,
                    seed=0, repetition_penalty=1.35):
        """The reference's call at batch 1: x int [1, T], x_lens, prompts int [1, P] or None, bert_feature float [1, 1024, T]
        (None: zeros).  Returns (y int64 [1, P + n - 1], idx) as infer_panel does: y[:, :-1] with the prompt, and 0 without
        a prompt, else the loop index minus one.  The reference's default top_k of -100 keeps every entry, as topk of
        min(-100, V) would not run; it is taken as V here."""
        x = np.asarray(x).reshape(-1)[: int(np.asarray(x_lens).reshape(-1)[0])]
        bert = None
        if bert_feature is not None:
            f = np.asarray(bert_feature, np.float32).reshape(1024, -1)[:, : x.size]
            bert = [np.ascontiguousarray(f.T)] if np.any(f) else None
        pr = None if prompts is None else [np.asarray(prompts).reshape(-1)]
        k = int(top_k) if top_k is not None and top_k >= 1 else int(self.cfg["t2s_vocab"])
        toks, idx = self.engine.t2s_decode([x], pr, bert, top_k=k, top_p=float(top_p), temperature=float(temperature),
                                           repetition_penalty=repetition_penalty, early_stop_num=int(early_stop_num), seeds=seed)
        return toks[0][None, :], int(idx[0])

    def decode(self, phones_list, prompts=None, bert=None, top_k=20, top_p=0.6, temperature=0.6, repetition_penalty=1.35,
               early_stop_num=-1, seeds=0, q=None, step_cap=1500):
        """A ragged batch: phones_list B phone-id sequences, prompts None or B token sequences, bert None or B [T_b, 1024].
        Each sentence is decoded as if alone; seeds: one per sentence, or one int s giving sentence b the seed s + b.  Returns (list of B int64 token arrays, idx int64 [B])."""
        return self.engine.t2s_decode(phones_list, prompts, bert, top_k=top_k, top_p=top_p, temperature=temperature,
                                      repetition_penalty=repetition_penalty, early_stop_num=early_stop_num, step_cap=step_cap,
                                      seeds=seeds, q=q)


class SemanticEncoder:
    """The prompt's semantic tokens of GPT-SoVITS on the GPU: chinese-hubert-base over a reference recording, then the s2
    model's SynthesizerTrn.extract_latent (inference_cli.py:176-200, module/models.py:990-993), whose codes prompt
    Text2Semantic.decode.  sovits_checkpoint: an s2 G_*.pth (either layout weights.load_sovits reads, with its config.json as
    `config`) or (state dict, config.sovits_config).  hubert: a chinese-hubert-base directory (weights.load_contentvec) or
    (state dict, config.contentvec_config).  precision 0 runs HuBERT on the fp32 FFMA pipe; >= 1 its GEMMs and attention on
    the split-bf16 tensor cores.  ssl_proj, the codebook scores and their argmax are fp32 in every mode."""

    def __init__(self, sovits_checkpoint, hubert, config=None, device=0, precision=1):
        hsd, hcv = _weights.load_contentvec(hubert) if isinstance(hubert, str) else hubert
        if isinstance(sovits_checkpoint, str):
            if config is None:
                raise ValueError("an s2 checkpoint path needs its config.json (config=...): the prompt pad comes from its sampling_rate")
            sd, cfg = _weights.load_sovits(sovits_checkpoint, config)
        else:
            sd, cfg = sovits_checkpoint
        cfg = dict(cfg)
        cfg.update(hcv)
        self.cfg = cfg
        blob, manifest = _weights.pack_sovits(sd, cfg, hsd, tc=precision >= 1)
        self.engine = Engine(cfg, blob, manifest, device=device, precision=precision)

    def close(self):
        self.engine.close()

    def extract_latent(self, ssl_content):
        """SynthesizerTrn.extract_latent: HuBERT's last_hidden_state float [B, 768, T] -> int64 codes [B, 1, T // 2]."""
        x = np.asarray(ssl_content, np.float32)
        if x.ndim != 3:
            raise ValueError("ssl_content must be [B, %d, T]" % int(self.cfg["cv_hidden"]))
        codes, _ = self.engine.sovits_latent(np.ascontiguousarray(x.transpose(0, 2, 1)))
        return codes[:, None, : x.shape[2] // 2]

    def prompts(self, wavs, sampling_rate=None):
        """Recordings -> their prompt tokens, one int64 array each, ready for Text2Semantic.decode(prompts=...).  wavs: a list of
        1-D float recordings at `sampling_rate` Hz (None: 16 kHz), resampled to 16 kHz on the GPU (Engine.resample) when
        another rate is given.  As inference_cli.py:180-192: a recording of fewer than 48000 or more than 320000 samples at
        16 kHz is refused, then int(0.3 * the s2 config's sampling_rate) zeros are appended.  One engine call per batch."""
        wavs = [np.asarray(w, np.float32).reshape(-1) for w in wavs]
        if not wavs:
            return []
        if sampling_rate is not None and int(sampling_rate) != 16000:
            wavs = self.engine.resample(wavs, int(sampling_rate), 16000)
        for w in wavs:
            if w.size > _config.SOVITS_PROMPT_MAX or w.size < _config.SOVITS_PROMPT_MIN:
                raise ValueError(_config.SOVITS_PROMPT_MESSAGE)
        pad = np.zeros(int(self.cfg["sovits_pad"]), np.float32)
        codes, n = self.engine.sovits_semantic([np.concatenate([w, pad]) for w in wavs])
        return [codes[b, : n[b]].copy() for b in range(len(wavs))]
