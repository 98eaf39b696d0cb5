"""GPT-SoVITS text-to-semantic decoding on the GPU: the reference's Text2SemanticDecoder.infer_panel
(training/gpt-sovits/ar/models/t2s_model.py:324-448) behind its own signature, and a ragged batch of sentences in one call."""
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
