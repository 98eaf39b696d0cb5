"""StableTTS on the GPU, as far as it is built: text-to-mel (MatchaTTS.synthesise of training/stabletts/matcha/models/
matcha_tts.py:93-211: multistream ids, BERT features and pause durations in, durations and mel out) and its
conditional-flow-matching decoder alone (CFM.forward of components/flow_matching.py, called at matcha_tts.py:183), and, with a
HiFi-GAN checkpoint (matcha/hifigan, as cli.py:65-71 loads it), the vocoder: mel to waveform, and text to waveform in one call.
With a BERT checkpoint (the model vosk_tts/synth.py's get_word_bert runs) the engine also computes BERT's features of word-piece
ids on the GPU (bert_features), and synthesise takes either the features per token, as the exported graph's `bert` feed does,
or each sentence's word pieces and the row each token reads, gathering BERT's rows on the device."""
import numpy as np

from . import config as _config
from . import weights as _weights


class StableTTS:
    """A MatchaTTS (StableTTS) checkpoint on one GPU: text-to-mel when it carries the text encoder, else the flow-matching
    decoder alone."""

    def __init__(self, config, checkpoint, device=0, precision=1, vocoder=None, vocoder_config=None, bert=None):
        """config: overrides of config.STABLETTS_CFM / STABLETTS_TEXT (n_vocab, n_spks, spk_emb_dim, ...) or None; checkpoint: a
        path (Lightning's `state_dict` entry is taken when present) or a state dict.  A state dict without encoder.* serves
        refine() only.  vocoder: a HiFi-GAN checkpoint path (weights.load_hifigan) or its folded `generator` state dict, or None;
        vocoder_config: the reference's config-dict keys (config.hifigan_config; None: v1).  bert: bert-export.py's graph (a multistream
        model's bert/ directory or its model.onnx) or a Hugging Face BERT checkpoint directory (weights.load_bert), or a
        (BertModel state dict, config.bert_config) pair, or None."""
        from .engine import Engine
        sd = _weights.load_checkpoint(checkpoint) if isinstance(checkpoint, str) else checkpoint
        sd = sd.get("state_dict", sd)
        self.has_text = "encoder.emb.weight" in sd
        voc = None
        if vocoder is not None:
            vsd = _weights.load_hifigan(vocoder) if isinstance(vocoder, str) else _weights.fold_weight_norm(vocoder)
            voc = (vsd, _config.hifigan_config(vocoder_config))
        bt = None
        if bert is not None:
            bsd, bcfg = _weights.load_bert(bert) if isinstance(bert, str) else bert
            bt = (bsd, bcfg, precision != 0)
        if self.has_text:
            self.cfg = _config.stabletts_config(dict({"n_vocab": int(sd["encoder.emb.weight"].shape[0])}, **(config or {})))
            blob, man = _weights.pack_stabletts(sd, self.cfg, vocoder=voc, bert=bt, precision=precision)
        else:
            self.cfg = _config.stabletts_cfm_config(config)
            blob, man = _weights.pack_stabletts_cfm(sd, self.cfg, vocoder=voc, bert=bt, precision=precision)
        if bt is not None:
            self.cfg["bert"] = bt[1]
        if voc is not None:
            if int(voc[1]["num_mels"]) != int(self.cfg["noise_channels"]):
                raise ValueError("the vocoder reads %d mel channels, the model makes %d" % (int(voc[1]["num_mels"]), int(self.cfg["noise_channels"])))
            self.cfg["vocoder"] = voc[1]
        self.hop = _config.hop_samples(voc[1]) if voc is not None else None
        self.mel_mean, self.mel_std = np.float32(sd["mel_mean"]), np.float32(sd["mel_std"])
        self.engine = Engine(self.cfg, blob, man, device=device, precision=precision)

    @classmethod
    def from_onnx(cls, path, device=0, precision=1, bert=None):
        """A multistream voice's model.onnx (matcha/onnx/export.py's graph, read by onnx_weights.stabletts_from_onnx) on one GPU,
        with its vocoder; bert as in __init__.  n_timesteps: the Euler steps the graph unrolls, which StableTTSSession runs.
        The graph carries no mel encoder, so synthesise(..., return_prior=True) is refused."""
        from . import onnx_weights
        g = onnx_weights.stabletts_from_onnx(path)
        tts = cls(g["config"], g["state_dict"], device=device, precision=precision, vocoder=g["vocoder"],
                  vocoder_config=g["vocoder_config"], bert=bert)
        tts.n_timesteps = g["n_timesteps"]
        return tts

    @staticmethod
    def from_scales(scales):
        """The exported graph's `scales` feed in the order its forward reads it (matcha/onnx/export.py:47-49): [temperature,
        length_scale, dp_temperature] -> keyword arguments of synthesise.  dp_temperature is not used by the deterministic
        duration predictor."""
        return {"temperature": float(scales[0]), "length_scale": float(scales[1])}

    def synthesise(self, x, bert, sid, phone_duration_extra=None, n_timesteps=10, temperature=1.0, length_scale=1.0,
                   guidance_scale=0.5, noise=None, seed=0, return_prior=False, return_wav=False, pieces=None, bert_rows=None):
        """x: the ids [n_streams, T] of one utterance, or a list of them; bert [bert_dim, T] and phone_duration_extra [T] (or
        None) alike; sid: a speaker id for all, or one per utterance; noise: [noise_channels, >= ceil4(frames)] per utterance
        standing in for torch.randn over the padded frame axis, or None for the engine's Philox(seed).  Returns the
        reference's names: mel and decoder_outputs [noise_channels, frames] (denormalised and as the model produces them),
        mel_lengths, durations [T] (w_round), with return_prior encoder_outputs / mel_enc, and with return_wav the vocoder's
        wav [hop * frames] (vocoder(mel).clamp(-1, 1), run on the device behind the mel) and wav_lengths; each a list for a list.
        pieces / bert_rows, with bert=None: the word pieces of each utterance's sentence ([CLS] ... [SEP]) and the row among them
        that each token reads [T] (an engine with BERT and a vocoder; return_wav is implied)."""
        single = not isinstance(x, (list, tuple))
        xs = [np.asarray(u, np.int64) for u in ([x] if single else x)]
        B, T = len(xs), max(u.shape[1] for u in xs)
        ids = np.zeros((B, xs[0].shape[0], T), np.int64)
        feats = rows = None
        if (bert is None) == (pieces is None) or (pieces is None) != (bert_rows is None):
            raise ValueError("give either bert, or pieces with bert_rows")
        if bert is not None:
            berts = [np.asarray(u, np.float32) for u in ([bert] if single else bert)]
            feats = np.zeros((B, T, berts[0].shape[0]), np.float32)
        if bert_rows is not None:
            rs = [np.asarray(u, np.int32).reshape(-1) for u in ([bert_rows] if single else bert_rows)]
            if len(rs) != B or any(r.size != u.shape[1] for r, u in zip(rs, xs)):
                raise ValueError("bert_rows must hold one row index per token")
            rows = np.zeros((B, T), np.int32)
            for b, r in enumerate(rs):
                rows[b, :r.size] = r
            pieces = [pieces] if single else pieces
        pause = None if phone_duration_extra is None else np.zeros((B, T), np.float32)
        for b, u in enumerate(xs):
            ids[b, :, :u.shape[1]] = u
            if feats is not None:
                if berts[b].shape[1] != u.shape[1]:
                    raise ValueError("bert must have one column per token")
                feats[b, :u.shape[1]] = berts[b].T
            if pause is not None:
                pause[b, :u.shape[1]] = np.asarray(phone_duration_extra if single else phone_duration_extra[b], np.float32).reshape(-1)
        nz = None
        if noise is not None:
            nz = [np.ascontiguousarray(np.asarray(n, np.float32).T) for n in ([noise] if single else list(noise))]
        return_wav = return_wav or rows is not None
        r = self.engine.stabletts_synthesise(ids, feats, sid, lengths=[u.shape[1] for u in xs], pause=pause, n_timesteps=n_timesteps,
                                             temperature=temperature, length_scale=length_scale, guidance_scale=guidance_scale,
                                             noise=nz, seed=seed, want_prior=return_prior, want_wav=return_wav,
                                             pieces=None if rows is None else [np.asarray(p, np.int64).reshape(-1) for p in pieces],
                                             bert_rows=rows)
        den = lambda a: a * self.mel_std + self.mel_mean          # denormalize (matcha/utils/model.py), fp32 like the reference
        cut = lambda a: [np.ascontiguousarray(a[b, :int(r["mel_lengths"][b])].T) for b in range(B)]
        out = {"decoder_outputs": cut(r["mel"]), "mel_lengths": [int(v) for v in r["mel_lengths"]],
               "durations": [r["durations"][b, :xs[b].shape[1]].copy() for b in range(B)]}
        out["mel"] = [den(m) for m in out["decoder_outputs"]]
        if return_prior:
            out["encoder_outputs"] = cut(r["prior"])
            out["mel_enc"] = [den(m) for m in out["encoder_outputs"]]
        if return_wav:
            out["wav_lengths"] = [int(v) for v in r["wav_lengths"]]
            out["wav"] = [r["wav"][b, :out["wav_lengths"][b]].copy() for b in range(B)]
        return {k: v[0] for k, v in out.items()} if single else out

    def bert_features(self, ids):
        """ids: the WordPiece ids of one sentence ([CLS] ... [SEP], as the reference's tokenizer encodes it), or a list of them.
        Returns BERT's rows [length, hidden] of each (a list for a list): bert-export.py's logits, hidden_states[-3]."""
        single = not isinstance(ids, (list, tuple)) or (len(ids) > 0 and np.isscalar(ids[0]))
        seqs = [ids] if single else list(ids)
        feats, lengths = self.engine.bert_features(seqs)
        out = [feats[b, :int(lengths[b])].copy() for b in range(len(seqs))]
        return out[0] if single else out

    def vocode(self, mel):
        """mel: the denormalised mel [num_mels, T] of one utterance (synthesise's `mel`), or a list of them.  Returns the
        waveform [hop * T] of each (a list for a list): vocoder(mel).clamp(-1, 1)."""
        single = not isinstance(mel, (list, tuple))
        rows = [np.ascontiguousarray(np.asarray(m, np.float32).T) for m in ([mel] if single else list(mel))]
        wav, wl = self.engine.hifigan_vocode(rows)
        out = [wav[b, :int(wl[b])].copy() for b in range(len(rows))]
        return out[0] if single else out

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
