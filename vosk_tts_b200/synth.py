"""`vosk_tts.Synth`-compatible front end (vosk_tts/synth.py:11-150) over the CUDA engine.

`synth_audio` / `synth` keep the reference signatures, defaults (config["inference"], synth.py:49-56), the
float->int16 conversion (:16-23), the RTF log line (:133-139) and the 22 050 Hz mono 16-bit WAV (:146-150).  The model_type
dispatch (:64-103) serves the VITS branch (`g2p_noembed`, :223-255) and the multistream StableTTS branches (`get_word_bert`,
`g2p_multistream`, `g2p_multistream_scales`, :25-44, :258-454); BERT-conditioned VITS graphs (`g2p` / `g2p_noblank`,
:88-99) are not implemented and raise.
"""
import logging
import re
import time
import wave

import numpy as np

from .g2p import convert
from .wav import read_pcm16

_PUNCT = "([,.?!;:\"() ])"
_MS_PUNCT = "(\\.\\.\\.|- |[ ,.?!;:\"()])"            # g2p_multistream (synth.py:276)
_MS_PUNCT_SCALES = "(\\.\\.\\.|- |[ ,.?!;:\"()_])"    # g2p_multistream_scales (:364): "_" is a pause mark
_BERT_PUNCT = "[-,.?!;:\"]"                           # the tokens get_word_bert drops with nopunc (:37)
_MULTISTREAM = ("multistream_v1", "multistream_v2", "multistream_v3")


class Synth:
    def __init__(self, model):
        self.model = model

    def audio_float_to_int16(self, audio, max_wav_value=32767.0):
        audio_norm = np.clip(audio * max_wav_value, -max_wav_value, max_wav_value)
        return audio_norm.astype("int16")

    def g2p_noembed(self, text):
        return self._g2p(text)[1]

    def _g2p(self, text):
        """(phonemes, ids, spans): spans[i] = (first, end) of phoneme i's ids in `ids`; the blank between phonemes i - 1
        and i is the id at spans[i][0] - 1."""
        phonemes = ["^"]
        for word in re.split(_PUNCT, text.lower()):
            if word == "":
                continue
            if re.match(_PUNCT, word) or word == "-":
                phonemes.append(word)
            elif word in self.model.dic:
                phonemes.extend(self.model.dic[word].split())
            else:
                phonemes.extend(convert(word).split())
        phonemes.append("$")
        id_map = self.model.config["phoneme_id_map"]
        ids, spans = [], []
        for i, p in enumerate(phonemes):            # intersperse the blank id 0 (synth.py:244-251)
            if i:
                ids.append(0)
            v = id_map[p]
            first = len(ids)
            ids.extend(v if isinstance(v, list) else [v])
            spans.append((first, len(ids)))
        logging.info(f"Text: {text}")
        logging.info(f"Phonemes: {phonemes}")
        return phonemes, ids, spans

    def add_pos(self, x):
        """Word-position suffixes of a word's phones (synth.py:258-270): _S alone, else _B, _I ..., _E."""
        if len(x) == 1:
            return [x[0] + "_S"]
        return [p + ("_B" if i == 0 else "_E" if i == len(x) - 1 else "_I") for i, p in enumerate(x)]

    def _word_pieces(self, text, nopunc=False):
        """The tokenizer's encoding of `text` without "+" and "_", and the indices of the tokens whose BERT rows
        get_word_bert keeps (synth.py:25-44): not "##" continuations, and with nopunc not punctuation."""
        enc = self.model.tokenizer.encode(text.replace("+", "").replace("_", ""))
        keep = [i for i, t in enumerate(enc.tokens) if t[0] != "#" and not (nopunc and re.match(_BERT_PUNCT, t))]
        return enc, keep

    def get_word_bert(self, text, nopunc=False):
        """BERT's rows [words, hidden] of the kept tokens of `text` (synth.py:25-44), BERT run on the GPU."""
        enc, keep = self._word_pieces(text, nopunc)
        return np.asarray(self.model.onnx.bert_features(enc.ids))[keep]

    def _multistream(self, text, word_pos, scales, n_rows=None):
        """The one pass behind g2p_multistream and g2p_multistream_scales (synth.py:273-454): the ids [T, 5] of every phone
        (phone, its punctuation, the in-quote flag, the last punctuation and the last sentence punctuation after it), each
        phone's word index into the kept BERT rows (0 for "^", words + 1 for the closing " " and "$") and the pause extras
        (20 where the punctuation holds "_"; scales only, where "_" is a mark of its own).  n_rows: the kept BERT rows, or
        None; a word index past them raises ValueError where the reference's bert_embeddings[...] raises IndexError, and so
        does a phone missing from phoneme_id_map (the reference's KeyError)."""
        pattern = _MS_PUNCT_SCALES if scales else _MS_PUNCT
        phonemes = [("^", [], 0, 0)]
        in_quote, cur_punc, word = 0, [], 1
        for w in re.split(pattern, text.replace(" -", "- ").lower()):
            if w == "":
                continue
            if w == "\"":
                in_quote = 1 - in_quote
            elif w == "- " or w == "-":
                cur_punc.append("-")
            elif re.match(pattern, w) and w != " ":
                cur_punc.append(w)
            elif w == " ":
                phonemes.append((" ", cur_punc, in_quote, word))
                cur_punc = []
            else:
                ph = (self.model.dic[w] if w in self.model.dic else convert(w)).split()
                phonemes.extend((p, [], in_quote, word) for p in (self.add_pos(ph) if word_pos else ph))
                cur_punc = []
                word += 1
        phonemes.append((" ", cur_punc, in_quote, word))
        phonemes.append(("$", [], 0, word))
        id_map = self.model.config["phoneme_id_map"]

        def pid(p):
            if p not in id_map:
                raise ValueError("phone %r is not in the model's phoneme_id_map" % p)
            return id_map[p]

        last_punc = last_sentence_punc = " "
        ids, rows, extra = [], [], []
        for p, punc, quote, w in reversed(phonemes):
            last_sentence_punc = next((m for m in ("...", ".", "!", "?", "-") if m in punc), last_sentence_punc)
            if punc:
                last_punc = punc[0]
            ids.append((pid(p), pid(punc[0] if punc else "_"), quote, pid(last_punc), pid(last_sentence_punc)))
            if n_rows is not None and w >= n_rows:
                raise ValueError("%r: phone %r reads BERT row %d of %d: the tokenizer splits a word that g2p keeps whole"
                                 % (text, p, w, n_rows))
            rows.append(w)
            extra.append(20.0 if "_" in punc else 0.0)
        logging.info(f"Text: {text}")
        logging.info(f"Phonemes: {[p[0] for p in phonemes]}")
        return ids[::-1], rows[::-1], extra[::-1]

    def g2p_multistream(self, text, bert_embeddings, word_pos=False):
        """(ids [T] of 5-tuples, each phone's BERT row, [] without bert_embeddings) as synth.py:273-358."""
        ids, rows, _ = self._multistream(text, word_pos, False, None if bert_embeddings is None else len(bert_embeddings))
        return ids, ([] if bert_embeddings is None else [bert_embeddings[r] for r in rows])

    def g2p_multistream_scales(self, text, bert_embeddings):
        """(ids, each phone's BERT row, pause extras) as synth.py:361-454."""
        ids, rows, extra = self._multistream(text, True, True, None if bert_embeddings is None else len(bert_embeddings))
        return ids, ([] if bert_embeddings is None else [bert_embeddings[r] for r in rows]), extra

    def _is_multistream(self):
        return self.model.config.get("model_type") in _MULTISTREAM

    def _require_vits(self):
        if self.model.tokenizer is not None or str(self.model.config.get("model_type", "")).startswith("multistream"):
            raise ValueError("model_type %r is not a VITS2 graph: not supported by this engine" % self.model.config.get("model_type"))

    def _synth_multistream(self, text, scales, speaker_id):
        """The multistream branches of synth.py:64-87 -> float samples.  With a tokenizer the session gets the word pieces
        and the row each phone reads, and BERT's rows never leave the GPU."""
        model_type, tok = self.model.config.get("model_type"), self.model.tokenizer
        if tok is None and model_type != "multistream_v2":
            raise ValueError("model_type %r needs BERT's tokenizer (bert/vocab.txt)" % model_type)
        extra = None
        if tok is None:
            ids, rows, _ = self._multistream(text, True, False)
        else:
            enc, keep = self._word_pieces(text.lower() if model_type == "multistream_v3" else text, nopunc=True)
            if model_type == "multistream_v3":
                ids, rows, extra = self._multistream(text, True, True, len(keep))
            else:
                ids, rows, _ = self._multistream(text, model_type == "multistream_v2", False, len(keep))
        T = len(ids)
        feeds = {"input": np.expand_dims(np.array(ids, dtype=np.int64).T, 0), "input_lengths": np.array([T], dtype=np.int64),
                 "scales": scales, "sid": np.array([0 if speaker_id is None else speaker_id], dtype=np.int64),
                 "phone_duration_extra": None if extra is None else np.array([extra], dtype=np.float32)}
        if tok is None:
            feeds["bert"] = np.zeros((1, 768, T), dtype=np.float32)
            return self.model.onnx.run(None, feeds)[0]
        bert_rows = np.array([[keep[r] for r in rows]], dtype=np.int32)
        return self.model.onnx.run_pieces(feeds, [np.array(enc.ids, dtype=np.int64)], bert_rows)[0]

    def synth_audio(self, text, speaker_id=0, noise_level=None, speech_rate=None, duration_noise_level=None, scale=None):
        inf = self.model.config.get("inference", {})
        noise_level = inf.get("noise_level", 0.8) if noise_level is None else noise_level
        speech_rate = inf.get("speech_rate", 1.0) if speech_rate is None else speech_rate
        duration_noise_level = inf.get("duration_noise_level", 0.8) if duration_noise_level is None else duration_noise_level
        scale = inf.get("scale", 1.0) if scale is None else scale
        if self._is_multistream():
            text = re.sub("—", "-", text.strip())
            scales = np.array([noise_level, 1.0 / speech_rate, duration_noise_level], dtype=np.float32)
            t0 = time.perf_counter()
            audio = self.audio_float_to_int16(np.asarray(self._synth_multistream(text, scales, speaker_id)).squeeze() * scale)
            infer_sec = time.perf_counter() - t0
            dur = audio.shape[-1] / 22050
            logging.info("Real-time factor: %0.2f (infer=%0.2f sec, audio=%0.2f sec)" % (infer_sec / dur if dur > 0 else 0.0, infer_sec, dur))
            return audio
        self._require_vits()
        text = re.sub("—", "-", text.strip())
        ids = self.g2p_noembed(text)
        feeds = {"input": np.expand_dims(np.array(ids, dtype=np.int64), 0),
                 "input_lengths": np.array([len(ids)], dtype=np.int64),
                 "scales": np.array([noise_level, 1.0 / speech_rate, duration_noise_level], dtype=np.float32),
                 "sid": np.array([0 if speaker_id is None else speaker_id], dtype=np.int64),
                 "bert": None, "phone_duration_extra": None}
        t0 = time.perf_counter()
        audio = self.model.onnx.run(None, feeds)[0].squeeze() * scale
        audio = self.audio_float_to_int16(audio)
        infer_sec = time.perf_counter() - t0
        dur = audio.shape[-1] / 22050
        logging.info("Real-time factor: %0.2f (infer=%0.2f sec, audio=%0.2f sec)" % (infer_sec / dur if dur > 0 else 0.0, infer_sec, dur))
        return audio

    def synth_audio_stream(self, text, speaker_id=0, noise_level=None, speech_rate=None, duration_noise_level=None, scale=None,
                           chunk_frames=64):
        """Generator of int16 chunks of the same utterance `synth_audio` would return (extension; the reference server sends one
        message with the whole utterance, server/tts_server.py:55-56): first audio after encoder + flow + one decoder window."""
        inf = self.model.config.get("inference", {})
        noise_level = inf.get("noise_level", 0.8) if noise_level is None else noise_level
        speech_rate = inf.get("speech_rate", 1.0) if speech_rate is None else speech_rate
        duration_noise_level = inf.get("duration_noise_level", 0.8) if duration_noise_level is None else duration_noise_level
        scale = inf.get("scale", 1.0) if scale is None else scale
        if self._is_multistream():     # one chunk: the whole utterance, as the reference server sends it
            yield self.synth_audio(text, speaker_id, noise_level, speech_rate, duration_noise_level, scale)
            return
        self._require_vits()
        text = re.sub("—", "-", text.strip())
        ids = self.g2p_noembed(text)
        feeds = {"input": np.expand_dims(np.array(ids, dtype=np.int64), 0),
                 "input_lengths": np.array([len(ids)], dtype=np.int64),
                 "scales": np.array([noise_level, 1.0 / speech_rate, duration_noise_level], dtype=np.float32),
                 "sid": np.array([0 if speaker_id is None else speaker_id], dtype=np.int64),
                 "bert": None, "phone_duration_extra": None}
        t0 = time.perf_counter()
        n = 0
        stream = self.model.onnx.run_stream(feeds, chunk_frames=chunk_frames)
        try:
            for chunk in stream:
                n += chunk.size
                yield self.audio_float_to_int16(chunk * scale)
        finally:
            stream.close()              # releases the session (its lock) also when the consumer abandons this generator
        infer_sec = time.perf_counter() - t0
        dur = n / 22050
        logging.info("Real-time factor: %0.2f (infer=%0.2f sec, audio=%0.2f sec)" % (infer_sec / dur if dur > 0 else 0.0, infer_sec, dur))

    def _sample_rate(self):
        cfg = getattr(self.model.onnx, "cfg", None)
        if isinstance(cfg, dict) and "sampling_rate" in cfg:
            return int(cfg["sampling_rate"])
        return int(self.model.config.get("audio", {}).get("sample_rate", self.model.config.get("data", {}).get("sampling_rate", 22050)))

    def convert_audio(self, audio, src_speaker, tgt_speaker, noise_scale=None, scale=None, sampling_rate=None):
        """Voice conversion (extension): re-voices `audio` of speaker `src_speaker` as `tgt_speaker` of the same model
        (SynthesizerTrn.voice_conversion, models.py:1710-1718).  audio: int16 samples (divided by 32768, data_utils.py:77) or
        float in [-1, 1], at the model's sample rate, or at `sampling_rate` Hz: it is then resampled to the model's rate on
        the GPU first (as librosa.load(path, sr=...) would, with resample_poly's filter).  Returns int16 [256 * (len // 256)]
        of the model-rate clip for the reference configuration."""
        self._require_vits()
        wav = self._at_model_rate(self._float_audio(audio, "convert_audio"), sampling_rate)
        if src_speaker is None or tgt_speaker is None:
            raise ValueError("voice conversion needs both a source and a target speaker id")
        inf = self.model.config.get("inference", {})
        noise_scale = 1.0 if noise_scale is None else noise_scale      # the reference samples the posterior at scale 1 (:841)
        scale = inf.get("scale", 1.0) if scale is None else scale
        t0 = time.perf_counter()
        out = self.model.onnx.convert(wav, int(src_speaker), int(tgt_speaker), noise_scale=noise_scale) * scale
        out = self.audio_float_to_int16(out)
        sec = time.perf_counter() - t0
        dur = out.shape[-1] / self._sample_rate()
        logging.info("Real-time factor: %0.2f (convert=%0.2f sec, audio=%0.2f sec)" % (sec / dur if dur > 0 else 0.0, sec, dur))
        return out

    def _at_model_rate(self, wav, sampling_rate):
        """wav at `sampling_rate` Hz (None: already at the model's rate) -> the model's rate, resampled on the GPU."""
        sr = self._sample_rate()
        if sampling_rate is None or int(sampling_rate) == sr:
            return wav
        return self.model.onnx.resample(wav, int(sampling_rate), sr)

    def _read_wav(self, iname):
        """A mono 16-bit WAV at the model's sample rate (no resampling) -> int16 samples."""
        sr = self._sample_rate()
        with wave.open(iname, "rb") as f:
            if f.getnchannels() != 1 or f.getsampwidth() != 2:
                raise ValueError("%s: expected a mono 16-bit WAV" % iname)
            if f.getframerate() != sr:
                raise ValueError("%s is sampled at %d Hz, the model at %d Hz: resample it first" % (iname, f.getframerate(), sr))
            return np.frombuffer(f.readframes(f.getnframes()), dtype="<i2").astype(np.int16)

    @staticmethod
    def _float_audio(audio, what):
        audio = np.asarray(audio)
        if audio.ndim != 1:
            raise ValueError("%s takes one mono clip ([n] samples)" % what)
        if audio.dtype == np.int16:
            return audio.astype(np.float32) / 32768.0          # data_utils.py:77
        if np.issubdtype(audio.dtype, np.floating):
            wav = audio.astype(np.float32)
            if wav.size and float(np.abs(wav).max()) > 1.0:
                raise ValueError("float audio must lie in [-1, 1]")
            return wav
        raise ValueError("audio must be int16 or float samples, not %s" % audio.dtype)

    def convert(self, iname, oname, src_speaker, tgt_speaker, noise_scale=None, scale=None, resample=False):
        """Reads a mono 16-bit WAV at the model's sample rate (no resampling), writes the converted clip as one at that rate.
        resample: read a 16-bit WAV at any rate, mono or multichannel (averaged to mono), and resample it on the GPU."""
        sr = self._sample_rate()
        if resample:
            audio, rate = read_pcm16(iname)
            out = self.convert_audio(audio, src_speaker, tgt_speaker, noise_scale, scale, sampling_rate=rate)
        else:
            out = self.convert_audio(self._read_wav(iname), src_speaker, tgt_speaker, noise_scale, scale)
        with wave.open(oname, "w") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(sr)
            f.writeframes(out.tobytes())

    def align_audio(self, text, audio, speaker_id=0, noise_scale=None, sampling_rate=None):
        """Forced alignment (extension): the phonemes of `text` (the g2p of synth_audio) against `audio` of speaker
        `speaker_id`, by the model's own monotonic alignment search (SynthesizerTrn.forward, models.py:1632-1660).  audio as
        in convert_audio (`sampling_rate`: its rate, resampled to the model's on the GPU).  Returns one dict per g2p phoneme, "^", "$" and punctuation included -- {"phoneme", "start", "end"}
        in seconds (frames * hop / sample rate) -- with each interspersed blank as its own entry with phoneme None; the
        frames of a phoneme that maps to several ids are merged, and the entries tile [0, frames * hop / sample rate).
        The best path's log-likelihood (higher: the audio fits the text better) is kept in `last_score`."""
        self._require_vits()
        wav = self._at_model_rate(self._float_audio(audio, "align_audio"), sampling_rate)
        phonemes, ids, spans = self._g2p(re.sub("—", "-", text.strip()))
        noise_scale = 1.0 if noise_scale is None else noise_scale      # the reference samples the posterior at scale 1 (:841)
        t0 = time.perf_counter()
        dur, _, score = self.model.onnx.align(np.array(ids, np.int64), wav, 0 if speaker_id is None else int(speaker_id),
                                              noise_scale=noise_scale)
        sec = time.perf_counter() - t0
        cum = np.concatenate([[0], np.cumsum(np.asarray(dur[: len(ids)], np.int64))])
        step = self._hop() / float(self._sample_rate())
        entries = []
        for i, (p, (a, e)) in enumerate(zip(phonemes, spans)):
            if i:
                entries.append({"phoneme": None, "start": float(cum[a - 1] * step), "end": float(cum[a] * step)})
            entries.append({"phoneme": p, "start": float(cum[a] * step), "end": float(cum[e] * step)})
        self.last_score = float(score)
        logging.info("Alignment: %d phonemes, %d frames, score %.1f (%.2f sec)" % (len(phonemes), int(cum[-1]), score, sec))
        return entries

    def align(self, wav_path, text, speaker_id=0, noise_scale=None, resample=False):
        """align_audio of a mono 16-bit WAV at the model's sample rate (no resampling).  resample: a 16-bit WAV at any rate,
        mono or multichannel (averaged to mono), resampled on the GPU; the segment times are those of the model-rate clip."""
        if resample:
            audio, rate = read_pcm16(wav_path)
            return self.align_audio(text, audio, speaker_id, noise_scale, sampling_rate=rate)
        return self.align_audio(text, self._read_wav(wav_path), speaker_id, noise_scale)

    def _hop(self):
        cfg = getattr(self.model.onnx, "cfg", None)
        return int(cfg.get("hop_length", 256)) if isinstance(cfg, dict) else 256

    def synth(self, text, oname, speaker_id=0, noise_level=None, speech_rate=None, duration_noise_level=None, scale=None):
        audio = self.synth_audio(text, speaker_id, noise_level, speech_rate, duration_noise_level, scale)
        with wave.open(oname, "w") as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(22050)
            f.writeframes(audio.tobytes())
