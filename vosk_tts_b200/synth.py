"""`vosk_tts.Synth`-compatible front end (vosk_tts/synth.py:11-150) over the CUDA engine.

`synth_audio` / `synth` keep the reference signatures, defaults (config["inference"], synth.py:49-56), the
float->int16 conversion (:16-23), the RTF log line (:133-139) and the 22 050 Hz mono 16-bit WAV (:146-150).  Only the
VITS branch of the model_type dispatch (`g2p_noembed`, :100-103, :223-255) exists here; the other branches feed
graphs this engine does not implement and raise.
"""
import logging
import re
import time
import wave

import numpy as np

from .g2p import convert
from .wav import read_pcm16

_PUNCT = "([,.?!;:\"() ])"


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

    def synth_audio(self, text, speaker_id=0, noise_level=None, speech_rate=None, duration_noise_level=None, scale=None):
        inf = self.model.config.get("inference", {})
        noise_level = inf.get("noise_level", 0.8) if noise_level is None else noise_level
        speech_rate = inf.get("speech_rate", 1.0) if speech_rate is None else speech_rate
        duration_noise_level = inf.get("duration_noise_level", 0.8) if duration_noise_level is None else duration_noise_level
        scale = inf.get("scale", 1.0) if scale is None else scale
        if self.model.tokenizer is not None or str(self.model.config.get("model_type", "")).startswith("multistream"):
            raise ValueError("model_type %r is not a VITS2 graph: not supported by this engine" % self.model.config.get("model_type"))
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
        if self.model.tokenizer is not None or str(self.model.config.get("model_type", "")).startswith("multistream"):
            raise ValueError("model_type %r is not a VITS2 graph: not supported by this engine" % self.model.config.get("model_type"))
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
        if self.model.tokenizer is not None or str(self.model.config.get("model_type", "")).startswith("multistream"):
            raise ValueError("model_type %r is not a VITS2 graph: not supported by this engine" % self.model.config.get("model_type"))
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
