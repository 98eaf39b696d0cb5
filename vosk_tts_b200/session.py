"""`onnxruntime.InferenceSession`-shaped facade over the CUDA engine.

The reference creates `self.onnx = onnxruntime.InferenceSession(model.onnx)` (vosk_tts/model.py:46) and
calls `self.model.onnx.run(None, args)[0]` (vosk_tts/synth.py:123-126).  `VitsSession` is assignable to
`Model.onnx`: `run(None, feeds)` takes the same feeds dict (keys `input`, `input_lengths`, `scales`,
`sid`; `bert` / `phone_duration_extra` must be None, synth.py:118-119) and returns
`[float32 [B,1,1,T_wav]]` like the exported graph (onnx_export.py:65-72).
"""
import logging
import threading

import numpy as np

from . import config as _config
from . import weights as _weights
from .engine import Engine


class VitsSession:
    def __init__(self, state_dict=None, cfg=None, device=0, seed=0, packed=None, precision=0, reserve=None, voice_conversion=False):
        """state_dict: reference checkpoint `['model']` dict (weight_g/weight_v allowed) or already folded.
        packed: optional (blob, manifest) to skip packing (e.g. received through an NCCL broadcast).
        reserve: optional (max_tokens, max_frames[, batch]) -- size the workspace for such requests now (Engine.reserve).
        voice_conversion: also pack the posterior encoder enc_q (training checkpoints only) so that `convert` works."""
        self.cfg = cfg or _config.DEFAULT_CONFIG
        if precision > 0 and not _weights.tc_supported(self.cfg):
            logging.warning("model widths are not multiples of 64: the tensor-core conv path is unavailable, using the fp32 kernels")
            precision = 0
        if packed is None:
            folded = _weights.fold_weight_norm(state_dict)
            packed = _weights.pack(folded, self.cfg, posterior=voice_conversion)
        self.engine = Engine(self.cfg, packed[0], packed[1], device=device, precision=precision)
        self._lock = threading.Lock()
        self._seed = int(seed)
        self._calls = 0
        self.last_y_lengths = None
        self.last_wav_lengths = None
        if reserve:
            self.reserve(*reserve)

    def reserve(self, max_tokens=256, max_frames=1024, batch=1):
        """Workspace reservation (see Engine.reserve): later calls within these bounds never move a buffer, so the CUDA graphs
        of the length buckets stay valid."""
        with self._lock:
            return self.engine.reserve(max_tokens, max_frames, batch)

    # -- onnxruntime-compatible surface ---------------------------------------------------------
    def get_providers(self):
        return ["B200VttsExecutionProvider"]

    def run(self, output_names, feeds, noise=None):
        """feeds as built at vosk_tts/synth.py:113-120.  `noise` (extension): dict(dp=[B,2,T], z=[B,C,>=T_y] or
        callable(max_frames)) to inject the two random draws; otherwise Philox with a per-call seed."""
        for k in ("bert", "phone_duration_extra"):
            if feeds.get(k) is not None:
                raise ValueError("feed %r is not None: model_type not supported by this engine (VITS2 graph only)" % k)
        ids = np.asarray(feeds["input"])
        if ids.ndim != 2:
            raise ValueError("multistream inputs ([1,5,T]) are not supported by this engine (VITS2 graph only)")
        lengths = np.asarray(feeds["input_lengths"]).reshape(-1)
        sid = feeds.get("sid")
        sid = np.zeros(ids.shape[0], np.int64) if sid is None else np.asarray(sid).reshape(-1)
        scales = np.asarray(feeds["scales"], dtype=np.float32).reshape(3)
        with self._lock:
            self._calls += 1
            seed = (self._seed * 0x9E3779B97F4A7C15 + self._calls) & 0xFFFFFFFFFFFFFFFF
            dp = z = None
            if noise is not None:
                dp, z = noise.get("dp"), noise.get("z")
            # one fused C call when the output capacity can be bounded up front (8 frames per phoneme covers the
            # duration predictor's range in practice; a CAPACITY status falls back to an exact second phase)
            hint = None if callable(z) else int(8 * ids.shape[1] + 16)
            if z is not None and not callable(z):
                hint = min(hint, int(np.asarray(z).shape[2]))
            wav, y_len = self.engine.infer(ids, lengths, sid, scales, dp, z, seed, frames_hint=hint)
            self.last_y_lengths = y_len
            self.last_wav_lengths = y_len * self.engine.hop
        return [wav[:, None, None, :]]

    def run_stream(self, feeds, chunk_frames=64):
        """Streaming variant for ONE utterance (no onnxruntime equivalent): the text encoder, duration predictor and flow
        run once, then the decoder is run over windows of `chunk_frames` frames (with the halo the engine reports) and every
        window's samples are yielded as float32 [n] as soon as they are on the host.  Concatenated, the chunks are what
        `run` returns for the same seed.  The handle keeps the flow output between the chunk calls, so the session lock is
        held for the whole stream (released when the generator is exhausted or closed)."""
        for k in ("bert", "phone_duration_extra"):
            if feeds.get(k) is not None:
                raise ValueError("feed %r is not None: model_type not supported by this engine (VITS2 graph only)" % k)
        ids = np.asarray(feeds["input"])
        if ids.ndim != 2 or ids.shape[0] != 1:
            raise ValueError("run_stream takes one utterance ([1, T] ids)")
        sid = feeds.get("sid")
        sid = 0 if sid is None else int(np.asarray(sid).reshape(-1)[0])
        scales = np.asarray(feeds["scales"], dtype=np.float32).reshape(3)
        n = int(np.asarray(feeds["input_lengths"]).reshape(-1)[0])
        with self._lock:
            self._calls += 1
            seed = (self._seed * 0x9E3779B97F4A7C15 + self._calls) & 0xFFFFFFFFFFFFFFFF
            total = 0
            stream = self.engine.synthesize_stream(ids[:, :n], sid, scales, chunk_frames=chunk_frames, seed=seed)
            try:
                for chunk in stream:
                    total += chunk.size
                    yield chunk
            finally:
                # closing THIS generator does not finalise a generator it iterates over (the frame keeps it alive): close it
                # explicitly so that an abandoned stream (client gone) ends here and the lock below is released now
                stream.close()
            self.last_wav_lengths = np.array([total], np.int64)
            self.last_y_lengths = self.last_wav_lengths // self.engine.hop

    def convert(self, wav, src, tgt, noise=None, noise_scale=1.0):
        """Voice conversion (SynthesizerTrn.voice_conversion, models.py:1710-1718; extension, no onnxruntime equivalent):
        float32 samples [L] in [-1, 1] of speaker `src` -> float32 [hop * frames] of speaker `tgt`, frames = L // 256 for the
        reference configuration.  noise: optional eps [1, inter_channels, >= frames] of the posterior sample; otherwise
        Philox with a per-call seed.  noise_scale = 1 is the reference."""
        wav = np.ascontiguousarray(wav, dtype=np.float32).reshape(-1)
        with self._lock:
            self._calls += 1
            seed = (self._seed * 0x9E3779B97F4A7C15 + self._calls) & 0xFFFFFFFFFFFFFFFF
            out, frames = self.engine.convert(wav, int(src), int(tgt), noise_scale=noise_scale, noise=noise, seed=seed)
            self.last_y_lengths = frames
            self.last_wav_lengths = frames * self.engine.hop
        return out[0, : int(frames[0]) * self.engine.hop]

    def align(self, ids, wav, sid=0, noise=None, noise_scale=1.0):
        """Forced alignment of one utterance (the alignment of SynthesizerTrn.forward, models.py:1632-1660; extension):
        phoneme ids [T] against float32 samples [L] in [-1, 1] of speaker `sid`.  Returns (durations int32 [T], token_of_frame
        int32 [frames], score) -- frames of every token, the token of every frame, the best path's log-likelihood.  noise:
        optional eps [1, inter_channels, >= frames] of the posterior sample, otherwise Philox with a per-call seed."""
        ids = np.ascontiguousarray(ids, dtype=np.int64).reshape(1, -1)
        wav = np.ascontiguousarray(wav, dtype=np.float32).reshape(-1)
        with self._lock:
            self._calls += 1
            seed = (self._seed * 0x9E3779B97F4A7C15 + self._calls) & 0xFFFFFFFFFFFFFFFF
            dur, frames, tof, score = self.engine.align(ids, ids.shape[1], sid, wav, noise_scale=noise_scale, noise=noise, seed=seed)
            self.last_y_lengths = frames
            self.last_wav_lengths = frames * self.engine.hop
        return dur[0], tof[0, : int(frames[0])], float(score[0])

    def resample(self, wav, from_rate, to_rate):
        """One clip float32 [L] at `from_rate` Hz resampled to `to_rate` Hz on the GPU (Engine.resample; extension)."""
        with self._lock:
            return self.engine.resample(np.asarray(wav, np.float32).reshape(-1), from_rate, to_rate)[0]

    def close(self):
        self.engine.close()


class StableTTSSession:
    """`Model.onnx` of a multistream StableTTS voice: an onnxruntime-shaped facade over the graph matcha/onnx/export.py writes
    (MatchaWithVocoder: text to waveform, n_timesteps baked in, guidance 0.5 as flow_matching.py:61 fixes it), plus the
    word-piece call that Synth uses so that BERT's rows are computed and gathered on the GPU."""
    multistream = True

    def __init__(self, tts, n_timesteps=5, seed=0):
        """tts: a stabletts.StableTTS with the text encoder and a vocoder (and BERT, for models with a tokenizer)."""
        if not tts.has_text or tts.hop is None:
            raise ValueError("a multistream session needs the StableTTS text encoder and a vocoder")
        self.tts = tts
        self.n_timesteps = int(n_timesteps)
        self.cfg = {"sampling_rate": 22050, "hop_length": int(tts.hop)}
        self._lock = threading.Lock()
        self._seed = int(seed)
        self._calls = 0
        self.last_wav_lengths = None

    def get_providers(self):
        return ["B200VttsExecutionProvider"]

    def _next_seed(self):
        self._calls += 1
        return (self._seed * 0x9E3779B97F4A7C15 + self._calls) & 0xFFFFFFFFFFFFFFFF

    @staticmethod
    def _feeds(feeds):
        ids = np.asarray(feeds["input"], np.int64)
        if ids.ndim != 3:
            raise ValueError("input must be the multistream ids [B, n_streams, T]")
        B = ids.shape[0]
        lengths = np.asarray(feeds["input_lengths"], np.int64).reshape(-1)
        if lengths.shape != (B,) or (lengths < 1).any() or (lengths > ids.shape[2]).any():
            raise ValueError("input_lengths must hold one length in [1, T] per utterance")
        sid = feeds.get("sid")
        sid = np.zeros(B, np.int64) if sid is None else np.broadcast_to(np.asarray(sid, np.int64).reshape(-1), (B,))
        extra = feeds.get("phone_duration_extra")
        if extra is not None:
            extra = np.broadcast_to(np.asarray(extra, np.float32).reshape(-1, ids.shape[2]), (B, ids.shape[2]))
        scales = np.asarray(feeds["scales"], np.float32).reshape(3)
        return ids, lengths, sid, extra, scales

    def _synthesise(self, ids, lengths, sid, extra, scales, **kw):
        xs = [ids[b, :, :lengths[b]] for b in range(ids.shape[0])]
        pause = None if extra is None else [extra[b, :lengths[b]] for b in range(ids.shape[0])]
        with self._lock:
            r = self.tts.synthesise(xs, kw.pop("bert", None), list(sid), phone_duration_extra=pause, n_timesteps=self.n_timesteps, guidance_scale=0.5,
                                    seed=self._next_seed(), return_wav=True, **kw, **self.tts.from_scales(scales))
        wl = np.array(r["wav_lengths"], np.int64)
        wav = np.zeros((len(xs), int(wl.max())), np.float32)
        for b, w in enumerate(r["wav"]):
            wav[b, :w.size] = w
        self.last_wav_lengths = wl
        return [wav, wl]

    def run(self, output_names, feeds):
        """feeds of export.py's graph: input int64 [B, n_streams, T], input_lengths [B], scales [temperature, length_scale,
        dp_temperature], sid [B] or None, bert float [B, bert_dim, T], phone_duration_extra [B, T] or None.  Returns [wav float32
        [B, max samples] (zeros after each utterance), wav_lengths int64 [B] = hop * mel_lengths]."""
        ids, lengths, sid, extra, scales = self._feeds(feeds)
        bert = np.asarray(feeds["bert"], np.float32)
        if bert.ndim != 3 or bert.shape[0] != ids.shape[0] or bert.shape[2] != ids.shape[2]:
            raise ValueError("bert must be [B, bert_dim, T]")
        return self._synthesise(ids, lengths, sid, extra, scales, bert=[bert[b, :, :lengths[b]] for b in range(ids.shape[0])])

    def run_pieces(self, feeds, pieces, bert_rows):
        """run() with the `bert` feed replaced by each utterance's word pieces (a list of int sequences, [CLS] ... [SEP]) and
        bert_rows int [B, T], the row among its own pieces that each token reads: BERT runs and its rows are gathered on the
        GPU (vtts_stabletts_synthesise_pieces_wav)."""
        ids, lengths, sid, extra, scales = self._feeds(feeds)
        rows = np.asarray(bert_rows, np.int64)
        if rows.ndim != 2 or rows.shape != (ids.shape[0], ids.shape[2]) or len(pieces) != ids.shape[0]:
            raise ValueError("bert_rows must be [B, T] and pieces hold one sentence per utterance")
        return self._synthesise(ids, lengths, sid, extra, scales, pieces=list(pieces),
                                bert_rows=[rows[b, :lengths[b]] for b in range(ids.shape[0])])

    def bert_features(self, ids):
        """BERT's rows [L, hidden] of one sentence's word pieces, as the reference's bert/model.onnx returns them."""
        with self._lock:
            return self.tts.bert_features(np.asarray(ids, np.int64).reshape(-1))

    def close(self):
        self.tts.close()
