"""`vosk_tts.Model`-compatible loader (vosk_tts/model.py:33-63) whose `.onnx` attribute is the CUDA engine session.

Same constructor and attributes (`onnx`, `dic`, `config`, `tokenizer`); the model directory holds what the reference
ships (`config.json`, `dictionary`) plus the checkpoint the ONNX graph was exported from (`G_*.pth` / `model.pth`,
training/vits2/onnx_export.py:55) and, optionally, the training json (`vits_config.json`) when `config.json` has no
`model` block.  A directory that holds only what vosk-tts ships (`model.onnx`, `config.json`, `dictionary`) works too: the
weights AND the architecture are read from the graph's initializers (`onnx_weights.py`, no `onnx` package needed).
Downloading models needs a network and is out of scope -- a missing model is an error, never a silent fallback.

A multistream StableTTS voice (`model_type` multistream_v1 / v2 / v3) holds what the reference ships (`config.json`,
`dictionary`, and `bert/vocab.txt` with BERT's `bert/model.onnx` for the models with a tokenizer) plus the checkpoints that
matcha/onnx/export.py reads: the Matcha checkpoint (`model.ckpt`, else the newest `*.ckpt`) and the HiFi-GAN generator
(`generator_v1`, `hifigan_T2_v1` or `hifigan_univ_v1`, config v1).  Without those, the exported `model.onnx` the reference
loads (matcha/onnx/export.py's graph, vocoder included) is read instead (onnx_weights.stabletts_from_onnx).  Its `.onnx` is a
StableTTSSession.
"""
import glob
import json
import logging
import os
import re
from pathlib import Path

from . import config as _config
from . import weights as _weights
from .session import StableTTSSession, VitsSession
from .wordpiece import BertWordPieceTokenizer

MULTISTREAM_TYPES = ("multistream_v1", "multistream_v2", "multistream_v3")
VOCODER_NAMES = ("generator_v1", "hifigan_T2_v1", "hifigan_univ_v1")      # matcha/cli.py's vocoders

MODEL_DIRS = [os.getenv("VOSK_MODEL_PATH"), Path("/usr/share/vosk"), Path.home() / "AppData/Local/vosk",
              Path.home() / ".cache/vosk"]


def list_models():
    raise RuntimeError("model listing needs network access to alphacephei.com; not available in this build")


def list_languages():
    raise RuntimeError("language listing needs network access to alphacephei.com; not available in this build")


def load_dictionary(path):
    """word -> phones, keeping the most probable pronunciation (vosk_tts/model.py:48-55)."""
    dic, probs = {}, {}
    with open(path, encoding="utf-8") as f:
        for line in f:
            items = line.split(maxsplit=2)
            if len(items) < 3:
                continue
            prob = float(items[1])
            if probs.get(items[0], 0) < prob:
                dic[items[0]] = items[2].strip()
                probs[items[0]] = prob
    return dic


def _reserve_from_env():
    """VTTS_RESERVE="tokens,frames[,batch]" (default "256,1024"; "0" = off): workspace reservation at load time, so that the
    first long sentence does not move buffers and invalidate the CUDA graphs captured for the short ones."""
    v = os.environ.get("VTTS_RESERVE", "256,1024")
    if v.strip() in ("", "0"):
        return None
    return tuple(int(x) for x in v.split(","))


class Model:
    def __init__(self, model_path=None, model_name=None, lang=None, device=0, precision=1, session=None, voice_conversion=False,
                 n_timesteps=None):
        """voice_conversion: also load the posterior encoder (Synth.convert_audio); needs the training checkpoint (G_*.pth)
        -- model.onnx is a trace of SynthesizerTrn.infer and holds no enc_q.  n_timesteps: the flow-matching steps of a
        multistream voice.  A checkpoint does not record them: None means export.py's default, 5.  An exported model.onnx
        unrolls its own count: None means that count, and any other is refused."""
        if model_path is None:
            model_path = self.get_model_path(model_name, lang)
        model_path = Path(model_path)
        logging.info(f"Loading model from {model_path}")
        self.config = json.load(open(model_path / "config.json"))
        self.dic = load_dictionary(model_path / "dictionary") if (model_path / "dictionary").exists() else {}
        self.tokenizer = None
        model_type = str(self.config.get("model_type", ""))
        if model_type in MULTISTREAM_TYPES:
            self._load_multistream(model_path, device, precision, session, n_timesteps)
            return
        if (model_path / "bert" / "vocab.txt").exists() or model_type.startswith("multistream"):
            raise ValueError("bert-conditioned / multistream models are not VITS2 graphs: not supported by this engine")
        if session is not None:
            self.onnx = session
            return
        cks = sorted(glob.glob(str(model_path / "G_*.pth")), key=lambda p: int(re.sub(r"\D", "", os.path.basename(p)) or 0))
        if (model_path / "model.pth").exists():
            cks.append(str(model_path / "model.pth"))
        if (model_path / "model.onnx").exists() and not (voice_conversion and cks):
            if voice_conversion:
                raise ValueError("voice conversion needs the training checkpoint (G_*.pth / model.pth) and its training json: "
                                 "%s holds model.onnx, a trace of SynthesizerTrn.infer without the posterior encoder enc_q" % model_path)
            # the deployed layout (vosk_tts/model.py:46): everything comes out of the graph.  Preferred over a checkpoint
            # lying next to it: model.onnx is what the reference itself would load, and it is not a pickle
            from . import onnx_weights as _onnx
            sr = int(self.config.get("audio", {}).get("sample_rate", 22050))
            cfg = _onnx.config_from_onnx(str(model_path / "model.onnx"), sampling_rate=sr)
            folded = _onnx.state_dict_from_onnx(str(model_path / "model.onnx"))
            self.onnx = VitsSession(state_dict=folded, cfg=cfg, device=device, precision=precision, reserve=_reserve_from_env())
            return
        if "model" in self.config and "data" in self.config:
            n_vocab = len(self.config.get("phoneme_id_map", {})) or 62
            cfg = _config.from_training_json(self.config, n_vocab=n_vocab)
        elif (model_path / "vits_config.json").exists():
            n_vocab = len(self.config.get("phoneme_id_map", {})) or 62
            cfg = _config.from_training_json(str(model_path / "vits_config.json"), n_vocab=n_vocab)
        else:
            cfg = _config.DEFAULT_CONFIG
        if not cks:
            raise FileNotFoundError("no weights in %s: expected model.onnx (deployed layout) or G_*.pth / model.pth" % model_path)
        folded = _weights.load_checkpoint(cks[-1])
        self.onnx = VitsSession(state_dict=folded, cfg=cfg, device=device, precision=precision, reserve=_reserve_from_env(),
                                voice_conversion=voice_conversion)

    def _load_multistream(self, model_path, device, precision, session, n_timesteps):
        has_bert = (model_path / "bert" / "vocab.txt").exists()
        if has_bert:
            self.tokenizer = BertWordPieceTokenizer(vocab=str(model_path / "bert" / "vocab.txt"), unk_token="[UNK]", lowercase=True)
        if session is not None:
            if not getattr(session, "multistream", False):
                raise ValueError("a multistream model needs a multistream session (StableTTSSession), not %s" % type(session).__name__)
            self.onnx = session
            return
        ckpt = model_path / "model.ckpt"
        if not ckpt.exists():
            cks = sorted(model_path.glob("*.ckpt"), key=lambda p: p.stat().st_mtime)
            ckpt = cks[-1] if cks else None
        voc = next((model_path / n for n in VOCODER_NAMES if (model_path / n).exists()), None)
        from .stabletts import StableTTS
        if ckpt is None or voc is None:
            if (model_path / "model.onnx").exists():
                # the deployed layout (vosk_tts/model.py:46): weights, shapes and the step count come out of the graph
                tts = StableTTS.from_onnx(str(model_path / "model.onnx"), device=device, precision=precision,
                                          bert=str(model_path / "bert") if has_bert else None)
                if n_timesteps is not None and int(n_timesteps) != tts.n_timesteps:
                    tts.close()
                    raise ValueError("%s unrolls %d flow-matching steps; n_timesteps=%d would not compute what the graph computes"
                                     % (model_path / "model.onnx", tts.n_timesteps, int(n_timesteps)))
                self.onnx = StableTTSSession(tts, n_timesteps=tts.n_timesteps)
                return
            raise FileNotFoundError("no weights in %s: a multistream model needs the Matcha checkpoint (model.ckpt or *.ckpt) and "
                                    "the HiFi-GAN generator (%s)" % (model_path, " / ".join(VOCODER_NAMES)))
        sd = _weights.load_lightning_state_dict(str(ckpt))
        if "spk_emb.weight" not in sd:
            raise ValueError("%s has no spk_emb: a single-speaker Matcha checkpoint (n_spks = 1) is not supported by this engine, "
                             "whose StableTTS encoder and decoder are conditioned on a speaker embedding" % ckpt)
        n_spks, spk_dim = (int(v) for v in sd["spk_emb.weight"].shape)
        bert = _weights.load_bert(str(model_path / "bert")) if has_bert else None
        tts = StableTTS({"n_spks": n_spks, "spk_emb_dim": spk_dim}, sd, device=device, precision=precision, vocoder=str(voc), bert=bert)
        self.onnx = StableTTSSession(tts, n_timesteps=5 if n_timesteps is None else n_timesteps)

    def get_model_path(self, model_name, lang):
        for directory in MODEL_DIRS:
            if directory is None or not Path(directory).exists():
                continue
            for entry in os.listdir(directory):
                if (model_name is not None and entry == model_name) or \
                        (model_name is None and lang and re.match(r"vosk-model(-small)?-{}".format(lang), entry)):
                    return Path(directory, entry)
        raise FileNotFoundError("model %r (lang %r) not found in %s and cannot be downloaded (no network)"
                                % (model_name, lang, [str(d) for d in MODEL_DIRS if d]))
