"""Writes tests/golden/stabletts_tiny_graph.pb.gz and tests/golden/ref_stabletts_onnx.npz: a small multi-speaker MatchaTTS with a
small HiFi-GAN, exported as a multistream model's model.onnx is (matcha/onnx/export.py: get_exportable_module's MatchaWithVocoder,
opset 17, constant folding, N_TIMESTEPS unrolled steps), and what the *unmodified* reference synthesise + vocoder give for a
few ragged inputs.  Needs the reference tree (ref_harness.REF_ROOT); the tests read only the fixture.

The reference hard-codes the widths of its text encoder stacks (text_encoder.py:72-92) and of the flow-matching estimator
(flow_matching.py:301); at those widths the graph would be about 180 MB.  The fixture is kept to a few MB by building both
through wrappers that override the hard-coded keyword arguments (TINY_ENC / TINY_DEC) before calling the reference classes;
the modules themselves are the reference's.  The text encoder's hidden width stays 256, which fake_content (matcha_tts.py:77)
fixes.  export.py's MatchaWithVocoder calls vocoder.decode, which the reference HiFi-GAN Generator does not define: the
Generator instance gets decode = forward.  Lightning's LightningModule.to_onnx is torch.onnx.export of the module under no_grad
(the stub LightningModule of make_golden_stabletts provides it), the legacy TorchScript exporter as the reference's torch
used; the onnx package is absent, so the post-processing step that attaches onnxscript functions (there are none) is
bypassed as oracle/ref_harness.py does.

The weights are not stored: they are seeded (tests/stabletts_onnx_inputs.py), and this script checks that the reference
modules hold exactly those tensors.  The HiFi-GAN is loaded from the seeded checkpoint and its weight norm removed as cli.py
does; then its conv weights are set to the seeded weight_v tensors themselves, so that what the graph holds follows from the
seed without depending on the rounding of a norm.  The graph is stored without the bytes of the seeded initializers
(stabletts_tiny_graph.pb.gz, their raw_data emptied in place), with the name of each one's source tensor and the SHA-1 of the
exported file; stabletts_onnx_inputs.graph_bytes rebuilds that file, and this script checks it does.  Also stored: the
configs, the FiLM rows [steps][n_layers][2 hidden] (gamma | beta) and the unconditional branch's adaLN rows
[n_layers][6 hidden] torch computes for the exported steps, and per utterance the inputs (ids, bert, pause, sid), the noise
the decoder draws (its first ceil4(frames) columns), w_round, mel and the vocoder's clamped wav."""
import contextlib
import functools
import gzip
import hashlib
import io
import json
import os
import sys
import tempfile
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import make_golden_hifigan as hifigan_maker  # noqa: E402
from oracle import make_golden_stabletts as st_maker  # noqa: E402
import stabletts_onnx_inputs as SI  # noqa: E402
from vosk_tts_b200 import onnx_weights, synthetic  # noqa: E402
from vosk_tts_b200.onnx_weights import read_graph  # noqa: E402

SEED, N_TIMESTEPS, CFG, VOCODER = SI.SEED, SI.N_TIMESTEPS, SI.CFG, SI.VOCODER
TINY_ENC = {"filter_channels": 64, "n_layers": 1}
TINY_DEC = {"hidden_channels": 64, "filter_channels": 64, "n_layers": 2, "n_heads": 2}
# (token count, speaker, pauses {token: frames}) of the utterances; synthesised alone and as one ragged batch in the tests
UTTERANCES = [(9, 0, {}), (23, 2, {4: 3.0}), (1, 1, {}), (14, 1, {0: 2.0, 13: 4.0})]
TEMPERATURE, LENGTH_SCALE = 0.8, 1.1
MAX_FRAMES = 512
config = SI.config


def model_state_dict():
    return synthetic.make_random_stabletts(config(), SEED)


def vocoder_checkpoint():
    return synthetic.make_random_hifigan(SEED, VOCODER)


def utterance_inputs(i, cfg=None):
    """ids [streams, T] int64, bert [768, T], pause [T] and noise [noise_channels, MAX_FRAMES] of utterance i."""
    cfg = cfg or config()
    T, _, pauses = UTTERANCES[i]
    g = torch.Generator().manual_seed(SEED * 100 + i)
    ids = torch.randint(0, int(cfg["n_vocab"]), (int(cfg["n_streams"]), T), generator=g).numpy()
    bert = torch.randn(int(cfg["bert_dim"]), T, generator=g).numpy()
    noise = torch.randn(int(cfg["noise_channels"]), MAX_FRAMES, generator=g).numpy()
    pause = np.zeros(T, np.float32)
    for k, v in pauses.items():
        pause[k] = v
    return ids, bert, pause, noise


def _shrink(mod, name, overrides):
    cls = getattr(mod, name)
    setattr(mod, name, functools.partial(lambda cls, **kw: cls(**dict(kw, **overrides)), cls))


def build_models():
    mt = st_maker.import_reference_matcha()
    from matcha.models.components import flow_matching, text_encoder
    _shrink(text_encoder, "Encoder", TINY_ENC)
    _shrink(flow_matching, "Decoder", TINY_DEC)
    cfg, sd = config(), model_state_dict()
    matcha = st_maker.build_reference(mt, cfg, sd)
    models, hconfig, env = hifigan_maker.import_reference_hifigan()
    h = dict(hconfig.v1, **VOCODER)
    gen = models.Generator(env.AttrDict(h))
    ck = vocoder_checkpoint()
    gen.load_state_dict(ck)
    with contextlib.redirect_stdout(io.StringIO()):
        gen.remove_weight_norm()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in SI.vocoder_state_dict().items()})
    gen.eval()
    gen.decode = gen.forward
    for k, v in sd.items():
        assert torch.equal(matcha.state_dict()[k], v), k
    return matcha, gen, cfg, sd


def import_export():
    """matcha/onnx/export.py as it is; the matcha.cli it imports (argument parsing, vocoder downloads) is stubbed."""
    if "matcha.cli" not in sys.modules:
        cli = types.ModuleType("matcha.cli")
        cli.VOCODER_URLS, cli.load_matcha, cli.load_vocoder = {}, None, None
        sys.modules["matcha.cli"] = cli
    import lightning

    @torch.no_grad()
    def to_onnx(self, file_path, input_sample, **kw):
        torch.onnx.export(self, input_sample, file_path, dynamo=False, **kw)
    lightning.LightningModule.to_onnx = to_onnx
    root = os.path.join(st_maker.cfm_maker.ref_harness.REF_ROOT, "training", "stabletts")
    if "matcha.onnx" not in sys.modules:
        m = types.ModuleType("matcha.onnx")
        m.__path__ = [os.path.join(root, "matcha", "onnx")]
        sys.modules["matcha.onnx"] = m
    import importlib
    return importlib.import_module("matcha.onnx.export")


def export(matcha, gen, path):
    ex = import_export()
    from torch.onnx._internal.torchscript_exporter import onnx_proto_utils
    model, output_names = ex.get_exportable_module(matcha, gen, N_TIMESTEPS)
    dummy, input_names = ex.get_inputs(True)
    dynamic_axes = {"input": {0: "batch_size", 2: "time"}, "input_lengths": {0: "batch_size"}, "bert": {0: "batch_size", 2: "time"},
                    "phone_duration_extra": {0: "batch_size", 1: "time"}, "wav": {0: "batch_size", 1: "time"},
                    "wav_lengths": {0: "batch_size"}, "sid": {0: "batch_size"}}
    orig = onnx_proto_utils._add_onnxscript_fn
    onnx_proto_utils._add_onnxscript_fn = lambda proto, custom_opsets: proto
    try:
        with warnings.catch_warnings(), contextlib.redirect_stdout(io.StringIO()):
            warnings.simplefilter("ignore")
            model.to_onnx(path, dummy, input_names=input_names, output_names=output_names, dynamic_axes=dynamic_axes,
                          opset_version=ex.DEFAULT_OPSET, export_params=True, do_constant_folding=True)
    finally:
        onnx_proto_utils._add_onnxscript_fn = orig
    del matcha.forward                 # get_exportable_module monkey-patched it onto the instance


def baked_rows(matcha, n):
    """What the exported graph folds: the FiLM rows of every step ((gamma | beta) of each block, decoder.py:35-62,103-120,
    at t_span of flow_matching.py:53-54 advanced as solve_euler advances t) and the unconditional branch's adaLN rows
    (fake_speaker through each block's adaLN_modulation)."""
    est = matcha.decoder.estimator
    t_span = 1 - torch.cos(torch.linspace(0, 1, n + 1) * 0.5 * torch.pi)
    t, dt = t_span[0], t_span[1] - t_span[0]
    film, ada = [], []
    with torch.no_grad():
        for s in range(n):
            te = est.time_mlp(est.time_embeddings(t))
            film.append(torch.stack([b.time_fusion.film(te.unsqueeze(2))[0, :, 0] for b in est.blocks]))
            t = t + dt
            if s + 1 < n:
                dt = t_span[s + 2] - t
        for b in est.blocks:
            ada.append(b.block.adaLN_modulation(matcha.fake_speaker)[0])
    return torch.stack(film).numpy(), torch.stack(ada).numpy()


def main():
    matcha, gen, cfg, sd = build_models()
    film, ada = baked_rows(matcha, N_TIMESTEPS)
    out = {"seed": np.int64(SEED), "n_timesteps": np.int64(N_TIMESTEPS), "config": np.array(json.dumps(CFG)),
           "vocoder_config": np.array(json.dumps(VOCODER)), "film": film, "ada_uncond": ada,
           "temperature": np.float32(TEMPERATURE), "length_scale": np.float32(LENGTH_SCALE)}
    for i, (T, sid, pauses) in enumerate(UTTERANCES):
        ids, bert, pause, noise = utterance_inputs(i, cfg)
        r = st_maker.reference_synthesise(matcha, ids, bert, pause if pauses else None, noise, sid, N_TIMESTEPS, TEMPERATURE,
                                          LENGTH_SCALE)
        with torch.no_grad():
            wav = gen.decode(torch.from_numpy(r["mel"])[None]).clamp(-1, 1)[0, 0].numpy()
        frames = int(r["mel_lengths"][0])
        assert wav.shape == (256 * frames,)
        k = "u%d." % i
        out[k + "ids"], out[k + "bert"], out[k + "pause"], out[k + "sid"] = ids, bert, pause, np.int64(sid)
        out[k + "noise"] = r["noise"]
        out[k + "w_round"], out[k + "mel"], out[k + "wav"] = r["w_round"], r["mel"], wav
        print("utterance", i, "tokens", T, "frames", frames, "max |wav|", float(np.abs(wav).max()))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.onnx")
        export(matcha, gen, path)
        with open(path, "rb") as f:
            data = f.read()
        out["graph_sources"], skeleton = skeleton_of(data, read_graph(path)[0])
    out["graph_sha1"] = np.array(hashlib.sha1(data).hexdigest())
    with open(SI.SKELETON, "wb") as f:
        f.write(gzip.compress(skeleton, 9, mtime=0))
    np.savez_compressed(SI.FIXTURE, **out)
    assert SI.graph_bytes(np.load(SI.FIXTURE)) == data
    for p in (SI.SKELETON, SI.FIXTURE):
        print("wrote", p, os.path.getsize(p), "bytes (the exported graph: %d)" % len(data))


def skeleton_of(data, inits):
    """The exported file with the raw_data of every initializer that is a seeded tensor (or its transpose) emptied, and the
    JSON {initializer: [source tensor, transposed]}."""
    src = {"matcha." + k: v for k, v in SI.model_state_dict().items()}
    src.update({"vocoder." + k: v for k, v in SI.vocoder_state_dict().items()})
    sources = {}
    for name, a in inits.items():
        if name in src and np.array_equal(a, src[name]):
            sources[name] = [name, False]
        elif name.startswith("onnx::") and a.ndim == 2:
            hit = [k for k, v in src.items() if v.ndim == 2 and v.T.shape == a.shape and np.array_equal(v.T, a)]
            if hit:
                sources[name] = [hit[0], True]
    assert any(v[1] for v in sources.values())            # encoder.bert_proj.1's MatMul operand

    def tensor(buf):
        name = next(bytes(v).decode() for fno, wt, v in onnx_weights._fields(buf) if fno == 8)
        return SI._message(buf, lambda fno, v: b"" if fno == 9 and name in sources else None)
    graph = lambda buf: SI._message(buf, lambda fno, v: tensor(v) if fno == 5 else None)
    return np.array(json.dumps(sources, sort_keys=True)), SI._message(memoryview(data), lambda fno, v: graph(v) if fno == 7 else None)


if __name__ == "__main__":
    main()
