"""The exported StableTTS graph of the model.onnx tests, rebuilt from what the repository keeps of it.

oracle/make_golden_stabletts_onnx.py exports a reduced-width multi-speaker MatchaTTS with a small HiFi-GAN through the
reference's matcha/onnx/export.py.  The weights are seeded (model_state_dict, vocoder_state_dict), so the fixture keeps the
graph without their bytes: tests/golden/stabletts_tiny_graph.pb.gz is the exported ModelProto, gzipped, in which the raw_data of every
initializer drawn from the seed is empty, and ref_stabletts_onnx.npz's "graph_sources" names each such initializer's tensor
("matcha.<key>" or "vocoder.<key>", and whether the graph holds it transposed: an nn.Linear's MatMul operand).  graph_bytes()
puts the bytes back in place and checks the SHA-1 of the whole file the exporter wrote."""
import gzip
import hashlib
import json
import os

import numpy as np

from vosk_tts_b200 import config as C, onnx_weights, synthetic

SEED = 4242
N_TIMESTEPS = 3
CFG = {"n_vocab": 40, "n_spks": 3, "spk_emb_dim": 32, "enc_filter_channels": 64, "enc_n_layers": 1,
       "hidden_channels": 64, "filter_channels": 64, "n_layers": 2, "n_heads": 2}
VOCODER = {"resblock": "1", "upsample_rates": [8, 8, 4], "upsample_kernel_sizes": [16, 16, 8], "upsample_initial_channel": 128,
           "resblock_kernel_sizes": [3], "resblock_dilation_sizes": [[1, 3, 5]], "num_mels": 80}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SKELETON = os.path.join(GOLDEN, "stabletts_tiny_graph.pb.gz")
FIXTURE = os.path.join(GOLDEN, "ref_stabletts_onnx.npz")


def config():
    return C.stabletts_config(CFG)


def model_state_dict():
    """MatchaTTS's tensors, seeded by name (numpy fp32)."""
    return {k: v.numpy() for k, v in synthetic.make_random_stabletts(config(), SEED).items()}


def vocoder_state_dict():
    """The HiFi-GAN's tensors as the graph holds them, without weight norm: the seeded weight_v of each conv is its weight (the
    norm's g is left out, so that every tensor follows from the seed by one rounded product and not by a reduction)."""
    ck = synthetic.make_random_hifigan(SEED, VOCODER)
    return {k[:-len("_v")] if k.endswith(".weight_v") else k: v.numpy() for k, v in ck.items() if not k.endswith(".weight_g")}


def _key(fno, wt):
    return _varint((fno << 3) | wt)


def _varint(v):
    out = bytearray()
    while True:
        out.append((v & 0x7F) | (0x80 if v > 0x7F else 0))
        v >>= 7
        if not v:
            return bytes(out)


def _message(buf, rewrite):
    """Re-serialises one message field by field; rewrite(fno, value) returns the new bytes of a length-delimited field's
    value, or None to keep it."""
    out = bytearray()
    for fno, wt, v in onnx_weights._fields(buf):
        out += _key(fno, wt)
        if wt == 0:
            out += _varint(v)
        elif wt == 2:
            nv = rewrite(fno, v)
            nv = bytes(v) if nv is None else nv
            out += _varint(len(nv)) + nv
        else:
            out += v
    return bytes(out)


def _fill(skeleton, tensors):
    def tensor(buf):
        name = next(bytes(v).decode() for fno, wt, v in onnx_weights._fields(buf) if fno == 8)
        return _message(buf, lambda fno, v: np.ascontiguousarray(tensors[name], np.float32).tobytes()
                        if fno == 9 and len(v) == 0 and name in tensors else None)
    graph = lambda buf: _message(buf, lambda fno, v: tensor(v) if fno == 5 else None)
    return _message(memoryview(skeleton), lambda fno, v: graph(v) if fno == 7 else None)


def graph_bytes(fix=None):
    """The bytes of the exported model.onnx."""
    fix = fix if fix is not None else np.load(FIXTURE)
    src = {"matcha": model_state_dict(), "vocoder": vocoder_state_dict()}
    tensors = {}
    for name, (key, transposed) in json.loads(str(fix["graph_sources"])).items():
        part, _, k = key.partition(".")
        tensors[name] = src[part][k].T if transposed else src[part][k]
    with gzip.open(SKELETON, "rb") as f:
        data = _fill(f.read(), tensors)
    if hashlib.sha1(data).hexdigest() != str(fix["graph_sha1"]):
        raise AssertionError("the rebuilt graph differs from the exported one")
    return data


def write_graph(directory, fix=None):
    """Writes the exported graph as <directory>/model.onnx and returns its path."""
    path = os.path.join(str(directory), "model.onnx")
    with open(path, "wb") as f:
        f.write(graph_bytes(fix))
    return path
