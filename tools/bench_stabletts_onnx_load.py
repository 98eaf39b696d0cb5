"""Load time of a multistream voice from its exported model.onnx: the host read of the graph (onnx_weights.stabletts_from_onnx:
protobuf parse, Linear recovery, shape inference), and the whole StableTTS.from_onnx (that read, packing, engine creation and
the upload to the GPU, ending in a device synchronise).  Median of --runs after one warm-up, over the test graph
(tests/stabletts_onnx_inputs.py rebuilds it into a temporary directory) unless --graph names another.  Prints one JSON line
with the GPU's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from vosk_tts_b200 import onnx_weights  # noqa: E402
from vosk_tts_b200.stabletts import StableTTS  # noqa: E402


def _gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graph", default=None, help="a model.onnx of matcha/onnx/export.py (default: the test graph)")
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no GPU: StableTTS.from_onnx needs one")
    with tempfile.TemporaryDirectory() as tmp:
        if a.graph is None:
            import stabletts_onnx_inputs
            a.graph = stabletts_onnx_inputs.write_graph(tmp)
        run(a)


def run(a):
    def timed(fn):
        out = []
        for i in range(a.runs + 1):
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            out.append(time.perf_counter() - t0)
            if hasattr(r, "close"):
                r.close()
        return statistics.median(out[1:])

    read = timed(lambda: onnx_weights.stabletts_from_onnx(a.graph))
    full = timed(lambda: StableTTS.from_onnx(a.graph, device=0, precision=1))
    print(json.dumps({"graph": os.path.basename(a.graph), "bytes": os.path.getsize(a.graph), "read_s": round(read, 4),
                      "from_onnx_s": round(full, 4), "gpu": _gpu()}))


if __name__ == "__main__":
    main()
