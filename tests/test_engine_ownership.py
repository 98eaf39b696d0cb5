"""Every CUDA allocation and release of the engine goes through the owner types of csrc/owned.cuh, so that destroying a handle
(or leaving a scope on an error) frees exactly what was allocated.  A direct call anywhere else would be a resource with
no owner."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vosk_tts_b200", "csrc")
RAW = ("cudaFree", "cudaFreeHost", "cudaMalloc", "cudaMallocHost", "cudaHostAlloc", "cudaEventDestroy", "cudaStreamDestroy",
       "cudaGraphDestroy", "cudaGraphExecDestroy")
CALL = re.compile(r"\b(%s)\s*\(" % "|".join(RAW))


def test_only_owned_cuh_allocates_or_releases():
    offenders = []
    for name in sorted(os.listdir(CSRC)):
        if name == "owned.cuh":
            continue
        with open(os.path.join(CSRC, name)) as f:
            for i, line in enumerate(f, 1):
                m = CALL.search(line)
                if m:
                    offenders.append("%s:%d %s" % (name, i, m.group(1)))
    assert not offenders, "raw CUDA allocation / release outside owned.cuh:\n" + "\n".join(offenders)


def test_owned_cuh_holds_the_owners():
    with open(os.path.join(CSRC, "owned.cuh")) as f:
        src = f.read()
    for nm in RAW:
        assert re.search(r"\b%s\s*[(,>]" % nm, src), nm
