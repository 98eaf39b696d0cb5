"""Every host input of a call reaches the device, and every output of a call reaches the host, through the engine's pinned
staging (struct Staging in csrc/engine.cu): the layout of a call's pinned block is decided in one place, so a replayed graph,
which copies to or from the pinned addresses it captured, finds every field at the offset where the host filled it or
reads it."""
import os
import re

ENGINE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vosk_tts_b200", "csrc", "engine.cu")
# Host-to-device copies that stay direct: the weight blob, the resampler's taps, the prefetch list, the handle-free
# maximum path, and the microbenchmark and unit-test hooks; "upload" is Staging::upload and the hooks' upload helper
DIRECT = ("vtts_create", "resample_taps", "build_prefetch_list", "vtts_maximum_path", "vtts_microbench", "upload")
# Device-to-host copies that stay direct: the T2S weights' alpha read at load, the handle-free maximum path, the timeline,
# and the microbenchmark and unit-test hooks; "download" is Staging::download
DIRECT_READ = ("bind_t2s", "vtts_maximum_path", "vtts_timeline", "vtts_microbench", "download")
MAPPED = {"map"}                # the mapped buffer phase 1 publishes the frame lengths into
ROUND64 = re.compile(r"\+ 63\) / 64 \* 64")


def _source():
    with open(ENGINE) as f:
        return re.sub(r"//[^\n]*", "", f.read())        # (comments may name anything)


def _block(src, start):
    """Span from `start` to the brace closing the first one opened after it."""
    depth = 0
    for j in range(src.index("{", start), len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return start, j + 1
    raise AssertionError("unbalanced braces in engine.cu")


def _definitions(src, name):
    """Spans of every function definition called `name` (member or free)."""
    spans = [_block(src, m.start()) for m in
             re.finditer(r"^[^\n;{}()]*?\b(?:vtts_engine::)?%s\s*\([^;{]*\)\s*(?:const\s*)?\{" % name, src, re.M)]
    assert spans, "no definition of %s in engine.cu" % name
    return spans


def _struct(src, name, within=None):
    lo, hi = within or (0, len(src))
    m = re.compile(r"\bstruct %s\s*\{" % name).search(src, lo, hi)
    assert m, "engine.cu has no struct %s" % name
    return _block(src, m.start())


def _line(src, pos):
    return src.count("\n", 0, pos) + 1


def _copies_outside(src, kind, direct, caller_arg):
    """Lines of every `kind` copy outside the definitions in `direct`, the unit-test hooks (vtts_debug_*) and, in
    impl_t2s_decode, the copy of the caller's array `caller_arg`."""
    allowed = [s for name in direct for s in _definitions(src, name)]
    allowed += [s for s in (_block(src, m.start()) for m in re.finditer(r"^\w.*\bvtts_debug_\w+\s*\([^;{]*\)\s*\{", src, re.M))]
    t2s = _definitions(src, "impl_t2s_decode")
    offenders = []
    for m in re.finditer(kind, src):
        if any(lo <= m.start() < hi for lo, hi in allowed):
            continue
        if any(lo <= m.start() < hi for lo, hi in t2s):
            call = src[src.rindex("cudaMemcpy", 0, m.start()):m.start()]
            if re.search(r"[(,]\s*%s\s*," % caller_arg, call):
                continue
        offenders.append("line %d" % _line(src, m.start()))
    return offenders


def test_host_to_device_copies_go_through_the_staging():
    # (the caller's sampling draws q, up to B * q_ld * V floats, are copied once straight from its memory)
    offenders = _copies_outside(_source(), "cudaMemcpyHostToDevice", DIRECT, "q")
    assert not offenders, "host-to-device copies outside Staging::upload:\n" + "\n".join(offenders)


def test_device_to_host_copies_go_through_the_staging():
    # (the caller's logits, up to B * logits_ld * V floats, are copied once straight to its memory)
    offenders = _copies_outside(_source(), "cudaMemcpyDeviceToHost", DIRECT_READ, "logits")
    assert not offenders, "device-to-host copies outside Staging::download:\n" + "\n".join(offenders)


def test_readback_helpers_are_gone():
    src = _source()
    assert not re.search(r"\bensure_pinned\b", src), "engine.cu still has ensure_pinned"


def test_pinned_members_are_the_staging_and_the_mapped_buffer():
    src = _source()
    eng = _struct(src, "vtts_engine")
    staging = _struct(src, "Staging", eng)
    body = src[eng[0]:staging[0]] + src[staging[1]:eng[1]]
    members = set()
    for decl in re.findall(r"\b(?:PinnedBuf|MappedBuf)<[^>]*>\s+([^;]+);", body):
        members.update(n.strip() for n in decl.split(","))
    assert members == MAPPED, "pinned members of vtts_engine besides its staging: %s" % sorted(members - MAPPED)
    assert re.findall(r"\b(?:PinnedBuf|MappedBuf)<[^>]*>\s+([^;]+);", src[staging[0]:staging[1]]) == ["pin"]
    assert re.search(r"\bStaging\s+stg\s*\[\s*STG_KINDS\s*\]\s*;", body), "vtts_engine has no staging array"


def test_pinned_layout_rounding_lives_in_the_staging():
    src = _source()
    spans = [_struct(src, "Staging", _struct(src, "vtts_engine"))]
    spans += [s for name in ("bucket_tok", "bucket_frm", "set_token_shape") for s in _definitions(src, name)]
    offenders = ["line %d" % _line(src, m.start()) for m in ROUND64.finditer(src) if not any(lo <= m.start() < hi for lo, hi in spans)]
    assert not offenders, "64-byte rounding outside Staging and the row buckets:\n" + "\n".join(offenders)
