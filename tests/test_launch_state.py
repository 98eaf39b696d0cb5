"""The launch helpers size every launch from the rows and the tuning they are handed (Rows, Tuning in csrc/engine.cu), not
from engine members a caller overwrites and puts back.  A fixed launch shape is then a value passed to the launches of one
path, and cannot leak into a launch of another or be lost by one that forgets to set it."""
import os
import re

ENGINE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "vosk_tts_b200", "csrc", "engine.cu")
ASSIGN = r"\s*(?:[-+*/%&|^]|<<|>>)?=(?!=)"
# the functions that set the call's host-side lengths: the shape of the call, and nothing else
SHAPE_FUNCTIONS = ("set_token_shape", "set_frame_shape", "pack_frames", "assume_frames", "read_published_lengths", "setup_lengths",
                   "finish1")
LENGTHS = r"\b(v_tok_len|v_frm_len|h_tok_len|h_frm_len)\b"


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


def _definition(src, name):
    m = re.search(r"\b(?:void|bool|int)\s+(?:vtts_engine::)?%s\s*\([^;{]*\{" % name, src)
    assert m, "no definition of %s in engine.cu" % name
    return _block(src, m.start())


def _line(src, pos):
    return src.count("\n", 0, pos) + 1


def _tuning(src):
    m = re.search(r"\bstruct Tuning\s*\{", src)
    assert m, "engine.cu has no struct Tuning holding the launch tuning"
    lo, hi = _block(src, m.start())
    head = src[lo:src.index("static Tuning from_env", lo)]
    fields = [f for decl in re.findall(r"\bint\s+([^;]+);", head) for f in re.findall(r"(\w+)\s*=", decl)]
    return (lo, hi), fields


def test_tuning_fields_are_set_only_inside_the_tuning_struct():
    src = _source()
    (lo, hi), fields = _tuning(src)
    for f in ("conv_max_s", "conv_target", "conv_max_g", "conv_big_g", "conv_min_g", "conv_auto_g", "tc_tall", "tc_baseoff",
              "tc_dbgskip", "tc_bn", "tc_mc", "tc_split", "tc_min_steps", "tc_persist", "tc_persist_min", "tc_wmc", "attn_rows",
              "attn_split", "attn_tc_mode"):
        assert f in fields, f
    outside = src[:lo] + "\n" * src[lo:hi].count("\n") + src[hi:]
    offenders = []
    for f in fields:
        for m in re.finditer(r"\b%s\b%s" % (f, ASSIGN), outside):
            offenders.append("line %d: %s assigned" % (_line(outside, m.start()), f))
        for m in re.finditer(r"(?<![.>\w])%s\b" % f, outside):   # a loose member or local of that name
            offenders.append("line %d: %s outside a Tuning" % (_line(outside, m.start()), f))
    assert not offenders, "launch tuning set outside struct Tuning (env parsing and the named policies):\n" + "\n".join(offenders)


def test_host_lengths_are_set_only_by_the_shape_functions():
    src = _source()
    spans = [_definition(src, name) for name in SHAPE_FUNCTIONS]
    offenders = []
    for m in re.finditer(LENGTHS + r"(?:\s*\[[^\]]*\])?(?:%s|\s*\.\s*(?:assign|resize|insert|push_back|clear|swap)\s*\()" % ASSIGN, src):
        if not any(lo <= m.start() < hi for lo, hi in spans):
            offenders.append("line %d: %s" % (_line(src, m.start()), m.group(1)))
    assert not offenders, "host lengths written outside " + ", ".join(SHAPE_FUNCTIONS) + ":\n" + "\n".join(offenders)


def test_no_launch_is_sized_by_the_identity_of_its_length_array():
    src = _source()
    hits = [_line(src, m.start()) for m in re.finditer(r"d_tok_len\.p\s*[!=]=|[!=]=\s*(?:\w+\s*->\s*)?d_tok_len\.p\b", src)]
    assert not hits, "d_tok_len.p compared with a pointer at lines %s" % hits
