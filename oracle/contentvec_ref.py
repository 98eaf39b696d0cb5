"""The unmodified reference ContentVec (vc/contentvec.py's HubertModelWithFinalProj on transformers), built for the oracle
tests and the fixture generator where the reference tree and transformers are present."""
import os
import sys
import types

import torch

REF_VC = os.path.join(os.environ.get("VTTS_REFERENCE_ROOT", "/root/reference"), "vc")


def available():
    if not os.path.isfile(os.path.join(REF_VC, "contentvec.py")):
        return False
    try:
        import transformers  # noqa: F401
    except Exception:
        return False
    return True


def build(sd):
    """The model with `sd` loaded, eager attention, in eval mode.  Two shims: the file uses torch without importing it, and
    transformers 5.x wants the defining module in sys.modules before it instantiates the class."""
    from transformers import HubertConfig
    name = "vc_contentvec_ref"
    if name not in sys.modules:
        mod = types.ModuleType(name)
        mod.torch = torch
        mod.__file__ = os.path.join(REF_VC, "contentvec.py")
        sys.modules[name] = mod
        with open(mod.__file__) as f:
            exec(compile(f.read(), mod.__file__, "exec"), mod.__dict__)
    cfg = HubertConfig(conv_bias=False, classifier_proj_size=256)
    cfg._attn_implementation = "eager"
    net = sys.modules[name].HubertModelWithFinalProj(cfg).eval()
    missing, unexpected = net.load_state_dict(sd, strict=False)
    # the state dict spells the positional conv's weight norm weight_g / weight_v, which the module maps onto its
    # parametrization (original0 / original1): those two may show as missing, nothing else may
    assert not unexpected, unexpected
    assert set(missing) <= {"encoder.pos_conv_embed.conv.parametrizations.weight.original0",
                            "encoder.pos_conv_embed.conv.parametrizations.weight.original1"}, missing
    return net
