"""Opt-in single-pass FP16 inference under the reference's name (det3d/core/fp16/hooks.py:84-93).

The reference's `wrap_fp16_model` casts the model to half and patches its norm layers back to fp32.  Here the
convolutions are the project's own kernels, which pack the fp32 parameters into f16 operands themselves, so the
parameters stay fp32: wrapping selects the "fp16" math (one f16 plane per activation, one MMA per product; DESIGN 3.0)
and sets `fp16_enabled` where a module declares it.  BatchNorm (folded into the kernels' epilogues from its fp32
statistics) and the heads' fp32 outputs are left as they are.  `InferencePipeline.set_math("fp16")` does the same for
a pipeline and also drops its captured graphs.
"""


def wrap_fp16_model(model):
    """Switch `model` (a detector with `set_math`) to single-pass FP16 in place and return it."""
    if not hasattr(model, "set_math"):
        raise TypeError("wrap_fp16_model: %s has no fused convolution path (set_math)" % type(model).__name__)
    model.set_math("fp16")
    for m in model.modules():
        if hasattr(m, "fp16_enabled"):
            m.fp16_enabled = True
    return model


__all__ = ["wrap_fp16_model"]
