"""Operand hook of the oracle for operand_format="fp16x3" (test infrastructure; may import oracle/)."""
import torch


def round_fp16x3(t):
    """fp16(x) + fp16(x - fp16(x)), evaluated in the tensor's own (fp64) precision: the value an fp16x3 hi / lo pair carries.
    The kernels also drop the lo * lo term of each product (relative 2^-22 of it), which this hook keeps."""
    hi = t.to(torch.float16).to(t.dtype)
    return hi + (t - hi).to(torch.float16).to(t.dtype)
