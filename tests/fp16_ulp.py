"""Unit in the last place of fp16, for tests that bound a kernel's once-rounded fp16 outputs against float64 references."""
import torch


def ulp16(x):
    """spacing of the fp16 numbers at |x| (2^-24 in the subnormal range)"""
    return torch.exp2(torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14))) - 10)
