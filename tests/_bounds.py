"""Rounding units shared by the float64-reference numerics tests."""
import torch

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
DT = {"f32": F32, "bf16": BF16, "f16": F16}
# half an ulp relative to the value, and half the smallest subnormal, of each dtype
UNIT = {BF16: 2.0 ** -8, F16: 2.0 ** -11, F32: 2.0 ** -24}
HALF_MIN_SUB = {BF16: 2.0 ** -134, F16: 2.0 ** -25, F32: 2.0 ** -150}


def stored(e_abs, b, dt):
    """Bound b on a value whose exact magnitude is e_abs, widened by one round-to-nearest store to dt."""
    return b + UNIT[dt] * (e_abs + b) + HALF_MIN_SUB[dt]
