"""fp64 reference and error bound of fz_gelu_f16 (exact erf GELU, the MLP activation of SD-2.x text encoders), shared by the GPU parity
test and its CPU self-check."""
import math

import torch

from _ref64 import ulp16


def gelu_ref(x: torch.Tensor):
    """0.5 x (1 + erf(x / sqrt 2)) in fp64 from the fp16 input -> (ref, bound).  The kernel evaluates it in fp32: the product x / sqrt 2,
    erff (2 ulp), 1 + erf and the two products round once each, so the fp32 result is off by at most 4 2^-24 of the O(1) factor
    (1 + erf), times 0.5 |x|, plus 4 2^-24 |ref| for the products; the fp16 store adds at most one fp16 ulp."""
    x64 = x.double()
    ref = 0.5 * x64 * (1.0 + torch.special.erf(x64 / math.sqrt(2.0)))
    return ref, ulp16(ref) + (0.5 * x64.abs() + ref.abs()) * 4 * 2.0 ** -24


def all_finite_f16() -> torch.Tensor:
    """Every finite fp16 value (63 488 of them, both zeros included)."""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    return x[torch.isfinite(x)].contiguous()
