"""fp64 references and the ulp-based comparator of the kernel edge-case tests (test_gpu_tapgemm_edges.py, test_gpu_attn_edges.py;
test_ref64_selfcheck.py proves on the CPU that the bounds reject the bugs they are meant to catch).

Every reference is built in float64 from the exact fp16 / fp32 tensors the kernel received, on the device they live on.

Tap-GEMM outputs (GEMM, conv3x3, tconv3: fp32 accumulation, one rounding to fp16) pass when, element-wise,

    |got - ref64| <= k_ulp * ulp16(ref64) + c * sqrt(K_eff) * 2^-24 * sum|terms|

  sum|terms|  fp64 sum of the absolute products plus the absolute bias, group-bias and residual terms
  K_eff       taps x K plus the number of epilogue terms (a folded skip tensor is one more term of the k-loop)
  k_ulp = 1   the final fp16 rounding (0.5 ulp) with 0.5 ulp to spare

Attention outputs (P rounded to fp16 before PV, fp32 accumulation) pass when

    |got - ref64| <= 2^-11 * sum_t p_t |v_t| + 2^-25 * sum_t |v_t| + ulp16(O)

  the middle term covers P entries in the fp16 subnormal range, whose rounding error is absolute (<= 2^-25), not relative; the kernels
  divide by a row sum >= 1, so it is not amplified.
"""
import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24  # fp32 unit roundoff
U16 = 2.0 ** -11  # fp16 unit roundoff

# c of the tap-GEMM bound.  Measured on an H100 SXM 80 GB (132 SMs, 700 W power limit) over every case of test_gpu_tapgemm_edges.py:
# the largest c any case needed was 0.12 (test_gemm_many_tiles[256]; each case records its own as "c_needed" in the report).
C_ACC = 0.5


def ulp16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers in the binade of |x| (2^-24 in the subnormal range), in float64."""
    m, e = torch.frexp(x.double().abs().clamp(min=2.0 ** -14))
    return torch.ldexp(torch.ones_like(m), e - 11)


def _record(report, key, stats):
    if report is not None:
        report[key] = stats


def check_bound(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, report=None, key="", extra=None) -> dict:
    """Element-wise |got - ref| <= bound.  Records max_ulps, max_abs and the bound at the worst element (largest err / bound)."""
    got = got.double()
    ref, bound = ref.double(), bound.double()
    assert got.shape == ref.shape == bound.shape, (got.shape, ref.shape, bound.shape)
    err = (got - ref).abs()
    ratio = err / bound
    worst = int(torch.argmax(torch.nan_to_num(ratio, nan=math.inf)).item())
    stats = dict(max_ulps=(err / ulp16(ref)).max().item(), max_abs=err.max().item(), worst_err_over_bound=ratio.flatten()[worst].item(),
                 bound_at_worst=bound.flatten()[worst].item(), n=ref.numel(), **(extra or {}))
    _record(report, key, stats)
    assert torch.isfinite(got).all(), f"{key}: non-finite output"
    bad = int((err > bound).sum().item())
    assert bad == 0, (f"{key}: {bad}/{ref.numel()} elements out of bound; worst at flat index {worst}: got {got.flatten()[worst].item():.6g} "
                      f"ref {ref.flatten()[worst].item():.6g} bound {bound.flatten()[worst].item():.3g} ({stats['max_ulps']:.2f} ulps max)")
    return stats


def check_tap(got, ref, terms, k_eff: int, report=None, key="", k_ulp: float = 1.0, c: float = C_ACC, fixed=0.0) -> dict:
    """Comparator of the tap-GEMM family (see the module docstring); `fixed` is an extra absolute term (an approximated activation).
    Also records c_needed: the smallest c this case passes with."""
    ref, terms = ref.double(), terms.double()
    u = k_ulp * ulp16(ref) + fixed
    acc = math.sqrt(k_eff) * U32 * terms
    err = (got.double() - ref).abs()
    c_needed = ((err - u).clamp(min=0) / acc.clamp(min=1e-300)).max().item()
    return check_bound(got, ref, u + c * acc, report, key, extra=dict(c_needed=c_needed, c=c, k_eff=k_eff))


# ------------------------------------------------------------------------------------------------------------------- tap-GEMM references
def epilogue_ref(ref, terms, bias=None, group_bias=None, rows_per_group=1, residuals=()):
    """ref/terms [M, N] fp64 (+ bias [N], + group_bias[m // rows_per_group], + each residual [M, N]) with their absolute values."""
    M, N = ref.shape
    if bias is not None:
        b = bias.double()[:N]
        ref, terms = ref + b, terms + b.abs()
    if group_bias is not None:
        g = group_bias.double()[torch.arange(M, device=ref.device) // rows_per_group, :N]
        ref, terms = ref + g, terms + g.abs()
    for r in residuals:
        r = r.double().reshape(M, N)
        ref, terms = ref + r, terms + r.abs()
    return ref, terms


def gemm_ref(a, w, **epi):
    """a [M, K] fp16, w [N, K] fp16 -> (ref, sum|terms|) [M, N] fp64."""
    a64, w64 = a.double(), w.double()
    return epilogue_ref(a64 @ w64.t(), a64.abs() @ w64.abs().t(), **epi)


def conv3x3_ref(x, w9, stride=1, asym_pad=False, **epi):
    """x [NB, H, W, Cin] fp16 NHWC, w9 [9, Cout, Cin] (tap = ky * 3 + kx) -> (ref, sum|terms|) [NB * Ho * Wo, Cout] fp64.
    asym_pad: F.pad(x, (0, 1, 0, 1)) then a stride-2 conv without padding (the VAE encoder's downsample)."""
    Cout, Cin = w9.shape[1], w9.shape[2]
    x64 = x.double().permute(0, 3, 1, 2)
    w64 = w9.double().reshape(3, 3, Cout, Cin).permute(2, 3, 0, 1)
    pad = 1
    if asym_pad:
        x64, pad = F.pad(x64, (0, 1, 0, 1)), 0

    def conv(xx, ww):
        return F.conv2d(xx, ww, stride=stride, padding=pad).permute(0, 2, 3, 1).reshape(-1, Cout)

    return epilogue_ref(conv(x64, w64), conv(x64.abs(), w64.abs()), **epi)


def tconv3_ref(x, w3, halo=False, **epi):
    """x [B, F, HW, Cin] fp16 (halo: [B, F + 2, HW, Cin], frames 0 and F + 1 are the neighbours' boundary frames), w3 [3, Cout, Cin]
    -> (ref, sum|terms|) [B * F * HW, Cout] fp64:  out[f] = sum_t w3[t] x[f + t - 1]  (zero frames beyond the clip unless halo)."""
    x64 = x.double()
    if not halo:
        x64 = F.pad(x64, (0, 0, 0, 0, 1, 1))
    Fo = x64.shape[1] - 2
    w64 = w3.double()
    ref = sum(torch.einsum("bfpc,oc->bfpo", x64[:, t:t + Fo], w64[t]) for t in range(3))
    terms = sum(torch.einsum("bfpc,oc->bfpo", x64[:, t:t + Fo].abs(), w64[t].abs()) for t in range(3))
    Cout = w3.shape[1]
    return epilogue_ref(ref.reshape(-1, Cout), terms.reshape(-1, Cout), **epi)


# ------------------------------------------------------------------------------------------------------------------ attention references
def softmax64(s: torch.Tensor) -> torch.Tensor:
    return torch.softmax(s.double(), dim=-1)


def attn_bound(p: torch.Tensor, v: torch.Tensor, o: torch.Tensor) -> torch.Tensor:
    """p [..., S, T] fp64 probabilities, v [..., T, d] fp64, o = p @ v: the attention bound of the module docstring."""
    va = v.abs()
    return U16 * (p @ va) + 2.0 ** -25 * va.sum(-2, keepdim=True) + ulp16(o)


def check_attn(got, p, v, report=None, key="") -> dict:
    """got [..., S, d] kernel output against o = p @ v; p [..., S, T], v [..., T, d] fp64."""
    o = p @ v
    return check_bound(got, o, attn_bound(p, v, o).expand_as(o), report, key)


def check_probs(got, p, report=None, key="", k_ulp: float = 1.0) -> dict:
    """Stored probabilities: within k_ulp fp16 ulps of fp16(softmax64)."""
    r = p.double().half().double()
    return check_bound(got, r, k_ulp * ulp16(r), report, key)
