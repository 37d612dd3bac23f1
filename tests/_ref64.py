"""fp64 references and the ulp-based comparator of the kernel edge-case tests (test_gpu_tapgemm_edges.py, test_gpu_attn_edges.py;
test_ref64_selfcheck.py proves on the CPU that the bounds reject the bugs they are meant to catch).

Every reference is built in float64 from the exact fp16 / fp32 tensors the kernel received, on the device they live on.

Tap-GEMM outputs (GEMM, conv3x3, tconv3: fp32 accumulation, one rounding to fp16) pass when, element-wise,

    |got - ref64| <= k_ulp * ulp16(ref64) + c * sqrt(K_eff) * 2^-24 * sum|terms|

  sum|terms|  fp64 sum of the absolute products plus the absolute bias, group-bias and residual terms
  K_eff       taps x K plus the number of epilogue terms (a folded skip tensor is one more term of the k-loop)
  k_ulp = 1   the final fp16 rounding (0.5 ulp) with 0.5 ulp to spare

Attention outputs (P rounded to fp16 before PV, fp32 accumulation) pass when

    |got - ref64| <= 2^-11 * sum_t |p_t| |v_t| + 2^-25 * sum_t |v_t| + ulp16(O)

  the middle term covers P entries in the fp16 subnormal range, whose rounding error is absolute (<= 2^-25), not relative; the kernels
  divide by a row sum >= 1, so it is not amplified.

The cross-attention edit (CROSSEDIT of fz_attn.cu: Refine / Replace, Reweight, alpha-lerp in fp32, one rounding to fp16) is built from the
stored fp16 P, the fp16 cached source rows and the fp32 tables, and passes when

    |got - ref64| <= ulp16(ref64) + c * 2^-24 * sum|terms|

  the terms being the edit evaluated on absolute values, with a factor keys_per_slot on the Replace sum (its running fp32 sum).
The fp16 running sums of the cross maps are checked bitwise: acc_new = acc_old + P_store in fp16 (one fp32 add, one rounding), the
columns past keys_per_slot unchanged.

GroupNorm / LayerNorm outputs (test_gpu_elem_edges.py): y = gamma (x - mu) rstd + beta, rstd = 1 / sqrt(var + eps), mu and var the fp64
statistics of the fp16 inputs, pass when

    |got - y| <= ulp16(y) + gamma rstd |mu - fp32(mu)| + c * 2^-24 * (|gamma| rstd sqrt(n_stat) (|x - mu| + sigma) + |beta|)

  the second term is the rounding of the mean to fp32, which no fp32 kernel can avoid; it is 0 when the mean is representable (a
  constant row).  The third is a Welford-class statistics error: it scales with sigma, never with |mu|, so a kernel that loses the
  variance to cancellation (E[x^2] - mu^2) or rounds a fused shift -mu * rstd fails it.  With SiLU the pre-activation terms are
  multiplied by max|silu'| = 1.1 and (5 + 1.2 |y|) 2^-23 |silu(y)| is added for __expf and __fdividef.
  The GroupNorm statistics ARE E[x^2] - mu^2 from fp32 partial sums (DESIGN.md, known limits); groups far from zero mean are therefore
  checked against that bound plus  c_dc * 2^-24 * |gamma| (mu / sigma_eps)^2 (1 + |x - mu| rstd),  sigma_eps = sqrt(var + eps).

Element-wise fp32 steps (DDIM, CFG + DDIM + blend, out_temporal, the time embedding): |got - ref64| <= c * 2^-24 * sum|terms|, the
terms being the expression evaluated on absolute values (the running-error bound of its fp32 evaluation).

VAE blocks (test_gpu_vae_blocks.py) are checked against VaeBlocks64, an fp64 restatement of the diffusers 0.11.1 AutoencoderKL blocks,
on the fp16 floor: the same restatement run in torch fp16 on the GPU (weights in half, as the reference's fp16 pipeline runs them) deviates
from fp64 by floor = max|o16 - ref64|; the engine's block passes when

    max|got - ref64| <= 1.5 floor + 2 ulp16(max|ref64|)

The GroupNorm statistics exchange of the frame-sharded forward (fz_gn_combine, test_gpu_p2p_edges.py) is checked bitwise: the fp64 total
in the first slot of every statistics set equals an fp64 replay in the kernel's order and lies within the recursive-summation bound
(m - 1) 2^-53 sum|v| of the exact sum of its m = world F_loc values; the other slots of the set are exactly 0.
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


def conv3x3_rows_ref(x, w9, rows, stride=1, asym_pad=False, **epi):
    """conv3x3_ref on the output rows `rows` (flat indices into [NB, Ho, Wo]) only: the 9 input pixels of each row are gathered, so the
    fp64 work scales with len(rows), not with the image.  -> (ref, sum|terms|) [len(rows), Cout] fp64; epilogue tensors already row-selected."""
    NB, H, W, Cin = x.shape
    Ho, Wo = H // stride, W // stride
    # output (y, x) reads input row stride y + ky - 1 (symmetric) or stride y + ky (right/bottom padding): index stride y + ky of xp
    xp = F.pad(x, (0, 0, 0, 1, 0, 1)) if asym_pad else F.pad(x, (0, 0, 1, 1, 1, 1))
    rows = rows.to(x.device)
    n, r = rows // (Ho * Wo), rows % (Ho * Wo)
    yy, xx = r // Wo, r % Wo
    a = torch.stack([xp[n, stride * yy + ky, stride * xx + kx] for ky in range(3) for kx in range(3)], 1).double()  # [R, 9, Cin]
    w64 = w9.double()
    return epilogue_ref(torch.einsum("rtc,toc->ro", a, w64), torch.einsum("rtc,toc->ro", a.abs(), w64.abs()), **epi)


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
    """p [..., S, T] fp64 probabilities, v [..., T, d] fp64, o = p @ v: the attention bound of the module docstring.  |p|: an edited row
    (CROSSEDIT with a negative equalizer) has negative entries, and each entry's rounding error scales with its magnitude."""
    va = v.abs()
    return U16 * (p.abs() @ va) + 2.0 ** -25 * va.sum(-2, keepdim=True) + ulp16(o)


def check_attn(got, p, v, report=None, key="") -> dict:
    """got [..., S, d] kernel output against o = p @ v; p [..., S, T], v [..., T, d] fp64."""
    o = p @ v
    return check_bound(got, o, attn_bound(p, v, o).expand_as(o), report, key)


def check_probs(got, p, report=None, key="", k_ulp: float = 1.0) -> dict:
    """Stored probabilities: within k_ulp fp16 ulps of fp16(softmax64)."""
    r = p.double().half().double()
    return check_bound(got, r, k_ulp * ulp16(r), report, key)


# ---------------------------------------------------------------------------------------------------------- cross-attention edit
# Layout of the CROSSEDIT table (include/fatezero_b200.h): [0] mode (0 refine, 1 replace), then alpha[80], eq[80], a[80], mapper[80] and
# M[80][80] (M[w][n]: source word w into target word n).
XEDIT_FLOATS = 8 + 4 * 80 + 80 * 80
X_ALPHA, X_EQ, X_A, X_MAP, X_M = 8, 88, 168, 248, 328

# c of the edit bound: the running-error bound of the few fp32 operations after the gather / sum (eq, the lerp's product and sum).
# Measured on an H100 80GB HBM3 (700 W power limit) over every case of test_gpu_attn_edges.py that edits (each records its own
# c_needed): the largest c any case needed was 0 (every edited P within 0.5 ulp of the fp64 edit, worst err / bound 0.50).
C_EDIT = 4.0


def cross_edit_table(kind: str, kps: int) -> torch.Tensor:
    """A CROSSEDIT table (fp32, CPU) for keys_per_slot = kps whose entries tell the edit's operations apart:
    alpha cycles through 0, 1 and fractional values, eq through 1, 0, -1, 2.5, 10 and 0.5 (so eq != 1 meets every kind of alpha);
    kind "refine": fractional a, a mapper with entries -1 where a != 0;  "reweight": identity mapper, a = 1 (pure Reweight);
    "replace": M with one-to-many and many-to-one columns and non-zero rows past 64 when kps > 64 (Reweight on Replace)."""
    n = torch.arange(80)
    t = torch.zeros(XEDIT_FLOATS)
    t[0] = 1.0 if kind == "replace" else 0.0
    t[X_ALPHA:X_ALPHA + 80] = torch.tensor([0.0, 1.0, 0.375, 1.0, 0.3])[n % 5]
    t[X_EQ:X_EQ + 80] = torch.tensor([1.0, 0.0, -1.0, 2.5, 10.0, 1.0, 0.5])[n % 7]
    if kind == "reweight":
        t[X_A:X_A + 80] = 1.0
        t[X_MAP:X_MAP + 80] = n.float()
    elif kind == "refine":
        a = torch.tensor([0.0, 1.0, 0.25, 0.7])[n % 4]
        mp = (7 * n + 3) % kps
        for i in (2, 11):  # a = 0.25, 0.7: the gather of word -1 (python: the last word) is visible
            mp[i] = -1
        t[X_A:X_A + 80] = a
        t[X_MAP:X_MAP + 80] = mp.float()
    else:
        M = torch.zeros(80, 80)
        k = torch.arange(kps)
        M[(5 * k + 1) % kps, k] = 0.625
        M[(11 * k + 7) % kps, k] += 0.375
        M[kps - 3:kps, 3] = 0.5          # many-to-one: the last three words into word 3
        M[kps - 5, :min(kps, 10)] += 0.3  # one-to-many: one late word into words 0..9
        t[X_M:] = M.reshape(-1)
    return t


def cross_edit_ref(cur, base, table, kps: int):
    """fz_attn.cu CROSSEDIT in fp64: cur [..., S, >= kps] the fp16 probabilities the kernel edits (stored P), base [..., S, >= kps] the fp16
    cached source rows, table the fp32 CROSSEDIT table ->  (ref, sum|terms|) [..., S, kps] fp64, before the final fp16 rounding:
        Refine   R = b[map[n] mod kps] a[n] + cur (1 - a[n])          Replace   R = sum_{w < kps} b[w] M[w][n]
        then     R = R eq[n],  x = R al[n] + (1 - al[n]) cur."""
    t = table.double().to(cur.device)
    c, b = cur[..., :kps].double(), base[..., :kps].double()
    al, eq = t[X_ALPHA:X_ALPHA + kps], t[X_EQ:X_EQ + kps]
    if t[0].item() == 1.0:
        M = t[X_M:].view(80, 80)[:kps, :kps]
        R, T = b @ M, kps * (b.abs() @ M.abs())
    else:
        a, mp = t[X_A:X_A + kps], t[X_MAP:X_MAP + kps].long() % kps
        R = b[..., mp] * a + c * (1 - a)
        T = b[..., mp].abs() * a.abs() + c.abs() * (1 - a).abs()
    R, T = R * eq, T * eq.abs()
    return R * al + (1 - al) * c, T * al.abs() + (1 - al).abs() * c.abs()


def check_edit(got, ref, terms, report=None, key="", c: float = C_EDIT) -> dict:
    """Edited probabilities against cross_edit_ref (bound: module docstring).  Also records c_needed: the smallest c this case passes with."""
    ref, terms = ref.double(), terms.double()
    u = ulp16(ref)
    acc = U32 * terms
    err = (got.double() - ref).abs()
    c_needed = ((err - u).clamp(min=0) / acc.clamp(min=1e-300)).max().item()
    return check_bound(got, ref, u + c * acc, report, key, extra=dict(c_needed=c_needed, c=c))


def check_running_sum(new, old, p16, kps: int, report=None, key="") -> dict:
    """fp16 running sum [..., S, acc_ld] after one add: columns < kps bitwise equal to old + p16 (fp16 tensors: one fp32 add, one rounding,
    which is the kernel's fp16(fp32(acc) + fp32(fp16 p)) and the reference's fp16 +=), columns >= kps bitwise unchanged."""
    want = old[..., :kps] + p16[..., :kps]
    bad_sum = int((new[..., :kps] != want).sum().item())
    bad_pad = int((new[..., kps:] != old[..., kps:]).sum().item())
    stats = dict(n=new.numel(), sum_mismatches=bad_sum, pad_changed=bad_pad)
    _record(report, key, stats)
    assert bad_sum == 0 and bad_pad == 0, f"{key}: running sum differs from old + P in {bad_sum} elements, {bad_pad} pad columns changed"
    return stats


# ---------------------------------------------------------------------------------------------------------------- normalisation
# c of the norm bound and c_dc of the GroupNorm DC-offset term.  Measured on an H100 SXM 80 GB (132 SMs, 700 W power limit) over every
# norm case of test_gpu_elem_edges.py (each records its own c_needed / c_dc_needed in the report): the largest c a strict case needed was
# 0.14 (GroupNorm at mean/sigma = 64), the largest c_dc 0.28 (near-constant groups).
C_NORM = 0.5
C_DC = 1.0


def f32(x: float) -> float:
    """The value a kernel sees for a float argument (passed as a C float)."""
    return torch.tensor(x, dtype=torch.float32).item()


def norm_check(got, x64, dims, gamma, beta, eps: float, silu=False, report=None, key="", c: float = C_NORM, c_dc=None) -> dict:
    """got and x64 of one shape; statistics over `dims` of x64; gamma / beta fp64, broadcastable to x64.  Bound: see the module docstring
    (c_dc None: the strict bound; otherwise the strict bound plus the DC-offset term, and the strict ratio is only recorded)."""
    n = math.prod(x64.shape[d] for d in dims)
    mu = x64.mean(dims, keepdim=True)
    d = x64 - mu
    var = (d * d).mean(dims, keepdim=True)
    rstd = (var + f32(eps)).rsqrt()
    g, b = gamma.double(), beta.double()
    out = d * rstd * g + b
    ga = g.abs()
    acc = U32 * (ga * rstd * math.sqrt(n) * (d.abs() + var.sqrt()) + b.abs())
    fixed = ga * rstd * (mu - mu.float().double()).abs()
    dc = U32 * ga * (mu * rstd) ** 2 * (1 + d.abs() * rstd)
    if silu:
        y = out
        out = y * torch.sigmoid(y)
        acc, fixed, dc = 1.1 * acc, 1.1 * fixed, 1.1 * dc
        fixed = fixed + out.abs() * (5 + 1.2 * y.abs()) * 2.0 ** -23
    acc, fixed, dc = (t.expand_as(out) for t in (acc, fixed, dc))
    u = ulp16(out) + fixed
    err = (got.double() - out).abs()
    strict = u + c * acc
    extra = dict(c_needed=((err - u).clamp(min=0) / acc.clamp(min=1e-300)).max().item(), c=c, n_stat=n)
    if c_dc is None:
        return check_bound(got, out, strict, report, key, extra=extra)
    extra.update(strict_worst_err_over_bound=(err / strict).max().item(), c_dc=c_dc,
                 c_dc_needed=((err - strict).clamp(min=0) / dc.clamp(min=1e-300)).max().item())
    return check_bound(got, out, strict + c_dc * dc, report, key, extra=extra)


def gn_check(got, x, gamma, beta, eps, groups, frames_per_stat, silu, report=None, key="", **kw) -> dict:
    """GroupNorm of x [NB, HW, C] fp16 with statistics over (C / groups channels, HW, frames_per_stat consecutive images)."""
    NB, HW, Cc = x.shape
    shape = (NB // frames_per_stat, frames_per_stat, HW, groups, Cc // groups)
    gb = [t.double().view(groups, Cc // groups) for t in (gamma, beta)]
    return norm_check(got.view(shape), x.double().view(shape), (1, 2, 4), *gb, eps, silu, report, key, **kw)


def ln_check(got, x, gamma, beta, eps, report=None, key="", **kw) -> dict:
    """LayerNorm of x [M, C] fp16 over C."""
    return norm_check(got, x.double(), (1,), gamma.double(), beta.double(), eps, False, report, key, **kw)


# ------------------------------------------------------------------------------------------------------------ element-wise steps
# c of the step bound.  Measured as C_NORM: the largest c any case of test_gpu_elem_edges.py needed was 2.8 (DDIM and CFG + DDIM near
# alpha-bar = 1); out_temporal needed 2.3, the sinusoid 1.3.
C_STEP = 4.0


def check_step(got, ref, terms, report=None, key="", c: float = C_STEP) -> dict:
    ref, terms = ref.double(), terms.double()
    acc = U32 * terms
    err = (got.double() - ref).abs()
    extra = dict(c_needed=(err / acc.clamp(min=1e-300)).max().item(), c=c)
    return check_bound(got, ref, c * acc, report, key, extra=extra)


def sqrt32(a: float) -> float:
    """sqrtf of the float argument, as the host code computes the step coefficients (torch's own fp32 sqrt in the reference)."""
    return torch.tensor(f32(a), dtype=torch.float32).sqrt().item()


def ddim_coef(a: float):
    """(sqrtf(a), sqrtf(1 - a)) in fp32 from the float alpha-bar."""
    one_m = (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(f32(a), dtype=torch.float32)).item()
    return sqrt32(a), sqrt32(one_m)


def ddim_invert_ref(x, e, a_prev, a_next):
    """x_next = sqrt(a_next) x0 + sqrt(1 - a_next) e,  x0 = (x - sqrt(1 - a_prev) e) / sqrt(a_prev)  -> (ref, sum|terms|) fp64."""
    sp, s1p = ddim_coef(a_prev)
    sn, s1n = ddim_coef(a_next)
    x, e = x.double(), e.double()
    ref = sn * (x - s1p * e) / sp + s1n * e
    terms = sn * (x.abs() + s1p * e.abs()) / sp + s1n * e.abs()
    return ref, terms


def cfg_ddim_ref(x, eps2, guidance, a_t, a_prev, x_inv=None, blends=None):
    """x [K, ...], eps2 [2K, ...] = [uncond ; cond]; blends: per item None or (mask_a, mask_b | None) [F, H, W] broadcast over channels,
    blending towards x_inv.  -> (ref, sum|terms|) fp64."""
    K = x.shape[0]
    g = f32(guidance)
    st, s1t = ddim_coef(a_t)
    sp, s1p = ddim_coef(a_prev)
    x, eu, ec = x.double(), eps2[:K].double(), eps2[K:].double()
    e = eu + g * (ec - eu)
    te = eu.abs() + abs(g) * (ec.abs() + eu.abs())
    ref = sp * (x - s1t * e) / st + s1p * e
    terms = sp * (x.abs() + s1t * te) / st + s1p * te
    for k, bl in enumerate(blends or [None] * K):
        if bl is None:
            continue
        m = bl[0].double() if bl[1] is None else torch.maximum(bl[0], bl[1]).double()
        xi = x_inv.double().reshape(ref.shape[1:])
        ref[k] = xi + m * (ref[k] - xi)
        terms[k] = xi.abs() + m.abs() * (terms[k] + xi.abs())
    return ref, terms


def _tconv_frames(y, w):
    """y [B, F, P, Ci], w [Co, Ci, 3] -> [B, F, P, Co]: sum_t w[:, :, t] y[f + t - 1] (zero frames outside)."""
    yp = F.pad(y, (0, 0, 0, 0, 1, 1))
    Fr = y.shape[1]
    return sum(torch.einsum("bfpc,oc->bfpo", yp[:, t:t + Fr], w[:, :, t]) for t in range(3))


def out_temporal_ref(y, B, Co, Fr, HW, down=None, up=None, w_full=None, b_full=None):
    """y [B F HW, ldy] fp16 (Co valid columns) -> (ref, sum|terms|, fixed) [B, Co, F, HW] fp64.  The LoRA path rounds its rank-R
    intermediate to fp16 as the reference's autocast path does; `fixed` allows that rounding to land one fp16 ulp either way."""
    y64 = y[:, :Co].double().reshape(B, Fr, HW, Co)
    fixed = torch.zeros_like(y64)
    if w_full is not None:
        w = w_full.double()
        ref = _tconv_frames(y64, w)
        terms = _tconv_frames(y64.abs(), w.abs())
        if b_full is not None:
            ref, terms = ref + b_full.double(), terms + b_full.double().abs()
    elif down is not None:
        mid_exact = _tconv_frames(y64, down.double())
        mid = mid_exact.half().double()
        mid_terms = _tconv_frames(y64.abs(), down.double().abs())
        ua = up.double().abs()
        ref = y64 + _tconv_frames(mid, up.double())
        terms = y64.abs() + _tconv_frames(mid.abs(), ua) + _tconv_frames(mid_terms, ua)
        fixed = _tconv_frames(ulp16(mid_exact), ua)
    else:
        ref, terms = y64, y64.abs()
    perm = (0, 3, 1, 2)
    return ref.permute(perm), terms.permute(perm), fixed.permute(perm)


def rowvec_ref(x, w16, bias, silu_in):
    """y = W act(x) + b (act = SiLU or identity) -> (ref, sum|terms|, fixed): `fixed` carries the __expf / division error of the SiLU."""
    x64, w = x.double(), w16.double()
    a = x64 * torch.sigmoid(x64) if silu_in else x64
    ref, terms = w @ a, w.abs() @ a.abs()
    fixed = w.abs() @ (a.abs() * (5 + 1.2 * x64.abs()) * 2.0 ** -23) if silu_in else torch.zeros_like(ref)
    if bias is not None:
        ref, terms = ref + bias.double(), terms + bias.double().abs()
    return ref, terms, fixed


def sinusoid_ref(t, c0, flip, freq_shift):
    """diffusers get_timestep_embedding in fp64 -> (ref, terms): terms = |a| (1 + |z|) + 1 for the argument a = t e^z, whose fp32
    evaluation (here and in the reference) carries a relative error of a few 2^-24 per unit of |z|, plus sinf / cosf themselves."""
    half = c0 // 2
    z = -math.log(10000.0) * torch.arange(half, dtype=torch.float64) / (half - f32(freq_shift))
    a = f32(t) * torch.exp(z)
    s, co = torch.sin(a), torch.cos(a)
    ref = torch.cat([co, s]) if flip else torch.cat([s, co])
    ta = a.abs() * (1 + z.abs()) + 1
    return ref, torch.cat([ta, ta])


def quick_gelu_ref(x):
    """x sigmoid(1.702 x) in fp64 from the fp16 input -> (ref, bound): 1 fp16 ulp plus (5 + 2 |x|) 2^-23 |ref| for __expf of the
    fp32 product 1.702 x and the division."""
    x64 = x.double()
    ref = x64 * torch.sigmoid(f32(1.702) * x64)
    return ref, ulp16(ref) + ref.abs() * (5 + 2 * x64.abs()) * 2.0 ** -23


# ------------------------------------------------------------------------------------------------- GroupNorm statistics exchange
def ulp64(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp64 numbers in the binade of |x| (2^-1074 in the subnormal range)."""
    m, e = torch.frexp(x.double().abs().clamp(min=2.0 ** -1022))
    return torch.ldexp(torch.ones_like(m), e - 53)


def gn_combine_ref(own: torch.Tensor, peers: torch.Tensor, me: int, F_loc: int):
    """fz_gn_combine in fp64.  own [NB, G, 2] fp32: this rank's per-image (sum, sumsq); peers [world, NB, G, 2] fp32: rank r's values as
    they arrive in the inbox (row `me` unused).  Images are [B, F_loc] (a statistics set = the F_loc consecutive images of one clip item).
    Returns (replay, exact), both [NB, G, 2] fp64 with every set's total in its first image and 0 in the others:
      replay  the kernel's order: own value first, then the other ranks in rank order, then the frames f = 0 .. F_loc - 1;
      exact   math.fsum over the same world * F_loc values;
    and the sum of their absolute values (for the summation bound)."""
    world = peers.shape[0]
    NB, G, _ = own.shape
    acc = own.double()
    for r in range(world):
        if r != me:
            acc = acc + peers[r].double()
    sets = acc.view(NB // F_loc, F_loc, G, 2)
    tot = sets[:, 0]
    for f in range(1, F_loc):
        tot = tot + sets[:, f]
    vals = torch.cat([own.double()[None]] + [peers[r].double()[None] for r in range(world) if r != me])  # [world, NB, G, 2]
    vals = vals.view(world, NB // F_loc, F_loc, G, 2).permute(1, 3, 4, 0, 2).reshape(NB // F_loc, G, 2, -1)
    exact = torch.tensor([math.fsum(v) for v in vals.reshape(-1, vals.shape[-1]).tolist()], dtype=torch.float64).view(NB // F_loc, G, 2)
    out = [torch.zeros(NB // F_loc, F_loc, G, 2, dtype=torch.float64) for _ in range(3)]
    out[0][:, 0], out[1][:, 0], out[2][:, 0] = tot, exact, vals.abs().sum(-1)
    return tuple(t.view(NB, G, 2) for t in out)


def check_gn_combine(got: torch.Tensor, own: torch.Tensor, peers: torch.Tensor, me: int, F_loc: int, report=None, key="") -> dict:
    """got [NB, G, 2] fp64 (the totals of fz_gn_combine) against gn_combine_ref: first slots bitwise equal to the replay and within
    (m - 1) 2^-53 sum|v| of the exact sum (m = world F_loc values), the other slots of every set exactly 0 (bitwise +0)."""
    replay, exact, abs_sum = gn_combine_ref(own.cpu(), peers.cpu(), me, F_loc)
    m = peers.shape[0] * F_loc
    got = got.cpu()
    NB, G, _ = got.shape
    first = torch.zeros(NB // F_loc, F_loc, G, 2, dtype=torch.bool)
    first[:, 0] = True
    first = first.view(NB, G, 2)
    assert got.dtype == torch.float64, got.dtype
    gb = got.view(torch.int64)
    bad_rest = int((gb[~first] != 0).sum().item())
    bad_replay = int((gb[first] != replay.view(torch.int64)[first]).sum().item())
    err = (got - exact).abs()[first]
    ratio = err / ((m - 1) * 2.0 ** -53 * abs_sum[first]).clamp(min=1e-300)
    stats = dict(n=got.numel(), sets=int(first.sum().item()), replay_mismatches=bad_replay, nonzero_rest=bad_rest,
                 max_ulps_from_exact=(err / ulp64(exact[first])).max().item(), worst_err_over_bound=ratio.max().item())
    _record(report, key, stats)
    assert bad_rest == 0, f"{key}: {bad_rest} non-first slots of the statistics sets are not 0"
    assert bad_replay == 0, f"{key}: {bad_replay} set totals differ from the fp64 replay in the kernel's order"
    assert stats["worst_err_over_bound"] <= 1.0, f"{key}: a set total is off the exact sum by {stats['worst_err_over_bound']:.2f} x the summation bound"
    return stats


# --------------------------------------------------------------------------------------------------------- blend mask and heat maps
MASK_TIE = 1e-5  # blend-mask pixels whose fp64 ratio lies this close to th are reported, not asserted
HEAT_TIE = 1e-4  # heat-map pixels whose fp64 255 a / max lies this close to an integer are reported, not asserted


def blend_mask_ratio(maps, word_w, h, w, ntok=77):
    """spatial_blend.py get_mask in fp64: maps [F, heads, r*r, >= ntok] (one per layer) -> (sum_n map w_n).mean(layers, heads), 3x3 max-pool
    (stride 1, pad 1), nearest resize to (h, w) with F.interpolate's fp32 source index, divided by the per-frame max.  Returns the ratio [F, h, w] (NaN where the max is 0)."""
    Fr, heads, rr, _ = maps[0].shape
    r = int(round(rr ** 0.5))
    ww = word_w.double()[:ntok].to(maps[0].device)
    st = torch.stack([(m[..., :ntok].double() * ww).sum(-1) for m in maps]).mean((0, 2)).reshape(Fr, 1, r, r)
    pooled = F.max_pool2d(st, 3, 1, 1)[:, 0]
    mk = pooled[:, nearest_index(r, h).to(pooled.device)][:, :, nearest_index(r, w).to(pooled.device)]
    return mk / mk.amax((-2, -1), keepdim=True)


def nearest_index(n_in: int, n_out: int) -> torch.Tensor:
    """F.interpolate(mode="nearest") source index as torch computes it for fp16 / fp32 tensors: min(floor(dst * ((float)n_in / n_out)),
    n_in - 1) in fp32.  (On fp64 tensors torch uses a double scale, which differs at some sizes: the reference's maps are fp16 / fp32.)"""
    scale = torch.tensor(n_in, dtype=torch.float32) / n_out
    return torch.floor(torch.arange(n_out, dtype=torch.float32) * scale).long().clamp(max=n_in - 1)


def check_mask(got, ratio, th, report=None, key="") -> dict:
    """Every pixel equal to ratio > th (NaN -> 0), except those with |ratio - th| <= MASK_TIE (counted as n_near, not asserted)."""
    want = ratio.gt(th).to(got.dtype)
    near = (ratio - th).abs() <= MASK_TIE
    bad = (got != want) & ~near
    stats = dict(n=got.numel(), n_near=int(near.sum().item()), ones=want.mean().item(), mismatches=int(bad.sum().item()))
    _record(report, key, stats)
    assert stats["mismatches"] == 0, f"{key}: {stats['mismatches']} mask pixels differ from the fp64 reference ({stats})"
    return stats


def heatmap_values(maps, ntok):
    """fz_cross_heatmaps in fp64: maps [F, heads, rr, ldm] -> 255 a / max over pixels, a = sum over maps and heads; [F, ntok, rr].
    A column whose maximum is 0 gives 0."""
    a = torch.stack([m[..., :ntok].double() for m in maps]).sum((0, 2)).transpose(1, 2)  # [F, ntok, rr]
    mx = a.amax(-1, keepdim=True)
    return torch.where(mx > 0, 255 * a / mx.clamp(min=1e-300), torch.zeros_like(a))


def check_heatmaps(got, v, report=None, key="") -> dict:
    """got uint8 [F, ntok, rr] == floor(min(255, v)) except where v is within HEAT_TIE of an integer (there: within 1)."""
    want = v.clamp(max=255).floor()
    near = (v - v.round()).abs() <= HEAT_TIE
    g = got.double()
    bad = ((g != want) & ~near) | ((g - v).abs() > 1)
    stats = dict(n=got.numel(), n_near=int(near.sum().item()), mismatches=int(bad.sum().item()))
    _record(report, key, stats)
    assert stats["mismatches"] == 0, f"{key}: {stats['mismatches']} heat-map pixels differ from the fp64 reference ({stats})"
    return stats


# ---------------------------------------------------------------------------------------------------------------------------- VAE blocks
class VaeBlocks64:
    """The blocks of diffusers 0.11.1 AutoencoderKL, NCHW, restated from the published forward code of that release (models/resnet.py
    ResnetBlock2D / Downsample2D(padding=0) / Upsample2D, models/attention.py AttentionBlock, models/vae.py Encoder / Decoder heads,
    AutoencoderKL quant_conv / post_quant_conv), independently of oracle/vae_oracle.py.

    It computes in the dtype it is given: float64 for the reference; float16 on the GPU for the fp16 floor (weights in half, the attention
    scores through baddbmm with alpha = scale and the softmax in fp32 cast back to half, as AttentionBlock runs under fp16).  `rnd` is
    applied to the result of every op: identity, or a rounding to fp16 to emulate the fp16 run in fp64 on the CPU.  `bug` selects one
    deliberate mistake from BUGS (test_ref64_selfcheck.py shows that check_block rejects each)."""
    BUGS = ("qk_swapped", "scale_1_over_c", "scale_c_quarter", "softmax_over_queries", "vbias_dropped", "vbias_unnormalised",
            "quant_wq_transposed", "conv_out_col_offset", "down_pad_left_top", "gn_eps_1e-5", "upsample_index_off_by_one")

    def __init__(self, sd, dtype, device, groups: int = 32, rnd=None, bug=None):
        assert bug is None or bug in self.BUGS, bug
        self.sd, self.dtype, self.dev, self.groups = sd, dtype, device, groups
        self.rnd = rnd or (lambda t: t)
        self.bug = bug

    def p(self, name):
        return self.sd[name].to(self.dev, self.dtype)

    def conv(self, n, x, stride=1, padding=1):
        return self.rnd(F.conv2d(x, self.p(n + ".weight"), self.p(n + ".bias"), stride=stride, padding=padding))

    def gn(self, n, x, silu):
        eps = 1e-5 if self.bug == "gn_eps_1e-5" else 1e-6
        y = self.rnd(F.group_norm(x, self.groups, self.p(n + ".weight"), self.p(n + ".bias"), eps))
        return self.rnd(F.silu(y)) if silu else y

    def resnet(self, n, x):
        h = self.conv(n + ".conv1", self.gn(n + ".norm1", x, True))
        h = self.conv(n + ".conv2", self.gn(n + ".norm2", h, True))
        if n + ".conv_shortcut.weight" in self.sd:
            x = self.conv(n + ".conv_shortcut", x, padding=0)
        return self.rnd(x + h)  # output_scale_factor 1

    def attn(self, n, x, probs_out=None):
        """AttentionBlock (one head of width C, rescale_output_factor 1).  probs_out: a list that receives the probabilities."""
        B, Cc, H, W = x.shape
        h = self.gn(n + ".group_norm", x, False).reshape(B, Cc, H * W).transpose(1, 2)
        q = self.rnd(F.linear(h, self.p(n + ".query.weight"), self.p(n + ".query.bias")))
        k = self.rnd(F.linear(h, self.p(n + ".key.weight"), self.p(n + ".key.bias")))
        bv = self.p(n + ".value.bias")
        v = self.rnd(F.linear(h, self.p(n + ".value.weight"), None if self.bug in ("vbias_dropped", "vbias_unnormalised") else bv))
        if self.bug == "qk_swapped":
            q, k = k, q
        scale = {"scale_1_over_c": 1.0 / Cc, "scale_c_quarter": Cc ** -0.25}.get(self.bug, Cc ** -0.5)
        s = self.rnd(torch.baddbmm(torch.empty(B, H * W, H * W, dtype=q.dtype, device=q.device), q, k.transpose(1, 2), beta=0, alpha=scale))
        dim = -2 if self.bug == "softmax_over_queries" else -1
        pr = self.rnd(torch.softmax(s.float() if s.dtype == torch.float16 else s, dim=dim).to(s.dtype))
        if probs_out is not None:
            probs_out.append(pr)
        o = self.rnd(torch.bmm(pr, v))
        if self.bug == "vbias_unnormalised":
            # the bias rides through the un-normalised exp(s - max): it comes out multiplied by the row sum instead of by 1
            e = torch.exp(s.double() - s.double().amax(-1, keepdim=True)).sum(-1, keepdim=True).to(o.dtype)
            o = self.rnd(o + e * bv)
        o = self.rnd(F.linear(o, self.p(n + ".proj_attn.weight"), self.p(n + ".proj_attn.bias")))
        return self.rnd(o.transpose(1, 2).reshape(B, Cc, H, W) + x)

    def down(self, n, x):
        pad = (1, 0, 1, 0) if self.bug == "down_pad_left_top" else (0, 1, 0, 1)
        return self.conv(n + ".conv", F.pad(x, pad), stride=2, padding=0)

    def up(self, n, x):
        H, W = x.shape[-2:]
        if self.bug == "upsample_index_off_by_one":
            iy, ix = ((torch.arange(2 * H) + 1) // 2).clamp(max=H - 1), ((torch.arange(2 * W) + 1) // 2).clamp(max=W - 1)
            x = x[:, :, iy.to(x.device)][:, :, :, ix.to(x.device)]
        else:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
        return self.conv(n + ".conv", x)

    def _col_offset(self, y):  # the conv_out's padded output read one column late: channel c from column c + 1 (the last from a zero pad)
        return torch.cat([y[:, 1:], torch.zeros_like(y[:, :1])], 1) if self.bug == "conv_out_col_offset" else y

    def encoder_in(self, img):
        return self.conv("encoder.conv_in", img)

    def encoder_out(self, x):
        """conv_norm_out + SiLU + conv_out + quant_conv -> moments (mean | logvar)."""
        h = self.conv("encoder.conv_out", self.gn("encoder.conv_norm_out", x, True))
        wq = self.p("quant_conv.weight")
        if self.bug == "quant_wq_transposed":
            wq = wq.transpose(0, 1)
        return self._col_offset(self.rnd(F.conv2d(h, wq, self.p("quant_conv.bias"))))

    def decoder_in(self, z):
        return self.conv("decoder.conv_in", self.conv("post_quant_conv", z, padding=0))

    def decoder_out(self, x):
        return self._col_offset(self.conv("decoder.conv_out", self.gn("decoder.conv_norm_out", x, True)))


def vae_block_state_dict(spec, seed: int = 0, qk_scale: float = 3.0):
    """Seeded fp32 AutoencoderKL weights {name: shape} -> {name: tensor} whose blocks are sensitive to the mistakes check_block must catch:
    biases of std 0.3 (the value bias is visible after P V), and query / key weights scaled by qk_scale over the fan_in^-1/2 default, so
    that the single-head attention over a GroupNorm'ed input is peaked (median row maximum ~0.7 at 4096 keys for qk_scale 3) instead of
    close to uniform."""
    sd = {}
    for i, name in enumerate(sorted(spec)):
        shape = tuple(spec[name])
        g = torch.Generator().manual_seed(seed * 100003 + i)
        t = torch.randn(shape, generator=g)
        if name.endswith("bias"):
            t = 0.3 * t
        elif len(shape) == 1:
            t = 1 + 0.2 * t
        else:
            t = t * math.prod(shape[1:]) ** -0.5
            if ".attentions.0.query." in name or ".attentions.0.key." in name:
                t = t * qk_scale
        sd[name] = t
    return sd


FLOOR_RATIO = 1.5  # the engine may deviate from fp64 1.5 times as much as the fp16 restatement does, plus K_ULP_BLOCK fp16 ulps
K_ULP_BLOCK = 2.0


def check_block(got, ref, o16, report=None, key="") -> dict:
    """A VAE block's output against its fp64 restatement on the fp16 floor (module docstring): got, ref, o16 of one shape."""
    got, ref, o16 = got.double(), ref.double(), o16.double()
    assert got.shape == ref.shape == o16.shape, (got.shape, ref.shape, o16.shape)
    assert torch.isfinite(got).all(), f"{key}: non-finite output"
    err = (got - ref).abs()
    floor = (o16 - ref).abs().max().item()
    bound = FLOOR_RATIO * floor + K_ULP_BLOCK * ulp16(ref.abs().max()).item()
    stats = dict(max_abs=err.max().item(), fp16_floor=floor, ratio_to_floor=err.max().item() / max(floor, 1e-300), bound=bound,
                 max_ulps=(err / ulp16(ref)).max().item(), ref_abs_max=ref.abs().max().item(), n=ref.numel())
    _record(report, key, stats)
    assert stats["max_abs"] <= bound, (f"{key}: max|got - ref64| {stats['max_abs']:.4g} > {FLOOR_RATIO} x fp16 floor {floor:.4g} + "
                                       f"{K_ULP_BLOCK:g} ulps = {bound:.4g}")
    return stats
