"""CPU proof that the fp64 comparators of tests/_ref64.py are tight enough: they accept a correctly rounded fp16 result and reject the same
result with one element moved by 3 ulps, a bias applied one column off, or one 64-wide k-block missing (and, for attention, probabilities
normalised slightly differently or one 64-key block missing).  The norm bounds reject a variance over n - 1, eps outside the square root,
per-frame instead of joint-frame statistics and the fused-shift rounding on a constant row; the softmax bound a scale one fp16 ulp off;
the mask and heat-map checks a resize index off by one (and the integer nearest index) and a white all-zero column; the step bound CFG
guidance applied to the wrong half.  The GroupNorm statistics-exchange check rejects sets read as [F_loc, B], the own rank counted twice,
non-first slots left unzeroed and a rounding to fp32 after every rank's add (or of the set total).  The VAE block check (check_block on
the fp16 floor, with the fp16 run emulated by a rounding to fp16 after every op) rejects q and k swapped, a softmax scale of 1/C or C^-1/4,
a softmax over the queries, the value bias dropped or carried through the un-normalised probabilities, quant_conv folded with its weight
transposed, the padded conv_out read one column late, downsample padding on the left / top, GroupNorm eps 1e-5 on a near-constant group
and the nearest-upsample index off by one.  No GPU: everything here is fp64 on the CPU."""
import pytest
import torch
import torch.nn.functional as F

from _ref64 import (X_A, X_ALPHA, X_EQ, X_M, X_MAP, VaeBlocks64, blend_mask_ratio, cfg_ddim_ref, check_attn, check_block, check_edit,
                    check_heatmaps, check_mask, check_gn_combine, check_probs, check_running_sum, check_step, check_tap, conv3x3_ref,
                    conv3x3_rows_ref, cross_edit_ref, cross_edit_table, ddim_invert_ref, gemm_ref, gn_check, heatmap_values, ln_check,
                    nearest_index, softmax64, ulp16, vae_block_state_dict)
from oracle.vae_oracle import vae_param_spec


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def gemm_case(M=96, N=80, K=200):
    a = rnd(M, K, seed=1).half()
    w = rnd(N, K, seed=2, scale=K ** -0.5).half()
    bias = rnd(N, seed=3)
    ref, terms = gemm_ref(a, w, bias=bias)
    return a, w, bias, ref, terms, K + 1


def test_ulp16_binades():
    x = torch.tensor([1.0, 1.5, 0.999, 2.0 ** -14, 2.0 ** -20, 0.0, -3.0, 65504.0], dtype=torch.float64)
    want = torch.tensor([2.0 ** -10, 2.0 ** -10, 2.0 ** -11, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 2.0 ** -9, 32.0], dtype=torch.float64)
    assert torch.equal(ulp16(x), want)
    # ulp16 is the spacing of fp16 itself: nextafter in fp16 differs by exactly one ulp16
    h = rnd(1000, seed=9).half()
    nxt = torch.nextafter(h, torch.full_like(h, float("inf")))
    assert torch.equal((nxt.double() - h.double()), ulp16(h.double()))


def test_tap_accepts_correct_rounding():
    _, _, _, ref, terms, k_eff = gemm_case()
    check_tap(ref.half(), ref, terms, k_eff)


@pytest.mark.parametrize("K", [200, 9 * 320])  # 9 * 320: the longest k-loop of the conv edge cases
def test_tap_rejects_3ulp_move(K):
    _, _, _, ref, terms, k_eff = gemm_case(K=K)
    got = ref.half()
    i = int(ref.abs().argmax())
    flat = got.flatten().clone()
    flat[i] = (flat[i].double() + 3 * ulp16(flat[i].double())).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(flat.view_as(got), ref, terms, k_eff)


def test_tap_rejects_bias_one_column_off():
    a, w, bias, ref, terms, k_eff = gemm_case()
    got = (a.double() @ w.double().t() + torch.roll(bias.double(), 1)).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(got, ref, terms, k_eff)


@pytest.mark.parametrize("kb", [0, 1, 3])
def test_tap_rejects_missing_kblock(kb):
    a, w, bias, ref, terms, k_eff = gemm_case()
    keep = torch.ones(a.shape[1], dtype=torch.bool)
    keep[64 * kb:64 * (kb + 1)] = False
    got = (a.double()[:, keep] @ w.double()[:, keep].t() + bias.double()).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(got, ref, terms, k_eff)


def attn_case(S=40, T=200, d=24, qscale=2.0):
    q = rnd(S, d, seed=4, scale=qscale).half()
    k = rnd(T, d, seed=5).half()
    v = rnd(T, d, seed=6).half()
    p = softmax64((q.double() @ k.double().t()) * d ** -0.5)
    return q, k, v, p


def test_attn_accepts_fp16_p_and_exact():
    _, _, v, p = attn_case()
    v64 = v.double()
    check_attn((p @ v64).half(), p, v64)
    check_attn((p.half().double() @ v64).half(), p, v64)
    check_probs(p.half(), p)
    # an edited row (negative equalizer): signed entries, each rounded to fp16
    ps = p * 10 * torch.where(torch.arange(p.shape[-1]) % 3 == 0, -1.0, 1.0).double()
    check_attn((ps.half().double() @ v64).half(), ps, v64)


def test_attn_rejects_missing_key_block():
    q, k, v, p = attn_case()
    s = (q.double() @ k.double().t()) * q.shape[1] ** -0.5
    s[:, 64:128] = -float("inf")
    got = (softmax64(s) @ v.double()).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_attn(got, p, v.double())


def test_probs_reject_other_normalisation():
    _, _, _, p = attn_case()
    with pytest.raises(AssertionError, match="out of bound"):
        check_probs((p * (1 + 2.0 ** -9)).half(), p)
    # a sum taken without the last key: every probability a little too large
    q = p.clone()
    q[:, :-1] = p[:, :-1] / p[:, :-1].sum(-1, keepdim=True)
    q[:, -1] = 0
    with pytest.raises(AssertionError, match="out of bound"):
        check_probs(q.half(), p)


# ------------------------------------------------------------------------------------------------------- normalisation, steps, masks
def ln_case(M=12, C=64, sigma=1.0, mean=0.5, seed=20):
    x = (rnd(M, C, seed=seed) * sigma + mean).half()
    g, b = 1 + 0.3 * rnd(C, seed=seed + 1), 0.2 * rnd(C, seed=seed + 2)
    return x, g, b


def ln64(x, g, b, eps=1e-5, unbiased=False, eps_outside=False):
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    var = x64.var(-1, unbiased=unbiased, keepdim=True)
    den = var.sqrt() + eps if eps_outside else (var + eps).sqrt()
    return (x64 - mu) / den * g.double() + b.double()


def test_norm_accepts_correct_rounding():
    x, g, b = ln_case()
    ln_check(ln64(x, g, b).half(), x, g, b, 1e-5)
    xg = (rnd(8, 16, 64, seed=30) + rnd(8, 1, 64, seed=31)).half()
    gg, bg = 1 + 0.3 * rnd(64, seed=32), 0.2 * rnd(64, seed=33)
    for fps, silu in [(1, False), (4, True), (8, False)]:
        y = F.group_norm(xg.double().view(8 // fps, fps, 16, 64).permute(0, 3, 1, 2), 8, gg.double(), bg.double(), 1e-5)
        y = y.permute(0, 2, 3, 1).reshape(8, 16, 64)
        gn_check((F.silu(y) if silu else y).half(), xg, gg, bg, 1e-5, 8, fps, silu)


def test_norm_rejects_unbiased_variance():
    x, g, b = ln_case()
    with pytest.raises(AssertionError, match="out of bound"):
        ln_check(ln64(x, g, b, unbiased=True).half(), x, g, b, 1e-5)


def test_norm_rejects_eps_outside_sqrt():
    x, g, b = ln_case(sigma=0.02)  # sigma^2 = 4e-4: eps = 1e-5 outside the root moves rstd by about 1 %
    with pytest.raises(AssertionError, match="out of bound"):
        ln_check(ln64(x, g, b, eps_outside=True).half(), x, g, b, 1e-5)


def test_norm_rejects_per_frame_statistics():
    xg = (rnd(8, 16, 64, seed=30) + 0.5 * rnd(8, 1, 64, seed=31)).half()
    gg, bg = 1 + 0.3 * rnd(64, seed=32), 0.2 * rnd(64, seed=33)
    y = F.group_norm(xg.double().permute(0, 2, 1), 8, gg.double(), bg.double(), 1e-5).permute(0, 2, 1)  # frames_per_stat = 1
    gn_check(y.half(), xg, gg, bg, 1e-5, 8, 1, False)
    with pytest.raises(AssertionError, match="out of bound"):
        gn_check(y.half(), xg, gg, bg, 1e-5, 8, 4, False)


def fma32(a, b, c):
    """fmaf on fp32 tensors: the product is exact in fp64, one rounding of the sum (to fp64, then fp32: a double rounding that cannot
    matter at the size of the errors checked here)."""
    return (a.double() * b.double() + c.double()).float()


@pytest.mark.parametrize("C", [64, 320, 768, 1280])
def test_norm_rejects_fused_shift_on_constant_row(C):
    """The LayerNorm of a constant row is beta exactly.  y = fma(fma(v, rstd, shift), gamma, beta) with shift = fp32(-mean * rstd) carries
    the rounding of shift (2^-24 |mean| rstd, rstd = eps^-1/2 = 316 here) into beta."""
    vals = torch.tensor([-150.0, -37.5, 100.0, 199.0, 0.3, 3.0])
    x = vals[:, None].expand(len(vals), C).half()
    g, b = 1 + 0.3 * rnd(C, seed=40), 0.02 * rnd(C, seed=41)
    ln_check(b.expand(len(vals), C).half(), x, g, b, 1e-5)  # the exact answer passes
    v = x.float()
    inv_c = torch.tensor(1.0 / C, dtype=torch.float32)
    s = v.sum(-1, keepdim=True)
    rstd = (torch.zeros(len(vals), 1) + torch.tensor(1e-5, dtype=torch.float32)).rsqrt()
    shift = (-s * inv_c) * rstd
    y = fma32(fma32(v, rstd.expand_as(v), shift.expand_as(v)), g.expand_as(v), b.expand_as(v))
    with pytest.raises(AssertionError, match="out of bound"):
        ln_check(y.half(), x, g, b, 1e-5)


def test_probs_reject_scale_one_fp16_ulp_off():
    x = (rnd(16, 512, seed=50) * 40).half()
    s = 512 ** -0.5
    p = softmax64(x.double() * s)
    check_probs(p.half(), p)
    with pytest.raises(AssertionError, match="out of bound"):
        check_probs(softmax64(x.double() * s * (1 + 2.0 ** -10)).half(), p)


def mask_maps(Fr=2, heads=4, r=16, seed=60):
    return [torch.softmax(rnd(Fr, heads, r * r, 80, seed=seed + i) * 2, -1).half() for i in range(3)]


def test_mask_rejects_index_off_by_one():
    maps = mask_maps()
    ww = torch.zeros(77)
    ww[[2, 76]] = 1
    h, w = 64, 40
    ratio = blend_mask_ratio(maps, ww, h, w)
    check_mask(ratio.gt(0.5).float(), ratio, 0.5)
    # the same pipeline with the nearest-resize source row one further down
    st = torch.stack([(m[..., :77].double() * ww.double()).sum(-1) for m in maps]).mean((0, 2)).reshape(2, 1, 16, 16)
    pooled = F.max_pool2d(st, 3, 1, 1)[:, 0]
    sy = (nearest_index(16, h) + 1).clamp(max=15)
    sx = nearest_index(16, w)
    mk = pooled[:, sy][:, :, sx]
    shifted = mk / mk.amax((-2, -1), keepdim=True)
    with pytest.raises(AssertionError, match="differ"):
        check_mask(shifted.gt(0.5).float(), ratio, 0.5)


def test_mask_rejects_integer_resize_index():
    """(y * r) / h in integers differs from F.interpolate's floor(y * (float)(r / h)) at r = 16, h = 82; a map that ramps along y with th
    between the two source rows makes that row of the mask differ."""
    r, h = 16, 82
    ramp = torch.arange(r, dtype=torch.float64).repeat_interleave(r) / r  # row y of the r x r grid holds y / r
    maps = [torch.zeros(1, 1, r * r, 80, dtype=torch.float16)]
    maps[0][0, 0, :, 5] = ramp.half()
    ww = torch.zeros(77)
    ww[5] = 1
    ratio = blend_mask_ratio(maps, ww, h, h)
    pooled = F.max_pool2d(ramp.view(1, 1, r, r), 3, 1, 1)[0, 0, :, 0]
    ours = (torch.arange(h) * r // h).clamp(max=r - 1)
    torch_idx = nearest_index(r, h)
    assert torch.equal(torch_idx, F.interpolate(torch.arange(r, dtype=torch.float32).view(1, 1, r), size=h).view(-1).long())
    y = int((ours != torch_idx).nonzero()[0])
    th = 0.5 * (pooled[ours[y]] + pooled[torch_idx[y]]).item() / pooled.max().item()
    mk = pooled[ours][:, None].expand(h, h)[None]
    with pytest.raises(AssertionError, match="differ"):
        check_mask((mk / mk.max()).gt(th).float(), ratio, th)


def test_heatmaps_reject_white_zero_column():
    maps = [torch.softmax(rnd(2, 4, 64, 80, seed=70), -1).half()]
    maps[0][..., 9] = 0
    v = heatmap_values(maps, 77)
    good = v.clamp(max=255).floor().to(torch.uint8)
    check_heatmaps(good, v)
    bad = good.clone()
    bad[:, 9] = 255  # fminf(255, 0/0) on a column whose maximum is 0
    with pytest.raises(AssertionError, match="differ"):
        check_heatmaps(bad, v)


# ------------------------------------------------------------------------------------------------------------ cross-attention edit
def edit_case(kind, kps=77, S=48):
    cur = softmax64(rnd(2, S, kps, seed=90) * 2).half()
    base = softmax64(rnd(2, S, kps, seed=91) * 2).half()
    return cur, base, cross_edit_table(kind, kps)


def with_table(t, **rows):
    """A copy of table t with the named ranges replaced: alpha / eq / a / mapper [80], M [80, 80]."""
    t = t.clone()
    for name, v in rows.items():
        off = dict(alpha=X_ALPHA, eq=X_EQ, a=X_A, mapper=X_MAP, M=X_M)[name]
        v = v.reshape(-1)
        t[off:off + v.numel()] = v
    return t


@pytest.mark.parametrize("kind", ["refine", "replace", "reweight"])
@pytest.mark.parametrize("kps", [77, 16, 80])
def test_edit_accepts_correct_rounding(kind, kps):
    cur, base, t = edit_case(kind, kps)
    ref, terms = cross_edit_ref(cur, base, t, kps)
    check_edit(ref.half(), ref, terms)
    # at alpha = 0 the edit is the current probability, whatever eq
    al = t[X_ALPHA:X_ALPHA + kps]
    assert torch.equal(ref[..., al == 0], cur[..., :kps][..., al == 0].double())


def eq_after_lerp(cur, base, t, kps):
    x, _ = cross_edit_ref(cur, base, with_table(t, eq=torch.ones(80)), kps)
    return x * t[X_EQ:X_EQ + kps].double()


def m_transposed(cur, base, t, kps):
    return cross_edit_ref(cur, base, with_table(t, M=t[X_M:].view(80, 80).t()), kps)[0]


def replace_first_atom(cur, base, t, kps):
    M = t[X_M:].view(80, 80).clone()
    M[64:] = 0
    return cross_edit_ref(cur, base, with_table(t, M=M), kps)[0]


def mapper_minus1_as_0(cur, base, t, kps):
    mp = t[X_MAP:X_MAP + 80]
    return cross_edit_ref(cur, base, with_table(t, mapper=torch.where(mp < 0, torch.zeros_like(mp), mp)), kps)[0]


def alpha_swapped(cur, base, t, kps):
    return cross_edit_ref(cur, base, with_table(t, alpha=1 - t[X_ALPHA:X_ALPHA + 80]), kps)[0]


def refine_lerp_reversed(cur, base, t, kps):
    return cross_edit_ref(cur, base, with_table(t, a=1 - t[X_A:X_A + 80]), kps)[0]


@pytest.mark.parametrize("kind,bug", [("refine", eq_after_lerp), ("replace", eq_after_lerp), ("reweight", eq_after_lerp),
                                      ("replace", m_transposed), ("replace", replace_first_atom), ("refine", mapper_minus1_as_0),
                                      ("refine", alpha_swapped), ("replace", alpha_swapped), ("refine", refine_lerp_reversed)],
                         ids=lambda v: v if isinstance(v, str) else v.__name__)
def test_edit_rejects(kind, bug):
    cur, base, t = edit_case(kind)
    ref, terms = cross_edit_ref(cur, base, t, 77)
    with pytest.raises(AssertionError, match="out of bound"):
        check_edit(bug(cur, base, t, 77).half(), ref, terms)


def test_edit_rejects_3ulp_move():
    cur, base, t = edit_case("replace")
    ref, terms = cross_edit_ref(cur, base, t, 77)
    got = ref.half().flatten().clone()
    i = int(terms.flatten().argmax())  # where the bound is widest
    got[i] = (got[i].double() + 3 * ulp16(got[i].double())).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_edit(got.view_as(ref), ref, terms)


def test_running_sum_rejects_edited_p_and_unrounded_add():
    cur, base, t = edit_case("refine")
    p64 = softmax64(rnd(2, 48, 77, seed=90) * 2)  # cur before its rounding to fp16
    old = (4 + 4 * torch.rand(2, 48, 96, generator=torch.Generator().manual_seed(92))).half()
    pad = torch.zeros(2, 48, 96, dtype=torch.float16)
    pad[..., :77] = cur
    check_running_sum(old + pad, old, cur, 77)
    edited = cross_edit_ref(cur, base, t, 77)[0].half()
    with pytest.raises(AssertionError, match="differs"):
        check_running_sum(old + torch.cat([edited, pad[..., 77:]], -1), old, cur, 77)
    unrounded = old.clone()
    unrounded[..., :77] = (old[..., :77].double() + p64).half()  # the fp32 probability added before its rounding to fp16
    with pytest.raises(AssertionError, match="differs"):
        check_running_sum(unrounded, old, cur, 77)
    touched = old + pad
    touched[..., 80] += 1  # a pad column written
    with pytest.raises(AssertionError, match="pad columns changed"):
        check_running_sum(touched, old, cur, 77)


def test_step_rejects_guidance_on_wrong_half():
    K = 3
    x, eps2, x_inv = rnd(K, 4, 2, 5, 6, seed=80), rnd(2 * K, 4, 2, 5, 6, seed=81), rnd(1, 4, 2, 5, 6, seed=82)
    blends = [((rnd(2, 5, 6, seed=83) > 0).float(), None), None, ((rnd(2, 5, 6, seed=84) > 0).float(), (rnd(2, 5, 6, seed=85) > 0).float())]
    ref, terms = cfg_ddim_ref(x, eps2, 7.5, 0.3, 0.4, x_inv, blends)
    check_step(ref.float(), ref, terms)
    swapped = torch.cat([eps2[K:], eps2[:K]])
    wrong, _ = cfg_ddim_ref(x, swapped, 7.5, 0.3, 0.4, x_inv, blends)
    with pytest.raises(AssertionError, match="out of bound"):
        check_step(wrong.float(), ref, terms)
    inv, inv_terms = ddim_invert_ref(x, eps2[:K], 0.3, 0.4)
    check_step(inv.float(), inv, inv_terms)


# ---------------------------------------------------------------------------------------------------- GroupNorm statistics exchange
def combine_case(world=4, me=1, B=3, F_loc=4, G=5, seed=100):
    """Per-image (sum, sumsq) of every rank with magnitudes spread over 2^-12 .. 2^12, so that any change of the fold order or of the
    rounding points moves some totals."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(world, B * F_loc, G, 2, generator=g) * torch.pow(2.0, torch.randint(-12, 13, (world, B * F_loc, G, 2), generator=g).float())
    v[..., 1] = v[..., 1].abs()
    return v[me].clone(), v


def fold64(acc, F_loc, sets_minor=True, zero_rest=True):
    """Fold the fp64 per-image totals acc [NB, G, 2] over the frames of each set; sets_minor=False reads the images as [F_loc, B]."""
    NB, G, _ = acc.shape
    v = acc.view(NB // F_loc, F_loc, G, 2) if sets_minor else acc.view(F_loc, NB // F_loc, G, 2).transpose(0, 1)
    tot = v[:, 0]
    for f in range(1, F_loc):
        tot = tot + v[:, f]
    out = torch.zeros(NB // F_loc, F_loc, G, 2, dtype=torch.float64) if zero_rest else acc.view(NB // F_loc, F_loc, G, 2).clone()
    out[:, 0] = tot
    return out.view(NB, G, 2)


def rank_sum(own, peers, me, own_times=1, round_each=False):
    acc = own.double() * own_times
    for r in range(peers.shape[0]):
        if r != me:
            acc = acc + peers[r].double()
            if round_each:
                acc = acc.float().double()
    return acc


def test_gn_combine_accepts_kernel_order():
    for world, me, F_loc in [(4, 1, 4), (1, 0, 2), (3, 2, 1)]:
        own, peers = combine_case(world, me, F_loc=F_loc)
        check_gn_combine(fold64(rank_sum(own, peers, me), F_loc), own, peers, me, F_loc)


@pytest.mark.parametrize("bug", ["sets_as_F_by_B", "own_rank_twice", "rest_not_zeroed", "per_rank_fp32_rounding", "fp32_set_total"])
def test_gn_combine_rejects(bug):
    own, peers = combine_case()
    me, F_loc = 1, 4
    if bug == "sets_as_F_by_B":
        got = fold64(rank_sum(own, peers, me), F_loc, sets_minor=False)
    elif bug == "own_rank_twice":
        got = fold64(rank_sum(own, peers, me, own_times=2), F_loc)
    elif bug == "rest_not_zeroed":
        got = fold64(rank_sum(own, peers, me), F_loc, zero_rest=False)
    elif bug == "per_rank_fp32_rounding":
        got = fold64(rank_sum(own, peers, me, round_each=True), F_loc)
    else:
        got = fold64(rank_sum(own, peers, me), F_loc).float().double()
    with pytest.raises(AssertionError, match="are not 0" if bug == "rest_not_zeroed" else "differ from the fp64 replay"):
        check_gn_combine(got, own, peers, me, F_loc)


# ------------------------------------------------------------------------------------------------------------------------ VAE blocks
@pytest.mark.parametrize("stride,asym", [(1, False), (2, False), (2, True)])
def test_conv_rows_ref_matches_full_conv(stride, asym):
    """The row-gathered conv reference of the sampled VAE checks equals the full fp64 conv on the rows it is asked for."""
    x, w9 = rnd(2, 6, 10, 16, seed=110).half(), rnd(9, 5, 16, seed=111, scale=0.1).half()
    bias, res = rnd(5, seed=112), rnd(2 * (6 // stride) * (10 // stride), 5, seed=113).half()
    ref, terms = conv3x3_ref(x, w9, stride, asym, bias=bias, residuals=(res,))
    rows = torch.tensor([0, 3, 7, ref.shape[0] - 1, ref.shape[0] // 2])
    r2, t2 = conv3x3_rows_ref(x, w9, rows, stride, asym, bias=bias, residuals=(res[rows],))
    assert torch.allclose(r2, ref[rows], rtol=1e-13, atol=1e-13) and torch.allclose(t2, terms[rows], rtol=1e-13, atol=1e-13)


VAE_SMALL = dict(in_channels=3, out_channels=3, block_out_channels=(32, 64), layers_per_block=1, latent_channels=4, norm_num_groups=8)
to16 = lambda t: t.half().double()  # noqa: E731  (an fp16 run emulated in fp64: one rounding after every op)


def vae_block_inputs():
    """Small NCHW fp16 inputs of every block; the resnet input's first group (4 channels) is near-constant (sigma 1e-3: var ~ eps)."""
    x = rnd(1, 32, 8, 8, seed=120).half()
    x[:, :4] = (1e-3 * rnd(1, 4, 8, 8, seed=121)).half()
    return dict(resnet_eps=("encoder.down_blocks.1.resnets.0", "resnet", rnd(1, 32, 8, 8, seed=122).half()),
                resnet_const=("encoder.down_blocks.0.resnets.0", "resnet", x),
                attn=("encoder.mid_block.attentions.0", "attn", rnd(1, 64, 8, 8, seed=123).half()),
                down=("encoder.down_blocks.0.downsamplers.0", "down", rnd(1, 32, 8, 8, seed=124).half()),
                up=("decoder.up_blocks.0.upsamplers.0", "up", rnd(1, 64, 4, 4, seed=125).half()),
                encoder_in=(None, "encoder_in", (2 * torch.rand(1, 3, 8, 8, generator=torch.Generator().manual_seed(126)) - 1).half()),
                encoder_out=(None, "encoder_out", rnd(1, 64, 4, 4, seed=127).half()),
                decoder_in=(None, "decoder_in", (0.8 * rnd(1, 4, 4, 4, seed=128)).half()),
                decoder_out=(None, "decoder_out", rnd(1, 32, 8, 8, seed=129).half()))


def run_block(sd, block, rnd16=False, bug=None, probs=None):
    name, method, x = vae_block_inputs()[block]
    r = VaeBlocks64(sd, torch.float64, "cpu", groups=VAE_SMALL["norm_num_groups"], rnd=to16 if rnd16 else None, bug=bug)
    args = (x.double(),) if name is None else (name, x.double())
    return getattr(r, method)(*args, **({} if probs is None else dict(probs_out=probs)))


@pytest.fixture(scope="module")
def vae_sd():
    return {k: v.double() for k, v in vae_block_state_dict(vae_param_spec(VAE_SMALL), seed=7).items()}


def test_block_check_accepts_fp16_and_fp32(vae_sd):
    for block in vae_block_inputs():
        probs = [] if block == "attn" else None
        ref = run_block(vae_sd, block, probs=probs)
        o16 = run_block(vae_sd, block, rnd16=True)
        check_block(o16, ref, o16)
        check_block(ref.half(), ref, o16)
        check_block(ref.float(), ref, o16)
        if probs:  # the attention is peaked, so that what P selects matters
            assert probs[0].amax(-1).median().item() > 0.5


@pytest.mark.parametrize("block,bug", [("attn", "qk_swapped"), ("attn", "scale_1_over_c"), ("attn", "scale_c_quarter"),
                                       ("attn", "softmax_over_queries"), ("attn", "vbias_dropped"), ("attn", "vbias_unnormalised"),
                                       ("encoder_out", "quant_wq_transposed"), ("encoder_out", "conv_out_col_offset"),
                                       ("decoder_out", "conv_out_col_offset"), ("down", "down_pad_left_top"),
                                       ("resnet_const", "gn_eps_1e-5"), ("up", "upsample_index_off_by_one")])
def test_block_check_rejects(vae_sd, block, bug):
    ref = run_block(vae_sd, block)
    o16 = run_block(vae_sd, block, rnd16=True)
    with pytest.raises(AssertionError, match="fp16 floor"):
        check_block(run_block(vae_sd, block, rnd16=True, bug=bug), ref, o16)
