"""Edge cases of the HBM-bound kernels of fz_elem.cu against fp64 references built from the same fp16 / fp32 inputs (tests/_ref64.py).

Code path                                                          reached by
-----------------------------------------------------------------  ----------------------------------------------------------------
gn_geometry: 1 slot (TX = 8 / 40 / 240, TY = 32 / 6 / 1, idle      test_groupnorm_geometry
  threads at C = 320), 2 slots (C = 2560), 4 slots (C = 4160,
  TX = 130; C = 8192, 64 KiB of statistics shared memory through
  cudaFuncSetAttribute), cpg = 1 (64 groups), one group
statistics chunks: HW = 1 and 3 (< TY), 4096 (256 chunks folded    test_groupnorm_chunks
  by the last CTA), 4099 (ragged last chunk)
frames_per_stat in {1, 2, 8, NB}, SiLU on and off                  test_groupnorm_frames_per_stat
shared workspace: arrival counters back at zero after every        test_groupnorm_workspace_interleaved
  call, repeated calls bitwise equal
fz_groupnorm_stats_f16 + fz_groupnorm_apply_f16 with count_frames  test_groupnorm_split_ranks
  > frames_per_stat (2 and 4 emulated ranks), batched GroupNorm    test_groupnorm_batched
  at K = 8 items; fz_groupnorm_apply_sums64_f16 with fp64 set     test_groupnorm_apply_fp64_sums
  totals that fp32 cannot hold (constant groups, 12 frames)
mean / sigma in {0, 4, 16, 64, 256}, constant and near-constant     test_groupnorm_dc_offset, test_layernorm_dc_offset,
  groups and rows (the fused-shift and E[x^2] - mu^2 paths);         test_groupnorm_constant_groups
  constant groups with SiLU, 2 slots, split statistics + apply
LayerNorm NV = 1 (31 idle lanes), partial second vector, CLIP      test_layernorm_shapes, test_layernorm_refuses_wide_rows
  width, NV = 8; M tails of the ROWS = 4 variant; C = 2056 refused
row softmax: n in {8, 72, 4096}, ld > n (padding untouched),       test_softmax_rows, test_softmax_rows_extremes,
  uniform / one-hot rows, logits near +-60000; n % 8 refused         test_softmax_rows_refuses_ragged_n
blend mask: r in {8, 16, 32} x ragged output sizes (nearest index  test_blend_mask, test_blend_mask_all_zero
  of F.interpolate), fp16 / fp32 maps, 1-8 layers, token 76, a
  map whose maximum is 0
cross heat maps: res in {8, 16, 32}, ldm = 80, an all-zero token   test_cross_heatmaps
  column, fp16 / fp32 maps
DDIM inversion step; CFG + DDIM over K in {1, 3, 8} items, n_item  test_ddim_invert, test_cfg_ddim
  not a multiple of 256, blend and plain items mixed, mask_b on
  some items, alpha-bar near 0 and 1
conv_out temporal tail: F in {1, 2, 8}, Co = 4 in ldy = 8, LoRA    test_out_temporal, test_out_temporal_refusals
  rank 1 / 4, full weight, identity; Co = 9 and rank 5 refused
time embedding: rowvec_linear K in {2, 320, 1280} (+-90 SiLU       test_rowvec_linear, test_timestep_sinusoid
  inputs, odd K refused), sinusoid t in {0, 1, 999}, flip, shift
CLIP helpers: embed_tokens (ids 0 and 49407), quick_gelu past one  test_embed_tokens, test_quick_gelu
  grid-stride pass
exact layout kernels: upsample (odd H != W), concat (Ca != Cb),    test_layout_kernels_exact
  latent im2col (Cl = 4, 7)
"""
import pytest
import torch
import torch.nn.functional as F

from _ref64 import (check_bound, check_heatmaps, check_mask, check_probs, check_step, check_tap, cfg_ddim_ref, ddim_invert_ref, f32,
                    gn_check, heatmap_values, blend_mask_ratio, ln_check, out_temporal_ref, quick_gelu_ref, rowvec_ref, sinusoid_ref,
                    softmax64, C_DC, C_STEP)

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from fatezero_b200 import ops

dev = "cuda"


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def affine(C, seed=0):
    return 1 + 0.3 * rnd(C, seed=seed), 0.2 * rnd(C, seed=seed + 1)


# ------------------------------------------------------------------------------------------------------------------------- GroupNorm
def gn_geometry(C, HW, NB, ctas_per_sm):
    """Host planner of fz_elem.cu (slots, TX, TY, px_per_cta, chunks), to state which geometry each case reaches."""
    CV = C // 8
    s = (CV + 255) // 256
    while CV % s or s == 3:
        s += 1
    TX = CV // s
    TY = 256 // TX
    want = max(1, ctas_per_sm * torch.cuda.get_device_properties(0).multi_processor_count // max(1, NB))
    ppc = max(TY, (HW + want - 1) // want)
    return dict(slots=s, TX=TX, TY=TY, ppc=ppc, chunks=(HW + ppc - 1) // ppc, smem=2 * TY * C * 4)


def counters():
    """The per-image arrival counters of the GroupNorm workspace (byte offset 960 KiB)."""
    ws = next(iter(ops._gn_ws.values()))
    off = 960 * 1024 // 4
    return ws.view(torch.int32)[off:off + 256]


def run_gn(NB, HW, C, G, fps, silu, x=None, seed=0, **kw):
    x = rnd(NB, HW, C, seed=seed).half() if x is None else x
    g, b = affine(C, seed + 1)
    out = ops.groupnorm(x, g, b, 1e-5, G, fps, silu, **kw)
    return x, g, b, out


# C, groups, HW, NB, fps, silu, expected (slots, TX, TY) of the statistics pass
GEOMETRY_CASES = [
    (64, 64, 1024, 2, 2, False, (1, 8, 32)),
    (320, 32, 576, 4, 4, True, (1, 40, 6)),
    (1920, 32, 64, 2, 1, True, (1, 240, 1)),
    (2560, 32, 64, 2, 2, False, (2, 160, 1)),
    (4160, 32, 48, 2, 1, True, (4, 130, 1)),
    (8192, 32, 40, 2, 2, False, (4, 256, 1)),
    (320, 1, 256, 2, 2, True, (1, 40, 6)),
]


@pytest.mark.parametrize("C,G,HW,NB,fps,silu,geo", GEOMETRY_CASES, ids=lambda v: str(v))
def test_groupnorm_geometry(C, G, HW, NB, fps, silu, geo, report):
    plan = gn_geometry(C, HW, NB, 2)
    assert (plan["slots"], plan["TX"], plan["TY"]) == geo
    if C == 8192:
        assert plan["smem"] > 48 * 1024
    x, g, b, out = run_gn(NB, HW, C, G, fps, silu, seed=1)
    gn_check(out, x, g, b, 1e-5, G, fps, silu, report, f"gn_geo_C{C}_G{G}")
    assert torch.all(counters() == 0)


@pytest.mark.parametrize("HW", [1, 3, 4096, 4099])
def test_groupnorm_chunks(HW, report):
    plan = gn_geometry(320, HW, 1, 2)
    if HW == 4096:
        assert plan["chunks"] == 256 or torch.cuda.get_device_properties(0).multi_processor_count != 132
    if HW == 4099:
        assert HW % plan["ppc"] != 0
    x, g, b, out = run_gn(1, HW, 320, 32, 1, True, seed=2)
    gn_check(out, x, g, b, 1e-5, 32, 1, True, report, f"gn_chunks_HW{HW}_chunks{plan['chunks']}")


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("fps", [1, 2, 8, 16])
def test_groupnorm_frames_per_stat(fps, silu, report):
    NB, HW, C = 16, 256, 640
    x = (rnd(NB, HW, C, seed=3) + rnd(NB, 1, C, seed=4)).half()  # per-image offsets: per-frame and joint statistics differ
    x, g, b, out = run_gn(NB, HW, C, 32, fps, silu, x=x, seed=3)
    gn_check(out, x, g, b, 1e-5, 32, fps, silu, report, f"gn_fps{fps}_silu{int(silu)}")


def test_groupnorm_workspace_interleaved(report):
    """Calls of different shapes share the 1 MiB workspace: each leaves the arrival counters at zero, and repeating a call gives the
    same bits (the fold order is fixed, not arrival order)."""
    shapes = [(8, 4096, 320, 32, 8), (2, 3, 1920, 32, 1), (16, 256, 1280, 32, 8), (1, 4099, 320, 32, 1), (4, 64, 8192, 32, 2)]
    first = {}
    for rep in range(2):
        for i, (NB, HW, C, G, fps) in enumerate(shapes):
            x, g, b, out = run_gn(NB, HW, C, G, fps, True, seed=10 + i)
            torch.cuda.synchronize()
            assert torch.all(counters() == 0), f"arrival counters left non-zero by shape {i}"
            if rep == 0:
                first[i] = out.clone()
                gn_check(out, x, g, b, 1e-5, G, fps, True, report, f"gn_ws_{NB}x{HW}x{C}")
            else:
                assert torch.equal(out, first[i]), f"shape {i}: repeated call not bitwise equal"
    sums = ops.groupnorm_stats(rnd(2, 64, 320, seed=20).half(), 32)
    torch.cuda.synchronize()
    assert torch.all(counters() == 0) and torch.isfinite(sums).all()


@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_split_ranks(R, silu, report):
    """Frame sharding on one GPU: each emulated rank computes the statistics of its frames, the per-image sums are added over the ranks
    in fp32 (the all-reduce), and each rank applies with count_frames = F.  Compared with fp64 GroupNorm over the whole clip."""
    B, Fr, HW, C, G = 2, 8, 256, 320, 32
    Fl = Fr // R
    x = (rnd(B, Fr, HW, C, seed=30) * 1.5 + rnd(B, Fr, 1, C, seed=31)).half()
    g, b = affine(C, 32)
    parts = [x[:, r * Fl:(r + 1) * Fl].reshape(B * Fl, HW, C).contiguous() for r in range(R)]
    stats = [ops.groupnorm_stats(p, G).clone() for p in parts]  # the sums live in the shared workspace
    total = stats[0].clone()
    for s in stats[1:]:
        total += s
    outs = [ops.groupnorm_apply(p, g, b, 1e-5, G, Fl, Fr, silu, total) for p in parts]
    got = torch.stack([o.view(B, Fl, HW, C) for o in outs], 1).reshape(B * Fr, HW, C)  # [B, R, Fl] -> frames in clip order
    gn_check(got, x.reshape(B * Fr, HW, C), g, b, 1e-5, G, Fr, silu, report, f"gn_split_R{R}_silu{int(silu)}")


def test_groupnorm_batched(report):
    K, Fr, HW, C, G = 8, 2, 256, 640, 32
    x = (rnd(K * Fr, HW, C, seed=40) + rnd(K * Fr, 1, C, seed=41)).half()
    x, g, b, out = run_gn(K * Fr, HW, C, G, Fr, True, x=x, seed=40, images_per_item=Fr)
    gn_check(out, x, g, b, 1e-5, G, Fr, True, report, "gn_batched_K8")


DC_CASES = [0, 4, 16, 64, 256, "const", "near_const"]


def dc_input(shape, mode, seed, set_shape):
    """fp32 values with mean / sigma = mode (sigma = 1; 0.5 at 256, to keep the fp16 spacing below sigma / 2), or, per statistics set
    (set_shape broadcasts over it), a constant 0.3, 3 or -150, plus sigma = 1e-3 noise for "near_const" (rounded away at -150)."""
    z = rnd(*shape, seed=seed)
    if mode in ("const", "near_const"):
        pick = torch.randint(0, 3, set_shape, generator=torch.Generator().manual_seed(seed)).to(dev)
        base = torch.tensor([0.3, 3.0, -150.0], device=dev)[pick].expand(shape)
        return base + (1e-3 * z if mode == "near_const" else 0.0)
    sigma = 0.5 if mode == 256 else 1.0
    return mode * sigma + sigma * z


@pytest.mark.parametrize("mode", DC_CASES, ids=str)
def test_groupnorm_dc_offset(mode, report):
    """Strict bound up to mean/sigma = 64 and on exactly constant groups (their fp32 sums are exact, so the output must be beta to within
    the final rounding: a fused shift beta - mean * rstd * gamma misses it by thousands of ulps at mean = -150).  At mean/sigma = 256 and on
    near-constant groups the E[x^2] - mu^2 statistics lose the variance to cancellation (DESIGN.md, known limits): the strict ratio is
    recorded and the bound with the c_dc (mu/sigma)^2 term asserted."""
    NB, HW, C, G = 8, 256, 320, 32
    x = dc_input((NB, HW, G, C // G), mode, 50, (1, 1, G, 1)).reshape(NB, HW, C).half()
    g, b = affine(C, 52)
    b = b * 0.05  # small beta: the exact answer of a constant group is beta, whose ulp is small
    out = ops.groupnorm(x, g, b, 1e-5, G, NB, False)
    loose = mode in (256, "near_const")
    gn_check(out, x, g, b, 1e-5, G, NB, False, report, f"gn_dc_{mode}", c_dc=C_DC if loose else None)


@pytest.mark.parametrize("C", [320, 2560])
def test_groupnorm_constant_groups(C, report):
    """Constant groups (0.3, 3, -150) through the one-call path with SiLU and through split statistics + apply (two emulated ranks):
    the output is silu(beta) to within the final rounding, under the strict bound."""
    NB, HW, G = 4, 64, 32
    x = dc_input((NB, HW, G, C // G), "const", 55, (1, 1, G, 1)).reshape(NB, HW, C).half()
    g, b = affine(C, 56)
    b = b * 0.05
    out = ops.groupnorm(x, g, b, 1e-5, G, NB, True)
    gn_check(out, x, g, b, 1e-5, G, NB, True, report, f"gn_const_C{C}_silu")
    parts = [x[r * 2:(r + 1) * 2].contiguous() for r in range(2)]
    stats = [ops.groupnorm_stats(p, G).clone() for p in parts]
    outs = [ops.groupnorm_apply(p, g, b, 1e-5, G, 2, NB, False, stats[0] + stats[1]) for p in parts]
    gn_check(torch.cat(outs), x, g, b, 1e-5, G, NB, False, report, f"gn_const_C{C}_split")


@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_apply_fp64_sums(silu, report):
    """The apply of the frame-sharded GroupNorm with fp64 set totals (what fz_gn_combine leaves): constant groups of 0.3 (fp16 1229 / 4096)
    over C / G * HW * F = 10 * 1023 * 12 elements, whose per-image sums are exact in fp32 but whose set total needs more than 24 bits.
    Four emulated ranks of 3 frames each; the total sits in the first image of each set, the other images hold 0.  Strict bound."""
    B, Fr, HW, C, G, R = 2, 12, 1023, 320, 32, 4
    Fl = Fr // R
    x = dc_input((B, Fr, HW, G, C // G), "const", 57, (1, 1, 1, G, 1)).reshape(B, Fr, HW, C).half()
    g, b = affine(C, 58)
    b = b * 0.05
    parts = [x[:, r * Fl:(r + 1) * Fl].reshape(B * Fl, HW, C).contiguous() for r in range(R)]
    stats = [ops.groupnorm_stats(p, G).double().view(B, Fl, G, 2) for p in parts]
    totals = torch.zeros(B, Fl, G, 2, dtype=torch.float64, device=dev)
    totals[:, 0] = sum(s.sum(1) for s in stats)
    outs = [ops.groupnorm_apply(p, g, b, 1e-5, G, Fl, Fr, silu, totals.view(B * Fl, G, 2)) for p in parts]
    got = torch.stack([o.view(B, Fl, HW, C) for o in outs], 1).reshape(B * Fr, HW, C)
    assert totals[:, 0].float().double().ne(totals[:, 0]).any(), "no set total is inexact in fp32: the case no longer tests fp64 sums"
    gn_check(got, x.reshape(B * Fr, HW, C), g, b, 1e-5, G, Fr, silu, report, f"gn_apply_fp64_silu{int(silu)}")


@pytest.mark.parametrize("mode", DC_CASES, ids=str)
@pytest.mark.parametrize("C", [320, 768])
def test_layernorm_dc_offset(C, mode, report):
    M = 77
    x = dc_input((M, C), mode, 60, (M, 1)).half()
    g, b = affine(C, 61)
    b = b * 0.05
    ln_check(ops.layernorm(x, g, b), x, g, b, 1e-5, report, f"ln_dc_{mode}_C{C}")


# ------------------------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("M", [1, 3, 77, 4097])
@pytest.mark.parametrize("C", [8, 64, 264, 768, 2048])
def test_layernorm_shapes(C, M, report):
    x = (rnd(M, C, seed=70) * 2 + 0.5).half()
    g, b = affine(C, 71)
    ln_check(ops.layernorm(x, g, b), x, g, b, 1e-5, report, f"ln_C{C}_M{M}")


def test_layernorm_refuses_wide_rows():
    x = torch.zeros(4, 2056, dtype=torch.float16, device=dev)
    g = torch.ones(2056, device=dev)
    with pytest.raises(RuntimeError, match="C=2056"):
        ops.layernorm(x, g, g)


# --------------------------------------------------------------------------------------------------------------------------- softmax
@pytest.mark.parametrize("rows", [1, 9, 4097])
@pytest.mark.parametrize("n", [8, 72, 4096])
def test_softmax_rows(n, rows, report):
    ld = n + 24
    buf = (rnd(rows, ld, seed=80) * 4).half()
    keep = buf.clone()
    scale = 512 ** -0.5
    p = softmax64(buf[:, :n].double() * f32(scale))
    ops.softmax_rows_(buf[:, :n], scale)
    check_probs(buf[:, :n], p, report, f"softmax_n{n}_rows{rows}")
    assert torch.equal(buf[:, n:], keep[:, n:]), "padding columns written"


def test_softmax_rows_extremes(report):
    n, scale = 512, 512 ** -0.5
    rows = torch.zeros(6, n, dtype=torch.float16, device=dev)
    rows[0] = 1.5                                        # uniform
    rows[1, 17] = 60000.0                                # one-hot at the fp16 range
    rows[2] = -60000.0
    rows[2, 300] = -59000.0                              # all very negative
    rows[3] = (rnd(n, seed=81) * 60000).clamp(-65000, 65000).half()
    rows[4] = 60000.0                                    # uniform at the top of the range
    rows[5] = torch.linspace(-60000, 60000, n, device=dev).half()
    p = softmax64(rows.double() * f32(scale))
    ops.softmax_rows_(rows, scale)
    check_probs(rows, p, report, "softmax_extremes")


def test_softmax_rows_refuses_ragged_n():
    with pytest.raises(RuntimeError, match="multiples of 8"):
        ops.softmax_rows_(torch.zeros(4, 80, dtype=torch.float16, device=dev)[:, :76], 0.1)


# ------------------------------------------------------------------------------------------------------------------------ blend mask
def attn_maps(Fr, heads, r, ldm, seed, dtype=torch.float16):
    return torch.softmax(rnd(Fr, heads, r * r, ldm, seed=seed) * 2, -1).to(dtype)


@pytest.mark.parametrize("hw", [(64, 64), (64, 40), (82, 94), (328, 16)], ids=str)
@pytest.mark.parametrize("r", [8, 16, 32])
def test_blend_mask(r, hw, report):
    h, w = hw
    Fr, heads = 2, 8
    cases = [(1, torch.float16, 0.3), (5, torch.float16, 0.6), (8, torch.float32, 0.5)]
    for n_maps, dtype, th in cases:
        maps = [attn_maps(Fr, heads, r, 80, 90 + i + r, dtype) * (n_maps if dtype == torch.float32 else 1) for i in range(n_maps)]
        ww = torch.zeros(77)
        ww[[2, 5, 76]] = 1
        got = ops.blend_mask(maps, ww, th, h, w)
        check_mask(got, blend_mask_ratio(maps, ww, h, w), f32(th), report, f"mask_r{r}_{h}x{w}_L{n_maps}_{str(dtype)[6:]}")


def test_blend_mask_all_zero(report):
    maps = [attn_maps(2, 8, 16, 80, 95)]
    maps[0][1] = 0  # frame 1: every map entry zero, so its maximum is 0 and ratio 0/0 -> no pixel passes
    ww = torch.zeros(77)
    ww[3] = 1
    got = ops.blend_mask(maps, ww, 0.3, 64, 64)
    assert torch.all(got[1] == 0)
    check_mask(got, blend_mask_ratio(maps, ww, 64, 64), f32(0.3), report, "mask_all_zero_frame")


# ------------------------------------------------------------------------------------------------------------------------- heat maps
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("res", [8, 16, 32])
def test_cross_heatmaps(res, dtype, report):
    Fr, heads, ldm, ntok = 2, 8, 80, 77
    maps = [attn_maps(Fr, heads, res, ldm, 100 + i + res, dtype) * (3 if dtype == torch.float32 else 1) for i in range(3)]
    for m in maps:
        m[..., 40] = 0  # token 40: an all-zero column, whose heat map is black
        m[..., ntok:] = 7  # beyond ntok: never read
    got = ops.cross_heatmaps(maps, ntok).view(Fr, ntok, res * res)
    assert torch.all(got[:, 40] == 0)
    check_heatmaps(got, heatmap_values(maps, ntok), report, f"heat_r{res}_{str(dtype)[6:]}")


# ------------------------------------------------------------------------------------------------------------------------ DDIM steps
@pytest.mark.parametrize("a_prev,a_next", [(0.9991, 0.9985), (0.5, 0.4), (0.0047, 0.0098)])
def test_ddim_invert(a_prev, a_next, report):
    x, e = rnd(2, 4, 3, 13, 11, seed=110), rnd(2, 4, 3, 13, 11, seed=111)
    ref, terms = ddim_invert_ref(x, e, a_prev, a_next)
    got = x.clone()
    ops.ddim_invert_step(got, e, a_prev, a_next)
    check_step(got, ref, terms, report, f"ddim_inv_{a_prev}")


@pytest.mark.parametrize("a_t,a_prev", [(0.0047, 0.0098), (0.9985, 0.9991)])
@pytest.mark.parametrize("K", [1, 3, 8])
def test_cfg_ddim(K, a_t, a_prev, report):
    Fr, H, W = 3, 13, 11  # n_item = 4 * 429 = 1716, not a multiple of 256
    x = rnd(K, 4, Fr, H, W, seed=120)
    eps2 = rnd(2 * K, 4, Fr, H, W, seed=121)
    x_inv = rnd(1, 4, Fr, H, W, seed=122)
    blends = []
    for k in range(K):
        if k % 3 == 1:
            blends.append(None)
            continue
        ma = (rnd(Fr, H, W, seed=123 + k) > 0).float()
        mb = (rnd(Fr, H, W, seed=140 + k) > 0.5).float() if k % 2 == 0 else None
        blends.append((ma, mb))
    ref, terms = cfg_ddim_ref(x, eps2, 7.5, a_t, a_prev, x_inv, blends)
    got = x.clone()
    if K == 1:
        bl = blends[0]
        ops.cfg_ddim_step(got, eps2, 7.5, a_t, a_prev, x_inv=x_inv, mask_a=bl[0], mask_b=bl[1], apply_blend=True)
    else:
        ops.cfg_ddim_step_batched(got, eps2, 7.5, a_t, a_prev, x_inv=x_inv,
                                  blends=[None if bl is None else dict(mask_a=bl[0], mask_b=bl[1], apply_blend=True) for bl in blends])
    check_step(got, ref, terms, report, f"cfg_ddim_K{K}_a{a_t}")


# ------------------------------------------------------------------------------------------------------------------ conv_out temporal
@pytest.mark.parametrize("path", ["lora1", "lora4", "full", "identity"])
@pytest.mark.parametrize("Fr", [1, 2, 8])
def test_out_temporal(Fr, path, report):
    B, Co, H, W = 2, 4, 5, 7
    y = rnd(B * Fr * H * W, 8, seed=150).half()  # ldy = 8, Co = 4 valid columns
    kw = {}
    if path.startswith("lora"):
        R = int(path[4:])
        kw = dict(down=(rnd(R, Co, 3, seed=151) * 0.5).contiguous(), up=(rnd(Co, R, 3, seed=152) * 0.5).contiguous())
    elif path == "full":
        kw = dict(w_full=(rnd(Co, Co, 3, seed=153) * 0.5).contiguous(), b_full=rnd(Co, seed=154))
    got = ops.out_temporal(y, B, Co, Fr, H, W, **kw)
    ref, terms, fixed = out_temporal_ref(y, B, Co, Fr, H * W, **kw)
    got = got.view(B, Co, Fr, H * W)
    if path == "identity":
        assert torch.equal(got.double(), ref)
    else:
        check_tap(got, ref, terms, 1, report, f"out_temporal_{path}_F{Fr}", k_ulp=0.0, c=C_STEP, fixed=fixed)


def test_out_temporal_refusals():
    y = torch.zeros(2 * 4, 16, dtype=torch.float16, device=dev)
    with pytest.raises(RuntimeError, match="fz_out_temporal"):
        ops.out_temporal(y, 1, 9, 2, 2, 2)
    with pytest.raises(RuntimeError, match="fz_out_temporal"):
        ops.out_temporal(y, 1, 4, 2, 2, 2, down=torch.zeros(5, 4, 3, device=dev), up=torch.zeros(4, 5, 3, device=dev))


# ---------------------------------------------------------------------------------------------------------------- time embedding
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("K", [2, 320, 1280])
def test_rowvec_linear(K, silu, report):
    N = 13
    x = rnd(K, seed=160) * 3
    x[0], x[-1] = 90.0, -90.0
    w = rnd(N, K, seed=161, scale=K ** -0.5).half()
    bias = rnd(N, seed=162) if K != 320 else None
    got = ops.rowvec_linear(x, w, bias, silu)
    ref, terms, fixed = rowvec_ref(x, w, bias, silu)
    check_tap(got, ref, terms, K + 1, report, f"rowvec_K{K}_silu{int(silu)}", k_ulp=0.0, fixed=fixed)


def test_rowvec_linear_refuses_odd_k():
    with pytest.raises(RuntimeError, match="fz_rowvec_linear"):
        ops.rowvec_linear(torch.zeros(5, device=dev), torch.zeros(3, 5, dtype=torch.float16, device=dev), None, False)


@pytest.mark.parametrize("shift", [0.0, 1.0])
@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("t", [0.0, 1.0, 999.0])
def test_timestep_sinusoid(t, flip, shift, report):
    got = ops.timestep_sinusoid(t, 320, flip, shift, dev)
    ref, terms = sinusoid_ref(t, 320, flip, shift)
    check_step(got, ref.to(dev), terms.to(dev), report, f"sinusoid_t{int(t)}_flip{int(flip)}_shift{int(shift)}", c=2.0)


# ------------------------------------------------------------------------------------------------------------------------ CLIP helpers
def test_embed_tokens():
    V, L, C = 49408, 77, 768
    tok = rnd(V, C, seed=170) * 0.02
    pos = rnd(L, C, seed=171) * 0.01
    ids = torch.randint(0, V, (2, L), generator=torch.Generator().manual_seed(172)).to(dev)
    ids[0, 0], ids[0, -1], ids[1, 5] = 0, V - 1, V - 1
    got = ops.embed_tokens(tok, pos, ids)
    want = (tok[ids.reshape(-1)] + pos.repeat(2, 1)).half()  # one fp32 add, one rounding
    assert torch.equal(got, want)


@pytest.mark.parametrize("n", [1, 7, 300000])
def test_quick_gelu(n, report):
    x = (rnd(n, seed=180) * 4).half()
    x[0] = -10.0
    ref, bound = quick_gelu_ref(x)
    got = ops.quick_gelu_(x.clone())
    check_bound(got, ref, bound, report, f"quick_gelu_n{n}")


# ---------------------------------------------------------------------------------------------------------------- layout kernels
@pytest.mark.parametrize("Cl", [4, 7])
def test_layout_kernels_exact(Cl):
    x = rnd(3, 7, 5, 24, seed=190).half()  # odd H != W
    up = ops.upsample2x(x)
    assert torch.equal(up, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    a, b = rnd(3, 11, 40, seed=191).half(), rnd(3, 11, 16, seed=192).half()
    assert torch.equal(ops.concat_channels(a, b), torch.cat([a, b], -1))
    B, Fr, H, W = 2, 3, 5, 6
    lat = rnd(B, Cl, Fr, H, W, seed=193)
    cols = ops.im2col_latents(lat)
    xp = F.pad(lat.permute(0, 2, 3, 4, 1).reshape(B * Fr, H, W, Cl), (0, 0, 1, 1, 1, 1))  # [BF, H+2, W+2, Cl]
    taps = torch.stack([xp[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], 3)  # [BF, H, W, 9, Cl]
    want = torch.zeros(B * Fr * H * W, 64, device=dev)
    want[:, :9 * Cl] = taps.reshape(-1, 9 * Cl)
    assert torch.equal(cols, want.half())
