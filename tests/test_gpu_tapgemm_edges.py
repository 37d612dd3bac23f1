"""Edge cases of the wgmma tap-GEMM (fz_gemm.cu) against fp64 references built from the exact fp16 / fp32 inputs (tests/_ref64.py).

BLOCK_N is pinned with force_bn, so the instantiations under test do not depend on the SM count.  Every case also runs twice and must be
bitwise reproducible (there is no split-K).

Code path                                                          reached by
-----------------------------------------------------------------  ----------------------------------------------------------------
every BLOCK_N (16, 32, 64, 128, 160, 256) x {none, bias,           test_gemm_grid (30 cases: M in {1, 63, 64, 65, 129}, odd N, N < 8,
  bias + group_bias (group boundary inside a tile), folded           N not a multiple of BLOCK_N, K in {8, 72, 64 (kStages + 3) + 8},
  residual, epilogue-path residual}                                  odd ldo -> pair_ok off)
epilogue-path residual: odd ldr / 2-byte-offset view               test_gemm_grid "res_epi" cases, test_gemm_two_residuals[*-epi]
two folded skip tensors (n_res = 2, resnet shortcut + LoRA)         test_gemm_two_residuals[*-fold]
CTAs that run several tiles (ring phase carried across tiles)      test_gemm_many_tiles
V^T epilogue: vt_ld > S, bias on V columns, tiles spanning two      test_gemm_vt
  (frame, batch) rows, vt_col_start inside a BLOCK_N tile
GEGLU at every packed width (BLOCK_N 256, 160, 128, 64, 32)        test_geglu
GEGLU + residual / group_bias / V^T refused on the host             test_geglu_refuses_other_terms
conv3x3 s1: 25-row tile (warpgroup 1 idle), Ho % bh adjustment,     test_conv3x3_s1
  several images per tile, 64x96, 128-pixel row segments (W 256),
  96- and 80-pixel row segments (W 192, 320, 576: VAE widths that
  are not multiples of 128), Cin in {8, 72, 320}, every BLOCK_N,
  bias + group_bias + residual
conv3x3 s2: symmetric and asymmetric (VAE downsample) padding,      test_conv3x3_s2
  odd output size, Cin not a multiple of 64 (c0 walks into the
  next pixel's channels, cancelled by the zero-filled W columns),
  256-, 192- and 288-wide outputs (128- and 96-pixel segments)
output widths without a divisor in [8, 128] refused on the host     test_conv3x3_refuses_width
tconv3: F in {1, 2, 3, 5, 16, 24}, several frames per tile with     test_tconv3
  F % bf adjustment, 100-pixel box (HW 200), 1-row tiles (HW 131),
  bias + residual + residual2 + group_bias (the LoRA path)
tconv3 halo (frame-sharded) with non-zero neighbour frames          test_tconv3_halo
"""
import ctypes as C

import pytest
import torch

from _ref64 import check_tap, conv3x3_ref, gemm_ref, tconv3_ref

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from fatezero_b200 import _lib, ops

dev = "cuda"
BLOCK_NS = [16, 32, 64, 128, 160, 256]
K_STAGES = {256: 4, 160: 6, 128: 7, 64: 8, 32: 8, 16: 8}  # TapGemmCfg<BLOCK_N>::kStages


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed * 1009 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def half_view(rows, cols, ld, seed, offset=0):
    """[rows, cols] fp16 view with row stride ld, starting `offset` elements into its storage (offset 1 = not 16-byte addressable)."""
    buf = rnd(rows * ld + offset, seed=seed).half()
    return buf[offset:].view(rows, ld)[:, :cols]


def twice(fn):
    a = fn()
    b = fn()
    assert torch.equal(a, b), "two identical launches differ: results must be bitwise reproducible"
    return a


# ------------------------------------------------------------------------------------------------------------------------------ GEMM
EPIS = ["none", "bias", "bias_gb", "res_fold", "res_epi"]
MS = [1, 63, 64, 65, 129]


def grid_cases():
    cases = []
    for b, bn in enumerate(BLOCK_NS):
        k_wrap = 64 * (K_STAGES[bn] + 3) + 8
        for e, epi in enumerate(EPIS):
            M = MS[(e + b) % 5]
            N = [5, bn + 3, 2 * bn + 8, 7, 3 * bn // 2 + 9][(e + 2 * b) % 5]
            K = [8, 72, k_wrap][(e + b) % 3]
            odd_ldo = (e + b) % 2 == 1
            cases.append((bn, epi, M, N, K, odd_ldo))
    return cases


def run_gemm(a, w, bn, N, odd_ldo, **kw):
    M = a.shape[0]
    ldo = N + 1 + (N % 2) if odd_ldo else (N + 7) // 8 * 8  # odd: pair_ok off, every column through the scalar store
    out = torch.full((M, ldo), float("nan"), dtype=torch.float16, device=dev)
    ops.gemm(a, w, out=out[:, :N], force_bn=bn, **kw)
    return out[:, :N]


@pytest.mark.parametrize("bn,epi,M,N,K,odd_ldo", grid_cases())
def test_gemm_grid(bn, epi, M, N, K, odd_ldo, report):
    a, w = rnd(M, K, seed=1).half(), rnd(N, K, seed=2, scale=K ** -0.5).half()
    kw, ref_kw = {}, {}
    if epi != "none":
        kw["bias"] = ref_kw["bias"] = rnd(N, seed=3)
    if epi == "bias_gb":
        rpg = max(1, (M + 2) // 3)  # 3 groups: boundaries inside the 128-row tile
        gb = rnd((M + rpg - 1) // rpg, N, seed=4)
        kw.update(group_bias=gb, rows_per_group=rpg)
        ref_kw.update(group_bias=gb, rows_per_group=rpg)
    if epi == "res_fold":
        kw["residual"] = half_view(M, N, (N + 7) // 8 * 8, seed=5)  # 16-byte rows: folded into the MMA as extra k-blocks
    if epi == "res_epi":
        # 2-byte-offset view, or an odd row stride: not TMA-addressable, added in the epilogue
        kw["residual"] = half_view(M, N, (N + 7) // 8 * 8, seed=5, offset=1) if M % 2 else half_view(M, N, N + 1 + N % 2, seed=5)
    if "residual" in kw:
        ref_kw["residuals"] = (kw["residual"],)
    got = twice(lambda: run_gemm(a, w, bn, N, odd_ldo, **kw).clone())
    ref, terms = gemm_ref(a, w, **ref_kw)
    check_tap(got, ref, terms, K + len(ref_kw), report, f"gemm_{epi}_bn{bn}_{M}x{N}x{K}_ldo{'odd' if odd_ldo else 'even'}")


@pytest.mark.parametrize("bn", BLOCK_NS)
def test_gemm_many_tiles(bn, report):
    """More tiles than SMs: each CTA runs several tiles back to back, with a k-loop (taps x k-blocks + folded blocks) that is not a multiple
    of the ring depth, so the ring phase carried from tile to tile is exercised."""
    M, N, K = 5000, 3 * bn + 24, 64 * (K_STAGES[bn] + 3) + 8
    a, w = rnd(M, K, seed=11).half(), rnd(N, K, seed=12, scale=K ** -0.5).half()
    bias, gb, res = rnd(N, seed=13), rnd(3, N, seed=14), rnd(M, N, seed=15).half()
    n_tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
    assert n_tiles > torch.cuda.get_device_properties(0).multi_processor_count
    got = twice(lambda: ops.gemm(a, w, bias=bias, group_bias=gb, rows_per_group=1700, residual=res, force_bn=bn)[:, :N].clone())
    ref, terms = gemm_ref(a, w, bias=bias, group_bias=gb, rows_per_group=1700, residuals=(res,))
    check_tap(got, ref, terms, K + 3, report, f"gemm_many_tiles_bn{bn}")


@pytest.mark.parametrize("path", ["fold", "epi"])
@pytest.mark.parametrize("bn", BLOCK_NS)
def test_gemm_two_residuals(bn, path, report):
    """Two skip tensors at once (n_res = 2 when both are TMA-addressable); ops.gemm does not expose residual2, so the C ABI is called."""
    M, N, K = 200, bn + 24, 136
    a, w = rnd(M, K, seed=21).half(), rnd(N, K, seed=22, scale=K ** -0.5).half()
    bias = rnd(N, seed=23)
    r1 = half_view(M, N, N, seed=24)
    r2 = half_view(M, N, N + 8, seed=25, offset=1 if path == "epi" else 0)

    def run():
        out = torch.empty(M, N, dtype=torch.float16, device=dev)
        e = ops._epilogue(bias, residual=r1, residual2=r2)
        _lib.call("fz_gemm_f16", ops._p(a), a.stride(0), ops._p(w), w.stride(0), M, N, K, C.byref(e), ops._p(out), out.stride(0), bn,
                  ops._stream())
        return out

    got = twice(run)
    ref, terms = gemm_ref(a, w, bias=bias, residuals=(r1, r2))
    check_tap(got, ref, terms, K + 3, report, f"gemm_two_res_{path}_bn{bn}")


@pytest.mark.parametrize("bn", BLOCK_NS)
def test_gemm_vt(bn, report):
    """Q|K row-major + V written transposed (the CLIP layout: S = 77 padded to vt_ld = 80): S is not a multiple of 128, so a tile spans two
    (frame, batch) rows, vt_col_start = 2 C = 160 sits inside a tile for BLOCK_N 64, 128 and 256, and the bias covers the V columns."""
    BF, S, heads, d, ld = 3, 77, 2, 40, 80
    Cc = heads * d
    M, K = BF * S, 72
    a, w = rnd(M, K, seed=31).half(), rnd(3 * Cc, K, seed=32, scale=K ** -0.5).half()
    bias = rnd(3 * Cc, seed=33)

    def run():
        vt = torch.full((BF, heads, d, ld), 7.0, dtype=torch.float16, device=dev)
        qk = ops.gemm(a, w, bias=bias, vt=dict(out=vt, col_start=2 * Cc, S=S, d=d, heads=heads, ld=ld), force_bn=bn)
        return torch.cat([qk.flatten(), vt.flatten()])

    got = twice(run)
    qk, vt = got[:M * 2 * Cc].view(M, 2 * Cc), got[M * 2 * Cc:].view(BF, heads, d, ld)
    ref, terms = gemm_ref(a, w, bias=bias)
    check_tap(qk, ref[:, :2 * Cc], terms[:, :2 * Cc], K + 1, report, f"vt_qk_bn{bn}")
    to_vt = lambda t: t[:, 2 * Cc:].reshape(BF, S, heads, d).permute(0, 2, 3, 1)
    check_tap(vt[..., :S], to_vt(ref), to_vt(terms), K + 1, report, f"vt_v_bn{bn}")
    assert torch.all(vt[..., S:] == 7.0), "V^T store wrote into the padding columns beyond S"


# GEGLU: two_n chosen so that pack_geglu lands on each BLOCK_N it can produce
GEGLU_CASES = [(512, 1, 64), (320, 63, 72), (384, 65, 136), (192, 129, 8), (96, 300, 200)]


@pytest.mark.parametrize("two_n,M,K", GEGLU_CASES)
def test_geglu(two_n, M, K, report):
    a = rnd(M, K, seed=41).half()
    w = rnd(two_n, K, seed=42, scale=K ** -0.5).half()
    b = rnd(two_n, seed=43) * 0.5
    wp, bp, bn = ops.pack_geglu(w, b)
    assert bn == {512: 256, 320: 160, 384: 128, 192: 64, 96: 32}[two_n]
    got = twice(lambda: ops.gemm(a, wp, bias=bp, geglu=True, force_bn=bn).clone())
    nout = two_n // 2
    proj, terms = gemm_ref(a, w, bias=b)
    x, g = proj[:, :nout], proj[:, nout:]
    tx, tg = terms[:, :nout], terms[:, nout:]
    gelu = 0.5 * g * (1 + torch.erf(g / 2 ** 0.5))
    ref = x * gelu
    # fp32 accumulation of x and of the gate propagated through x * gelu(g) (|gelu'| <= 1.13), and the erf approximation of the kernel
    # (|error| <= 1.5e-7, with approximate rcp / ex2): 2^-20 |x| (|g| + 1)
    terms_out = tx * gelu.abs() + 1.13 * x.abs() * tg
    check_tap(got[:, :nout], ref, terms_out, K + 1, report, f"geglu_bn{bn}_{M}x{nout}x{K}", fixed=2.0 ** -20 * x.abs() * (g.abs() + 1))


@pytest.mark.parametrize("term", ["residual", "residual2", "group_bias", "vt"])
def test_geglu_refuses_other_terms(term):
    """The GEGLU epilogue applies the bias only: any other epilogue term must be refused before launch, not silently dropped."""
    M, K, two_n = 64, 64, 128
    a, w = rnd(M, K, seed=51).half(), rnd(two_n, K, seed=52).half()
    wp, bp, bn = ops.pack_geglu(w, rnd(two_n, seed=53))
    out = torch.zeros(M, two_n // 2, dtype=torch.float16, device=dev)
    res = rnd(M, two_n // 2, seed=54).half()
    kw = dict(residual=res, residual2=res, group_bias=rnd(1, two_n // 2, seed=55), rows_per_group=M,
              vt_out=torch.zeros(1, 1, 64, M, dtype=torch.float16, device=dev), vt_col_start=32, vt_S=M, vt_d=64, vt_heads=1)
    sel = {"residual": ["residual"], "residual2": ["residual2"], "group_bias": ["group_bias", "rows_per_group"],
           "vt": ["vt_out", "vt_col_start", "vt_S", "vt_d", "vt_heads"]}[term]
    e = ops._epilogue(bp, geglu=True, **{k: kw[k] for k in sel})
    with pytest.raises(RuntimeError, match="GEGLU"):
        _lib.call("fz_gemm_f16", ops._p(a), a.stride(0), ops._p(wp), wp.stride(0), M, two_n, K, C.byref(e), ops._p(out), out.stride(0), bn,
                  ops._stream())
    torch.cuda.synchronize()
    assert torch.all(out == 0), "refused call must not launch"


# ------------------------------------------------------------------------------------------------------------------------------ conv
def conv_inputs(NB, H, W, Cin, Cout, seed):
    x = rnd(NB, H, W, Cin, seed=seed).half()
    w9 = rnd(9, Cout, Cin, seed=seed + 1, scale=(9 * Cin) ** -0.5).half()
    return x, w9


# NB, H, W, Cin, Cout, BLOCK_N: (rows per tile)
CONV_S1 = [
    (1, 5, 5, 72, 40, 16),     # 25-row tile: warpgroup 1 has no rows
    (2, 20, 20, 8, 24, 32),    # bh 6 -> 5 (Ho % bh): 100-row tiles
    (1, 24, 24, 320, 160, 160),  # bh 5 -> 4: 96-row tiles
    (3, 8, 8, 72, 45, 64),     # NB 3: images per tile 2 -> 1; odd Cout: epilogue-path residual, scalar stores
    (4, 8, 8, 8, 300, 256),    # 2 images per tile
    (6, 4, 4, 320, 96, 128),   # 6 images per tile (96 rows)
    (1, 64, 96, 8, 64, 64),    # non-square, one 96-pixel row per tile
    (1, 3, 256, 72, 48, 32),   # 256-wide: two 128-pixel row segments per image row
    (1, 3, 192, 72, 40, 64),   # 192-wide (VAE at 768: encoder level 2, decoder level 0): two 96-pixel segments
    (2, 2, 320, 8, 48, 160),   # 320-wide (VAE at 640): four 80-pixel segments, two images
    (1, 2, 576, 32, 24, 16),   # 576-wide (VAE at 576): six 96-pixel segments
    (1, 4, 192, 320, 160, 256),  # 192-wide at Cin 320: 5 k-blocks per tap
]


@pytest.mark.parametrize("NB,H,W,Cin,Cout,bn", CONV_S1)
def test_conv3x3_s1(NB, H, W, Cin, Cout, bn, report):
    x, w9 = conv_inputs(NB, H, W, Cin, Cout, seed=61)
    bias = rnd(Cout, seed=63)
    rpg = H * W if NB > 1 else 17  # one group per image (the engine's layout) or, for one image, boundaries inside a tile
    M = NB * H * W
    gb = rnd((M + rpg - 1) // rpg, Cout, seed=64)
    res = rnd(NB, H, W, Cout, seed=65).half()
    got = twice(lambda: ops.conv3x3(x, w9, bias=bias, residual=res, group_bias=gb, rows_per_group=rpg, force_bn=bn))
    ref, terms = conv3x3_ref(x, w9, bias=bias, group_bias=gb, rows_per_group=rpg, residuals=(res,))
    check_tap(got.reshape(-1, Cout), ref, terms, 9 * Cin + 3, report, f"conv_s1_{NB}x{H}x{W}x{Cin}->{Cout}_bn{bn}")


# NB, H, W, Cin, Cout, BLOCK_N, asym_pad
CONV_S2 = [
    (2, 18, 18, 72, 40, 64, False),   # 9x9 output, Cin 72 under stride 2
    (2, 18, 18, 32, 24, 16, True),    # asymmetric padding, odd output size
    (3, 16, 16, 72, 64, 128, True),   # asymmetric, Cin 72
    (1, 32, 32, 32, 160, 160, False),
    (1, 4, 512, 32, 33, 32, True),    # 256-wide output (VAE resolutions), odd Cout
    (2, 10, 10, 72, 256, 256, False),
    (1, 4, 384, 32, 40, 32, True),    # 192-wide output (the VAE encoder's second downsample at 768): 96-pixel segments
    (2, 4, 384, 72, 64, 128, False),  # the same width, symmetric padding
    (1, 6, 576, 8, 24, 256, True),    # 288-wide output (VAE at 576), three output rows
    (1, 2, 576, 32, 160, 160, False),
    (1, 4, 384, 72, 24, 16, True),
]


@pytest.mark.parametrize("NB,H,W,Cin,Cout,bn,asym", CONV_S2)
def test_conv3x3_s2(NB, H, W, Cin, Cout, bn, asym, report):
    x, w9 = conv_inputs(NB, H, W, Cin, Cout, seed=71)
    bias = rnd(Cout, seed=73)
    res = rnd(NB, H // 2, W // 2, Cout, seed=74).half()
    got = twice(lambda: ops.conv3x3(x, w9, bias=bias, stride=2, residual=res, force_bn=bn, asym_pad=asym))
    ref, terms = conv3x3_ref(x, w9, stride=2, asym_pad=asym, bias=bias, residuals=(res,))
    check_tap(got.reshape(-1, Cout), ref, terms, 9 * Cin + 2, report, f"conv_s2_{'asym' if asym else 'sym'}_{NB}x{H}x{W}x{Cin}->{Cout}_bn{bn}")


@pytest.mark.parametrize("W,stride,asym", [(262, 1, False), (524, 2, True), (524, 2, False), (131 * 3, 1, False)])
def test_conv3x3_refuses_width(W, stride, asym):
    """An output width above 128 whose largest divisor up to 128 is below 8 (262 = 2 x 131, 393 = 3 x 131) would need 1- to 3-row tiles:
    refused before launch, whatever the stride."""
    Wo = W // stride
    x, w9 = conv_inputs(1, 2 * stride, W, 8, 16, seed=75)
    with pytest.raises(RuntimeError, match=f"output width {Wo} has no divisor"):
        ops.conv3x3(x, w9, stride=stride, asym_pad=asym, force_bn=16)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------------------------------------- tconv3
# B, F, HW, Cin, Cout, BLOCK_N: (rows per tile)
TCONV = [
    (1, 1, 16, 72, 40, 64),     # 16-row tile
    (2, 3, 16, 8, 24, 16),      # 3 frames per tile (48 rows)
    (1, 5, 16, 72, 48, 32),     # 5 frames per tile (80 rows)
    (2, 3, 64, 320, 160, 160),  # bf 2 -> 1 (F % bf)
    (1, 5, 64, 8, 136, 128),    # bf 2 -> 1
    (1, 16, 96, 72, 64, 256),   # 96-pixel box
    (1, 24, 200, 8, 45, 64),    # 128-pixel box shrinks to 100; odd Cout: epilogue-path skip tensors
    (1, 2, 131, 72, 32, 32),    # prime HW: 1-row tiles
    (2, 24, 16, 32, 16, 16),    # 8 frames per tile (128 rows)
]


@pytest.mark.parametrize("B,Fr,HW,Cin,Cout,bn", TCONV)
def test_tconv3(B, Fr, HW, Cin, Cout, bn, report):
    x = rnd(B, Fr, HW, Cin, seed=81).half()
    w3 = rnd(3, Cout, Cin, seed=82, scale=(3 * Cin) ** -0.5).half()
    bias, gb = rnd(Cout, seed=83), rnd(B, Cout, seed=84)
    r1, r2 = rnd(B, Fr, HW, Cout, seed=85).half(), rnd(B, Fr, HW, Cout, seed=86).half()
    kw = dict(bias=bias, group_bias=gb, rows_per_group=Fr * HW)
    got = twice(lambda: ops.tconv3(x, w3, residual=r1, residual2=r2, force_bn=bn, **kw))
    ref, terms = tconv3_ref(x, w3, residuals=(r1, r2), **kw)
    check_tap(got.reshape(-1, Cout), ref, terms, 3 * Cin + 4, report, f"tconv_{B}x{Fr}x{HW}x{Cin}->{Cout}_bn{bn}")


@pytest.mark.parametrize("B,Fr,HW,Cin,Cout,bn", [(1, 1, 64, 72, 40, 64), (2, 4, 16, 32, 24, 16), (1, 3, 200, 8, 160, 160)])
def test_tconv3_halo(B, Fr, HW, Cin, Cout, bn, report):
    """Frame-sharded temporal conv on one GPU: frames 0 and F + 1 of x hold non-zero neighbour frames, which the conv must read."""
    x = rnd(B, Fr + 2, HW, Cin, seed=91).half()
    w3 = rnd(3, Cout, Cin, seed=92, scale=(3 * Cin) ** -0.5).half()
    bias, res = rnd(Cout, seed=93), rnd(B, Fr, HW, Cout, seed=94).half()
    got = twice(lambda: ops.tconv3(x, w3, bias=bias, residual=res, force_bn=bn, halo=True))
    ref, terms = tconv3_ref(x, w3, halo=True, bias=bias, residuals=(res,))
    check_tap(got.reshape(-1, Cout), ref, terms, 3 * Cin + 2, report, f"tconv_halo_{B}x{Fr}x{HW}x{Cin}->{Cout}_bn{bn}")
