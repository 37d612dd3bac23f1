"""GPU parity tests of every C-ABI kernel against a plain PyTorch fp32 restatement of the same reference op.
(op-level; the pipeline-level parity against oracle/fz_oracle.py lives in test_gpu_pipeline.py)"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from fatezero_b200 import _lib, ops

dev = "cuda"


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def stats(got, ref):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    return dict(max_abs=err.max().item(), mean_abs=err.mean().item(), ref_max=ref.abs().max().item(), ref_std=ref.std().item(),
                nan=bool(torch.isnan(got).any().item()))


def close(got, ref, report, key, atol, rtol=0.0):
    s = stats(got, ref)
    report[key] = s
    assert not s["nan"], f"{key}: NaN in output"
    lim = atol + rtol * s["ref_max"]
    assert s["max_abs"] <= lim, f"{key}: max_abs {s['max_abs']:.4g} > {lim:.4g} (ref_max {s['ref_max']:.3g})"


# ---------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 128), (256, 256, 128, 256), (1000, 320, 640, 0), (384, 640, 320, 160),
                                       (130, 48, 72, 0), (512, 1280, 1280, 0), (2048, 16, 320, 16), (300, 64, 64, 64),
                                       (300, 96, 200, 32)])
def test_gemm_plain(M, N, K, bn, report):
    a, w = rnd(M, K).half(), rnd(N, K, scale=K ** -0.5, seed=1).half()
    bias = rnd(N, seed=2)
    res = rnd(M, N, seed=3).half()
    out = ops.gemm(a, w, bias=bias, residual=res, force_bn=bn)
    ref = a.float() @ w.float().t() + bias + res.float()
    close(out[:, :N], ref, report, f"gemm_{M}x{N}x{K}_bn{bn}", atol=2e-2, rtol=2e-3)


def test_gemm_nobias_strided_a(report):
    big = rnd(512, 3 * 320).half()
    a = big[:, 320:640]  # strided view (lda = 960)
    w = rnd(640, 320, scale=320 ** -0.5, seed=1).half()
    out = ops.gemm(a, w)
    close(out, a.float() @ w.float().t(), report, "gemm_strided", atol=2e-2, rtol=2e-3)


def test_gemm_group_bias(report):
    M, N, K = 1024, 320, 320
    a, w = rnd(M, K).half(), rnd(N, K, scale=K ** -0.5, seed=1).half()
    gb = rnd(2, N, seed=5)
    out = ops.gemm(a, w, group_bias=gb, rows_per_group=512)
    ref = a.float() @ w.float().t() + gb.repeat_interleave(512, 0)
    close(out, ref, report, "gemm_group_bias", atol=2e-2, rtol=2e-3)


@pytest.mark.parametrize("C", [64, 320, 640])
def test_gemm_geglu(C, report):
    M = 777
    a = rnd(M, C).half()
    w = rnd(8 * C, C, scale=C ** -0.5, seed=1).half()
    b = rnd(8 * C, seed=2) * 0.1
    wp, bp, bn = ops.pack_geglu(w, b)
    out = ops.gemm(a, wp, bias=bp, geglu=True, force_bn=bn)
    proj = a.float() @ w.float().t() + b
    x, g = proj.chunk(2, dim=-1)
    close(out, x * F.gelu(g), report, f"geglu_{C}", atol=2e-2, rtol=3e-3)


@pytest.mark.parametrize("d,heads,S,BF", [(40, 8, 64, 3), (80, 8, 256, 2), (16, 4, 128, 2), (40, 8, 4096, 2), (160, 8, 64, 4), (80, 8, 1024, 3)])
def test_gemm_qkv_vt(d, heads, S, BF, report):
    C_ = d * heads
    M = BF * S
    a = rnd(M, C_).half()
    w = rnd(3 * C_, C_, scale=C_ ** -0.5, seed=1).half()
    vt = torch.zeros(BF, heads, d, S, dtype=torch.float16, device=dev)
    out = ops.gemm(a, w, vt=dict(out=vt, col_start=2 * C_, S=S, d=d, heads=heads))
    ref = a.float() @ w.float().t()
    close(out[:, :2 * C_], ref[:, :2 * C_], report, f"qk_{d}", atol=2e-2, rtol=2e-3)
    v = ref[:, 2 * C_:].reshape(BF, S, heads, d).permute(0, 2, 3, 1)
    close(vt, v, report, f"vt_{d}", atol=2e-2, rtol=2e-3)


# ---------------------------------------------------------------------------------------------------------------- conv
@pytest.mark.parametrize("NB,H,Cin,Cout,stride", [(2, 64, 64, 64, 1), (3, 32, 128, 320, 1), (4, 16, 320, 160, 1), (4, 8, 64, 128, 1),
                                                    (2, 64, 64, 64, 2), (3, 32, 320, 320, 2), (4, 16, 128, 64, 2), (2, 24, 64, 64, 1)])
def test_conv3x3(NB, H, Cin, Cout, stride, report):
    x = rnd(NB, H, H, Cin).half()
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=1).half()
    b = rnd(Cout, seed=2)
    w9 = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    out = ops.conv3x3(x, w9, bias=b, stride=stride)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b, stride=stride, padding=1).permute(0, 2, 3, 1)
    close(out, ref, report, f"conv_{NB}_{H}_{Cin}_{Cout}_s{stride}", atol=2e-2, rtol=2e-3)


def test_conv3x3_group_bias_residual(report):
    NB, H, Cin, Cout = 4, 16, 64, 64
    x = rnd(NB, H, H, Cin).half()
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=1).half()
    w9 = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    gb = rnd(2, Cout, seed=4)
    res = rnd(NB, H, H, Cout, seed=5).half()
    out = ops.conv3x3(x, w9, residual=res, group_bias=gb, rows_per_group=2 * H * H)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), None, padding=1).permute(0, 2, 3, 1)
    ref = ref + gb.repeat_interleave(2, 0)[:, None, None, :] + res.float()
    close(out, ref, report, "conv_gb_res", atol=2e-2, rtol=2e-3)


@pytest.mark.parametrize("B,Fr,HW,Cin,Cout", [(1, 8, 256, 64, 32), (2, 8, 64, 320, 160), (2, 3, 1024, 160, 320), (1, 8, 4096, 32, 64)])
def test_tconv3(B, Fr, HW, Cin, Cout, report):
    x = rnd(B, Fr, HW, Cin).half()
    w = rnd(Cout, Cin, 3, scale=(3 * Cin) ** -0.5, seed=1).half()
    w3 = w.permute(2, 0, 1).contiguous()
    out = ops.tconv3(x, w3)
    x1 = x.float().permute(0, 2, 3, 1).reshape(B * HW, Cin, Fr)
    ref = F.conv1d(x1, w.float(), padding=1).reshape(B, HW, Cout, Fr).permute(0, 3, 1, 2)
    close(out, ref, report, f"tconv_{B}_{Fr}_{HW}_{Cin}_{Cout}", atol=2e-2, rtol=2e-3)


# ---------------------------------------------------------------------------------------------------------------- norms etc.
@pytest.mark.parametrize("NB,HW,C,fps,silu", [(8, 4096, 320, 8, True), (16, 256, 1280, 8, True), (6, 1024, 64, 1, False),
                                               (4, 64, 2560, 2, True), (4, 256, 1920, 4, True), (2, 576, 160, 2, False)])
def test_groupnorm(NB, HW, C, fps, silu, report):
    x = (rnd(NB, HW, C) * 1.5 + 0.7).half()
    g, b = rnd(C, seed=1) * 0.2 + 1, rnd(C, seed=2) * 0.2
    out = ops.groupnorm(x, g, b, 1e-5, 32, fps, silu)
    xr = x.float().reshape(NB // fps, fps * HW, C).permute(0, 2, 1)  # [S, C, L]
    ref = F.group_norm(xr, 32, g, b, 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(NB, HW, C)
    close(out, ref, report, f"gn_{NB}_{HW}_{C}_{fps}", atol=5e-3, rtol=2e-3)


@pytest.mark.parametrize("M,C", [(1000, 320), (333, 640), (64, 1280), (77, 64)])
def test_layernorm(M, C, report):
    x = (rnd(M, C) * 2 + 0.3).half()
    g, b = rnd(C, seed=1) * 0.2 + 1, rnd(C, seed=2) * 0.2
    out = ops.layernorm(x, g, b)
    close(out, F.layer_norm(x.float(), (C,), g, b, 1e-5), report, f"ln_{M}_{C}", atol=5e-3, rtol=2e-3)


def test_upsample_concat(report):
    x = rnd(3, 8, 8, 64).half()
    up = ops.upsample2x(x)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    close(up, ref, report, "upsample", atol=0)
    a, b = rnd(5, 16, 64).half(), rnd(5, 16, 128, seed=1).half()
    close(ops.concat_channels(a, b), torch.cat([a, b], -1), report, "concat", atol=0)


def test_im2col_conv_in(report):
    B, Fr, H, C0 = 2, 3, 16, 64
    x = rnd(B, 4, Fr, H, H)
    w = rnd(C0, 4, 3, 3, scale=1 / 6, seed=1)
    bias = rnd(C0, seed=2)
    cols = ops.im2col_latents(x)
    wp = torch.zeros(C0, 64, device=dev)
    wp[:, :36] = w.permute(0, 2, 3, 1).reshape(C0, 36)  # col = tap*4 + c
    out = ops.gemm(cols, wp.half().contiguous(), bias=bias)
    ref = F.conv2d(x.permute(0, 2, 1, 3, 4).reshape(B * Fr, 4, H, H), w, bias, padding=1).permute(0, 2, 3, 1).reshape(-1, C0)
    close(out, ref, report, "conv_in", atol=2e-2, rtol=2e-3)


def test_out_temporal(report):
    B, Fr, H = 2, 5, 8
    y = rnd(B * Fr * H * H, 8).half()
    down, up = rnd(2, 4, 3, seed=1) * 0.5, rnd(4, 2, 3, seed=2) * 0.5
    eps = ops.out_temporal(y, B, 4, Fr, H, H, down=down.contiguous(), up=up.contiguous())
    y5 = y[:, :4].float().reshape(B, Fr, H * H, 4)
    x1 = y5.permute(0, 2, 3, 1).reshape(B * H * H, 4, Fr)
    ref = F.conv1d(F.conv1d(x1, down, padding=1), up, padding=1) + x1
    ref = ref.reshape(B, H, H, 4, Fr).permute(0, 3, 4, 1, 2)
    close(eps, ref, report, "out_temporal_lora", atol=5e-3, rtol=2e-3)
    wf, bf_ = rnd(4, 4, 3, seed=3) * 0.5, rnd(4, seed=4)
    eps2 = ops.out_temporal(y, B, 4, Fr, H, H, w_full=wf.contiguous(), b_full=bf_)
    ref2 = F.conv1d(x1, wf, bf_, padding=1).reshape(B, H, H, 4, Fr).permute(0, 3, 4, 1, 2)
    close(eps2, ref2, report, "out_temporal_full", atol=5e-3, rtol=2e-3)


def test_time_embedding(report):
    t = 481.0
    s = ops.timestep_sinusoid(t, 320, True, 0.0, dev)
    half = 160
    e = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / half).to(dev) * t
    ref = torch.cat([torch.cos(e), torch.sin(e)])
    close(s, ref, report, "sinusoid", atol=2e-4)
    w, b = rnd(1280, 320, scale=320 ** -0.5).half(), rnd(1280, seed=1)
    y = ops.rowvec_linear(s, w, b, False)
    close(y, w.float() @ ref + b, report, "rowvec", atol=2e-3, rtol=1e-3)
    y2 = ops.rowvec_linear(y, rnd(640, 1280, scale=1280 ** -0.5, seed=2).half(), None, True)
    close(y2, rnd(640, 1280, scale=1280 ** -0.5, seed=2).half().float() @ F.silu(y), report, "rowvec_silu", atol=2e-3, rtol=1e-3)


@pytest.mark.parametrize("B,Fr,HW,heads,d", [(2, 8, 64, 8, 40), (1, 3, 256, 4, 16), (1, 8, 16, 8, 160), (2, 8, 1024, 8, 80), (1, 4, 64, 8, 40),
                                             (1, 2, 96, 4, 16)])
def test_temporal_attn(B, Fr, HW, heads, d, report):
    C_ = heads * d
    qkv = rnd(B * Fr * HW, 3 * C_).half()
    out = ops.temporal_attn(qkv, B, Fr, HW, heads, d, d ** -0.5)
    t = qkv.float().reshape(B, Fr, HW, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # [3, B, HW, heads, F, d]
    q, k, v = t[0], t[1], t[2]
    p = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, dim=-1)
    ref = (p @ v).permute(0, 3, 1, 2, 4).reshape(B * Fr * HW, C_)
    close(out, ref, report, f"tattn_{d}", atol=5e-3, rtol=2e-3)


def test_ddim_steps(report):
    x, e = rnd(1, 4, 8, 16, 16), rnd(1, 4, 8, 16, 16, seed=1)
    x1 = x.clone()
    ops.ddim_invert_step(x1, e, 0.9, 0.8)
    x0 = (x - (1 - 0.9) ** 0.5 * e) / 0.9 ** 0.5
    close(x1, 0.8 ** 0.5 * x0 + (1 - 0.8) ** 0.5 * e, report, "ddim_inv", atol=1e-5)
    e2 = rnd(2, 4, 8, 16, 16, seed=2)
    xinv = rnd(1, 4, 8, 16, 16, seed=3)
    m = (rnd(8, 16, 16, seed=4) > 0).float()
    x2 = x.clone()
    ops.cfg_ddim_step(x2, e2, 7.5, 0.5, 0.6, x_inv=xinv, mask_a=m, apply_blend=True)
    eps = e2[0:1] + 7.5 * (e2[1:2] - e2[0:1])
    x0 = (x - 0.5 ** 0.5 * eps) / 0.5 ** 0.5
    xn = 0.6 ** 0.5 * x0 + 0.4 ** 0.5 * eps
    close(x2, xinv + m[None, None] * (xn - xinv), report, "cfg_ddim_blend", atol=2e-5)


def test_blend_mask(report):
    Fr, heads, r = 3, 8, 16
    maps = [torch.softmax(rnd(Fr, heads, r * r, 80, seed=i) * 2, -1).half() for i in range(5)]
    w = torch.zeros(77)
    w[[2, 3]] = 1
    for (h, th) in [(32, 0.6), (16, 0.8), (64, 0.5), (8, 0.7)]:
        out = ops.blend_mask(maps, w, th, h, h)
        st = torch.cat([(m[..., :77].float() * w.to(dev)).sum(-1).reshape(Fr, heads, r, r).permute(1, 0, 2, 3) for m in maps], 0).mean(0)
        mp = F.max_pool2d(st[None], 3, 1, 1)
        mk = F.interpolate(mp, size=(h, h))[0]
        mk = mk / mk.amax(dim=(-2, -1), keepdim=True)
        ref = mk.gt(th).float()
        frac = (out != ref).float().mean().item()
        report[f"mask_{h}"] = dict(mismatch_frac=frac, ones=ref.mean().item())
        assert frac < 2e-3  # ties at the threshold can flip with summation order


def test_limits_conv_row_segments_and_groupnorm_batch(report):
    """Hard limits of the C ABI with a test AT the limit and an error beyond it: 3x3 conv output width 128 (one TMA box row), wider rows
    tiled in segments of their largest divisor up to 128 (136: two 68-pixel segments), a width without such a divisor of at least 8
    refused (262 = 2 x 131); GroupNorm over 256 images with 64 groups (the 1 MiB workspace)."""
    w = rnd(64, 64, 3, 3, scale=(64 * 9) ** -0.5, seed=1)
    w9 = w.permute(2, 3, 0, 1).reshape(9, 64, 64).half().contiguous()
    for width in (128, 136):
        x = rnd(1, 8, width, 64).half()
        out = ops.conv3x3(x, w9)
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w9.float().reshape(3, 3, 64, 64).permute(2, 3, 0, 1), padding=1).permute(0, 2, 3, 1)
        close(out, ref, report, f"conv_w{width}", atol=2e-2, rtol=2e-3)
    with pytest.raises(RuntimeError, match="width"):
        ops.conv3x3(rnd(1, 8, 262, 64).half(), w9)
    xg = rnd(256, 16, 128).half()
    g, b = 1 + 0.1 * rnd(128, seed=3), 0.1 * rnd(128, seed=4)
    y = ops.groupnorm(xg, g, b, 1e-5, 64, 1, False)
    refg = F.group_norm(xg.float().permute(0, 2, 1), 64, g, b, 1e-5).permute(0, 2, 1)
    close(y, refg, report, "groupnorm_nb256_g64", atol=2e-2, rtol=2e-3)
    with pytest.raises(RuntimeError, match="workspace|unsupported"):
        ops.groupnorm(rnd(257, 16, 128).half(), g, b, 1e-5, 64, 1, False)


def test_small_m_long_k(report):
    """Small-M problems with long k-loops (the r = 8 layers: a few dozen tiles with 60-180 serial k-blocks each), bitwise reproducible.
    (A deterministic split-K variant of the tap-GEMM was built and measured in round 2: 698 vs 682 ms per 1-frame clip, 1897 vs 1889 ms per
    8-frame clip — the dump / fence / atomic / read-back of the partial tiles cost what the shorter k-loops saved, so it was dropped.)"""
    # 3x3 conv 1280 -> 1280 at 8x8, 8 images (180 k-blocks, 4 M tiles)
    x = rnd(8, 8, 8, 1280).half()
    w = rnd(1280, 1280, 3, 3, scale=(1280 * 9) ** -0.5, seed=1)
    b = rnd(1280, seed=2) * 0.1
    res = rnd(8, 8, 8, 1280, seed=4).half()
    w9 = w.permute(2, 3, 0, 1).reshape(9, 1280, 1280).half().contiguous()
    out = ops.conv3x3(x, w9, bias=b, residual=res)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w9.float().reshape(3, 3, 1280, 1280).permute(2, 3, 0, 1), b, padding=1).permute(0, 2, 3, 1) + res.float()
    close(out, ref, report, "small_m_conv_r8", atol=2e-2, rtol=2e-3)
    assert torch.equal(out, ops.conv3x3(x, w9, bias=b, residual=res))
    # one image (64 rows: half an M tile)
    out1 = ops.conv3x3(x[:1].contiguous(), w9, bias=b)
    close(out1, ref[:1] - res[:1].float(), report, "small_m_conv_r8_one_image", atol=2e-2, rtol=2e-3)
    # linear 512 x 1280 x 5120 with bias + skip (80 k-blocks)
    a = rnd(512, 5120, seed=5).half()
    wl = rnd(1280, 5120, scale=5120 ** -0.5, seed=6).half()
    r2 = rnd(512, 1280, seed=7).half()
    got = ops.gemm(a, wl, bias=b, residual=r2)
    close(got, a.float() @ wl.float().t() + b + r2.float(), report, "small_m_linear", atol=2e-2, rtol=2e-3)
    assert torch.equal(got, ops.gemm(a, wl, bias=b, residual=r2))
    # temporal conv 1280 -> 160 over 8 frames of 64 pixels (60 k-blocks)
    xt = rnd(2, 8, 64, 1280, seed=8).half()
    w3 = rnd(3, 160, 1280, scale=(3 * 1280) ** -0.5, seed=9).half()
    yt = ops.tconv3(xt, w3)
    xp = F.pad(xt.float(), (0, 0, 0, 0, 1, 1))
    reft = sum(torch.einsum("bfpc,oc->bfpo", xp[:, t:t + 8], w3[t].float()) for t in range(3))
    close(yt, reft, report, "small_m_tconv", atol=2e-2, rtol=2e-3)
