"""Thin torch-tensor wrappers over the C ABI (include/fatezero_b200.h).  PyTorch is plumbing here: device memory,
streams, and nothing else — every compute call below lands in libfatezero_b200.so."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import AttnArgs, Epilogue

f16 = torch.float16


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"fatezero_b200.ops.{name}: tensor must live on a CUDA device (no CPU fallback)")
    if t.dtype != dtype:
        raise TypeError(f"fatezero_b200.ops.{name}: expected {dtype}, got {t.dtype}")


def geglu_block_n(gemm_cols: int) -> int:
    for bn in (256, 160, 128, 64):
        if gemm_cols % bn == 0:
            return bn
    return 32


def pack_geglu(weight: torch.Tensor, bias: Optional[torch.Tensor]):
    """[2*Nout, K] (x rows then gate rows, diffusers GEGLU.proj) -> tile-interleaved so each BLOCK_N tile holds x|gate."""
    two_n, k = weight.shape
    nout = two_n // 2
    bn = geglu_block_n(two_n)
    half = bn // 2
    assert nout % half == 0
    wx, wg = weight[:nout].reshape(nout // half, half, k), weight[nout:].reshape(nout // half, half, k)
    w = torch.cat([wx, wg], dim=1).reshape(two_n, k).contiguous()
    b = None
    if bias is not None:
        bx, bg = bias[:nout].reshape(nout // half, half), bias[nout:].reshape(nout // half, half)
        b = torch.cat([bx, bg], dim=1).reshape(two_n).contiguous()
    return w, b, bn


def _epilogue(bias=None, group_bias=None, rows_per_group=0, residual=None, geglu=False, residual2=None, vt_out=None, vt_col_start=0, vt_S=0, vt_d=0,
              vt_heads=0, vt_ld=0) -> Epilogue:
    e = Epilogue()
    e.bias = _p(bias)
    e.group_bias = _p(group_bias)
    e.rows_per_group = int(rows_per_group)
    e.residual = _p(residual)
    e.ldr = residual.stride(-2) if residual is not None else 0
    e.residual2 = _p(residual2)
    e.ldr2 = residual2.stride(-2) if residual2 is not None else 0
    e.mode = _lib.EPI_GEGLU if geglu else _lib.EPI_ROWMAJOR
    e.out_vt = _p(vt_out)
    e.vt_col_start = int(vt_col_start)
    e.vt_S, e.vt_d, e.vt_heads, e.vt_ld = int(vt_S), int(vt_d), int(vt_heads), int(vt_ld)
    return e


def gemm(a: torch.Tensor, w: torch.Tensor, bias=None, residual=None, out=None, group_bias=None, rows_per_group=0, geglu=False,
         n_out: Optional[int] = None, vt: Optional[dict] = None, force_bn: int = 0) -> torch.Tensor:
    """out[M, N] = a[M, K] @ w[N, K]^T (+bias +group_bias +residual) ; geglu: w packed by pack_geglu, N_out = N/2."""
    _chk(a, f16, "gemm"); _chk(w, f16, "gemm")
    M, K = a.shape
    N = w.shape[0]
    assert a.stride(1) == 1 and w.stride(1) == 1 and w.shape[1] == K
    cols_out = N // 2 if geglu else N
    if vt is not None:
        cols_out = vt["col_start"]
    if n_out is not None:
        cols_out = n_out
    if out is None:
        out = torch.empty((M, max(cols_out, 8)), dtype=f16, device=a.device)
    e = _epilogue(bias, group_bias, rows_per_group, residual, geglu, **({} if vt is None else dict(
        vt_out=vt["out"], vt_col_start=vt["col_start"], vt_S=vt["S"], vt_d=vt["d"], vt_heads=vt["heads"], vt_ld=vt.get("ld", 0))))
    _lib.call("fz_gemm_f16", _p(a), a.stride(0), _p(w), w.stride(0), M, N, K, C.byref(e), _p(out), out.stride(0), force_bn, _stream())
    return out


def conv3x3(x: torch.Tensor, w9: torch.Tensor, bias=None, stride: int = 1, residual=None, group_bias=None, rows_per_group=0,
            force_bn: int = 0, asym_pad: bool = False) -> torch.Tensor:
    """x [NB,H,W,Cin] fp16 NHWC, w9 [9,Cout,Cin] -> [NB,H/stride,W/stride,Cout].  asym_pad (stride 2): right/bottom-only padding.
    Output widths above 128 are tiled in row segments of the largest divisor of the width up to 128; a width whose largest such divisor
    is below 8 (e.g. 262 = 2 x 131) is refused."""
    _chk(x, f16, "conv3x3"); _chk(w9, f16, "conv3x3")
    NB, H, W, Cin = x.shape
    Cout = w9.shape[1]
    assert x.is_contiguous() and w9.is_contiguous() and w9.shape == (9, Cout, Cin)
    out = torch.empty((NB, H // stride, W // stride, Cout), dtype=f16, device=x.device)
    e = _epilogue(bias, group_bias, rows_per_group, residual)
    if residual is not None:
        e.ldr = residual.shape[-1]
    if asym_pad:
        assert stride == 2
        _lib.call("fz_conv3x3_down_asym_nhwc_f16", _p(x), Cin, NB, H, W, Cin, _p(w9), Cout, C.byref(e), _p(out), Cout, force_bn, _stream())
    else:
        _lib.call("fz_conv3x3_nhwc_f16", _p(x), Cin, NB, H, W, Cin, _p(w9), Cout, stride, C.byref(e), _p(out), Cout, force_bn, _stream())
    return out


def tconv3(x: torch.Tensor, w3: torch.Tensor, bias=None, residual=None, group_bias=None, rows_per_group=0, force_bn: int = 0,
           residual2=None, halo: bool = False):
    """x [B,F,HW,Cin], w3 [3,Cout,Cin]: Conv1d(k=3,pad=1) over F -> [B,F,HW,Cout] (+bias +residual +group_bias).
    halo (frame-sharded execution): x is [B,F+2,HW,Cin] with the neighbour ranks' boundary frames in frames 0 and F+1."""
    _chk(x, f16, "tconv3"); _chk(w3, f16, "tconv3")
    B, F, HW, Cin = x.shape
    if halo:
        F -= 2
    Cout = w3.shape[1]
    assert x.is_contiguous() and w3.is_contiguous()
    out = torch.empty((B, F, HW, Cout), dtype=f16, device=x.device)
    e = _epilogue(bias, group_bias, rows_per_group, residual, residual2=residual2)
    if residual is not None:
        e.ldr = residual.shape[-1]
    if residual2 is not None:
        e.ldr2 = residual2.shape[-1]
    _lib.call("fz_tconv3_halo_f16" if halo else "fz_tconv3_f16", _p(x), Cin, B, F, HW, Cin, _p(w3), Cout, C.byref(e), _p(out), Cout, force_bn,
              _stream())
    return out


_gn_ws = {}


def _workspace(device, nbytes: int) -> torch.Tensor:
    ws = _gn_ws.get(device)
    if ws is None or ws.numel() * 8 < nbytes:
        ws = torch.zeros(max(nbytes // 8 + 1, 4096), dtype=torch.float64, device=device)  # arrival counters start at zero
        _gn_ws[device] = ws
    return ws


def groupnorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, groups: int, frames_per_stat: int, silu: bool,
              out: Optional[torch.Tensor] = None, images_per_item: Optional[int] = None) -> torch.Tensor:
    """x [NB, HW, C] fp16; statistics over (C/groups, HW, frames_per_stat consecutive NB rows).
    images_per_item (batched edits): x holds NB / images_per_item items (prompts); each image's statistics are then bitwise those of a
    call over its item alone."""
    _chk(x, f16, "groupnorm")
    NB, HW, Cc = x.shape
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    ws = _workspace(x.device, 1 << 20)  # per-(image, chunk, group) partial sums
    if images_per_item is None:
        _lib.call("fz_groupnorm_nhwc_f16", _p(x), _p(out), NB, HW, Cc, groups, frames_per_stat, _p(gamma), _p(beta), float(eps), int(silu),
                  _p(ws), _stream())
    else:
        _lib.call("fz_groupnorm_batched_nhwc_f16", _p(x), _p(out), NB, HW, Cc, groups, frames_per_stat, int(images_per_item), _p(gamma),
                  _p(beta), float(eps), int(silu), _p(ws), _stream())
    return out


def groupnorm_stats(x: torch.Tensor, groups: int) -> torch.Tensor:
    """Per-image (sum, sumsq) of every group: fp32 view [NB, groups, 2] INTO the shared workspace (valid until the next groupnorm call)."""
    _chk(x, f16, "groupnorm_stats")
    NB, HW, Cc = x.shape
    assert x.is_contiguous()
    ws = _workspace(x.device, 1 << 20)
    _lib.call("fz_groupnorm_stats_f16", _p(x), NB, HW, Cc, groups, _p(ws), _stream())
    off = (768 * 1024) // 4
    return ws.view(torch.float32)[off: off + NB * groups * 2].view(NB, groups, 2)


def groupnorm_apply(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, groups: int, frames_per_stat: int, count_frames: int,
                    silu: bool, sums: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Second half of the frame-sharded GroupNorm: sums [NB, groups, 2] fp32 per-image sums or fp64 set totals (fz_gn_combine); the
    apply adds frames_per_stat consecutive images in fp64."""
    _chk(x, f16, "groupnorm_apply")
    NB, HW, Cc = x.shape
    assert x.is_contiguous() and sums.is_contiguous() and sums.dtype in (torch.float32, torch.float64) and sums.numel() == NB * groups * 2
    if out is None:
        out = torch.empty_like(x)
    _lib.call("fz_groupnorm_apply_sums64_f16" if sums.dtype == torch.float64 else "fz_groupnorm_apply_f16", _p(x), _p(out), NB, HW, Cc, groups, frames_per_stat, count_frames, _p(gamma), _p(beta), float(eps),
              int(silu), _p(sums), _stream())
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    _chk(x, f16, "layernorm")
    M, Cc = x.shape
    assert x.is_contiguous()
    out = torch.empty_like(x)
    _lib.call("fz_layernorm_f16", _p(x), _p(out), M, Cc, _p(gamma), _p(beta), float(eps), _stream())
    return out


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    _chk(x, f16, "upsample2x")
    NB, H, W, Cc = x.shape
    out = torch.empty((NB, 2 * H, 2 * W, Cc), dtype=f16, device=x.device)
    _lib.call("fz_upsample2x_nhwc_f16", _p(x), _p(out), NB, H, W, Cc, _stream())
    return out


def concat_channels(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    _chk(a, f16, "concat"); _chk(b, f16, "concat")
    rows = a.numel() // a.shape[-1]
    out = torch.empty((*a.shape[:-1], a.shape[-1] + b.shape[-1]), dtype=f16, device=a.device)
    _lib.call("fz_concat_channels_f16", _p(a), a.shape[-1], _p(b), b.shape[-1], _p(out), rows, _stream())
    return out


def im2col_latents(x: torch.Tensor) -> torch.Tensor:
    """latents [B,Cl,F,H,W] fp32 -> [B*F*H*W, 64] fp16."""
    _chk(x, torch.float32, "im2col_latents")
    B, Cl, F, H, W = x.shape
    out = torch.empty((B * F * H * W, 64), dtype=f16, device=x.device)
    _lib.call("fz_im2col_latents_f16", _p(x.contiguous()), _p(out), B, Cl, F, H, W, _stream())
    return out


def out_temporal(y: torch.Tensor, B: int, Co: int, F: int, H: int, W: int, down=None, up=None, w_full=None, b_full=None) -> torch.Tensor:
    """y [B*F*H*W, ld] fp16 (Co valid) -> eps [B,Co,F,H,W] fp32 with the conv_out temporal conv applied."""
    eps = torch.empty((B, Co, F, H, W), dtype=torch.float32, device=y.device)
    rank = 0 if down is None else down.shape[0]
    _lib.call("fz_out_temporal_f32", _p(y), y.stride(0), _p(eps), B, Co, F, H * W, _p(down), _p(up), rank, _p(w_full), _p(b_full), _stream())
    return eps


def rowvec_linear(x: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor], silu_in: bool) -> torch.Tensor:
    N, K = w16.shape
    y = torch.empty((N,), dtype=torch.float32, device=x.device)
    _lib.call("fz_rowvec_linear", _p(x), _p(w16), _p(bias), _p(y), N, K, int(silu_in), _stream())
    return y


def timestep_sinusoid(t: float, c0: int, flip: bool, freq_shift: float, device) -> torch.Tensor:
    out = torch.empty((c0,), dtype=torch.float32, device=device)
    _lib.call("fz_timestep_sinusoid", float(t), _p(out), c0, int(flip), float(freq_shift), _stream())
    return out


def temporal_attn(qkv: torch.Tensor, B: int, F: int, HW: int, heads: int, d: int, scale: float) -> torch.Tensor:
    _chk(qkv, f16, "temporal_attn")
    out = torch.empty((B * F * HW, heads * d), dtype=f16, device=qkv.device)
    _lib.call("fz_temporal_attn_f16", _p(qkv), _p(out), B, F, HW, heads, d, float(scale), _stream())
    return out


def ddim_invert_step(x: torch.Tensor, eps: torch.Tensor, a_prev: float, a_next: float):
    _lib.call("fz_ddim_invert_step", _p(x), _p(eps), x.numel(), float(a_prev), float(a_next), _stream())


def cfg_ddim_step(x: torch.Tensor, eps2: torch.Tensor, guidance: float, a_t: float, a_prev: float, x_inv=None, mask_a=None, mask_b=None,
                  apply_blend: bool = False):
    fhw = x.shape[-3] * x.shape[-2] * x.shape[-1]
    _lib.call("fz_cfg_ddim_step", _p(x), _p(eps2), x.numel(), float(guidance), float(a_t), float(a_prev), _p(x_inv), _p(mask_a), _p(mask_b),
              fhw, int(apply_blend), _stream())


def cfg_ddim_step_batched(x: torch.Tensor, eps2: torch.Tensor, guidance: float, a_t: float, a_prev: float, x_inv=None,
                          blends: Optional[Sequence[Optional[dict]]] = None):
    """x [K, 4, F, h, w] fp32 (K prompts), eps2 [2K, ...] = [uncond_1..K ; cond_1..K]; blends: one latent_blend_args() dict (or None) per
    item, all sharing x_inv."""
    K = x.shape[0]
    fhw = x.shape[-3] * x.shape[-2] * x.shape[-1]
    blends = list(blends) if blends is not None else [None] * K
    assert len(blends) == K and eps2.shape[0] == 2 * K
    ma = (C.c_void_p * K)(*[None if b is None else b["mask_a"].data_ptr() for b in blends])
    mb = (C.c_void_p * K)(*[None if b is None or b["mask_b"] is None else b["mask_b"].data_ptr() for b in blends])
    ap = (C.c_int * K)(*[int(b is not None and bool(b["apply_blend"])) for b in blends])
    _lib.call("fz_cfg_ddim_step_batched", _p(x), _p(eps2), K, x.numel() // K, float(guidance), float(a_t), float(a_prev), _p(x_inv), ma, mb, ap,
              fhw, _stream())


def cfg_ddim_step_multi(x: torch.Tensor, eps2: torch.Tensor, guidance: float, a_t: float, a_prev: float,
                        blends: Optional[Sequence[Optional[dict]]] = None):
    """x [K, 4, F, h, w] fp32 (K items, possibly of different clips), eps2 [2K, ...] = [uncond_1..K ; cond_1..K]; blends: one
    latent_blend_args() dict (or None) per item, each with the x_inv of its own clip."""
    K = x.shape[0]
    fhw = x.shape[-3] * x.shape[-2] * x.shape[-1]
    blends = list(blends) if blends is not None else [None] * K
    assert len(blends) == K and eps2.shape[0] == 2 * K
    xi = (C.c_void_p * K)(*[None if b is None else b["x_inv"].data_ptr() for b in blends])
    ma = (C.c_void_p * K)(*[None if b is None else b["mask_a"].data_ptr() for b in blends])
    mb = (C.c_void_p * K)(*[None if b is None or b["mask_b"] is None else b["mask_b"].data_ptr() for b in blends])
    ap = (C.c_int * K)(*[int(b is not None and bool(b["apply_blend"])) for b in blends])
    _lib.call("fz_cfg_ddim_step_multi", _p(x), _p(eps2), K, x.numel() // K, float(guidance), float(a_t), float(a_prev), xi, ma, mb, ap, fhw,
              _stream())


def _same_map_geometry(maps: Sequence[torch.Tensor], what: str):
    """The map kernels read every map with the first one's [F, heads, r*r] and row stride and average over maps x heads: a map of another
    head count (SD-2.x stores 5 / 10 / 20 heads at different levels) would be misread and misweighted."""
    m0 = maps[0]
    for m in maps[1:]:
        if m.shape[:3] != m0.shape[:3] or m.stride(2) != m0.stride(2) or m.dtype != m0.dtype:
            raise ValueError(f"fatezero_b200.ops.{what}: maps of different geometry {tuple(m.shape)} vs {tuple(m0.shape)} in one call")


def blend_mask(maps: Sequence[torch.Tensor], word_w: torch.Tensor, th: float, h: int, w: int) -> torch.Tensor:
    """maps: list of [F, heads, r*r, ld] (fp16 cache slabs or fp16 running sums) -> mask [F, h, w] float 0/1."""
    m0 = maps[0]
    Fm, heads, rr, ld = m0.shape
    _same_map_geometry(maps, "blend_mask")
    r = int(round(rr ** 0.5))
    arr = (C.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
    ww = [float(v) for v in word_w.tolist()]
    wv = (C.c_float * len(ww))(*ww)
    out = torch.empty((Fm, h, w), dtype=torch.float32, device=m0.device)
    _lib.call("fz_blend_mask", arr, len(maps), int(m0.dtype == torch.float32), Fm, heads, r, m0.stride(2), min(len(ww), 77), wv,
              float(th), h, w, _p(out), _stream())
    return out


def softmax_rows_(x: torch.Tensor, scale: float) -> torch.Tensor:
    """x [rows, n] fp16 (row stride multiple of 8) <- softmax(scale * x) row-wise, in place."""
    _chk(x, f16, "softmax_rows")
    rows, n = x.shape
    assert x.stride(1) == 1
    _lib.call("fz_softmax_rows_f16", _p(x), rows, n, x.stride(0), float(scale), _stream())
    return x


def embed_tokens(tok: torch.Tensor, pos: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    """tok [V, C] fp32, pos [L, C] fp32, ids [B, L] int64 (CUDA) -> [B*L, C] fp16."""
    B, L = ids.shape
    out = torch.empty((B * L, tok.shape[1]), dtype=f16, device=tok.device)
    _lib.call("fz_embed_tokens_f16", _p(tok), _p(pos), _p(ids.contiguous()), _p(out), B * L, L, tok.shape[1], _stream())
    return out


def quick_gelu_(x: torch.Tensor) -> torch.Tensor:
    _chk(x, f16, "quick_gelu")
    assert x.is_contiguous()
    _lib.call("fz_quick_gelu_f16", _p(x), x.numel(), _stream())
    return x


def gelu_(x: torch.Tensor) -> torch.Tensor:
    """Exact (erf) GELU in place: the MLP activation of SD-2 text encoders (hidden_act "gelu")."""
    _chk(x, f16, "gelu")
    assert x.is_contiguous()
    _lib.call("fz_gelu_f16", _p(x), x.numel(), _stream())
    return x


def frames_to_u8(x: torch.Tensor) -> torch.Tensor:
    """decoded frames [N, 3, H, W] fp32 / fp16 in [-1, 1] -> uint8 [N, H, W, 3], bitwise numpy_to_pil's bytes."""
    if x.dtype not in (torch.float32, f16):
        raise TypeError(f"fatezero_b200.ops.frames_to_u8: expected float32 or float16, got {x.dtype}")
    _chk(x, x.dtype, "frames_to_u8")
    N, c, H, W = x.shape
    if c != 3:
        raise ValueError(f"fatezero_b200.ops.frames_to_u8: {c} channels (RGB expected)")
    x = x.contiguous()
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=x.device)
    _lib.call("fz_frames_to_u8", _p(x), int(x.dtype == f16), _p(out), N, H, W, _stream())
    return out


def resize_bicubic_u8(img: torch.Tensor, tables, crop_bottom_square: bool = False) -> torch.Tensor:
    """img [N, H, W, 3] uint8 -> [N, Ho, Wo, 3] uint8 with PIL's bicubic resample.  tables: device dict(kx, bx, ky, by) of
    clip_eval.resize_tables for the (cropped) input size."""
    _chk(img, torch.uint8, "resize_bicubic_u8")
    N, H, W, c = img.shape
    assert c == 3 and img.is_contiguous()
    kx, bx, ky, by = tables["kx"], tables["bx"], tables["ky"], tables["by"]
    for t in (kx, bx, ky, by):
        _chk(t, torch.int32, "resize_bicubic_u8")
        assert t.is_contiguous()
    Wo, Ho = kx.shape[0], ky.shape[0]
    hc = W if crop_bottom_square and H > W else H
    tmp = torch.empty((N, hc, Wo, 3), dtype=torch.uint8, device=img.device)
    out = torch.empty((N, Ho, Wo, 3), dtype=torch.uint8, device=img.device)
    _lib.call("fz_resize_bicubic_u8", _p(img), N, H, W, int(crop_bottom_square), _p(kx), _p(bx), kx.shape[1], Wo, _p(ky), _p(by), ky.shape[1],
              Ho, _p(tmp), _p(out), _stream())
    return out


def clip_patchify(img: torch.Tensor, res: int, patch: int, mean: Sequence[float], std: Sequence[float]) -> torch.Tensor:
    """resized uint8 [N, Hr, Wr, 3] -> CenterCrop(res) + ToTensor + Normalize as fp16 conv1 im2col rows [N*(res/patch)^2, 3*patch^2]."""
    _chk(img, torch.uint8, "clip_patchify")
    N, Hr, Wr, c = img.shape
    assert c == 3 and img.is_contiguous()
    g = res // patch if patch > 0 else 0
    out = torch.empty((max(N * g * g, 1), 3 * patch * patch), dtype=f16, device=img.device)
    _lib.call("fz_clip_patchify_f16", _p(img), N, Hr, Wr, int(res), int(patch), (C.c_float * 3)(*map(float, mean)),
              (C.c_float * 3)(*map(float, std)), _p(out), _stream())
    return out


def clip_embed(patches: torch.Tensor, class_emb: torch.Tensor, pos_emb: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float,
               N: int) -> torch.Tensor:
    """patch-GEMM rows [N*(T-1), C] fp16 -> ln_pre(cat(class, patches) + pos) [N*T, C] fp16 (T = pos_emb rows)."""
    _chk(patches, f16, "clip_embed")
    for t in (class_emb, pos_emb, gamma, beta):
        _chk(t, torch.float32, "clip_embed")
    T, Cc = pos_emb.shape
    assert patches.is_contiguous() and patches.shape == (N * (T - 1), Cc)
    out = torch.empty((N * T, Cc), dtype=f16, device=patches.device)
    _lib.call("fz_clip_embed_f16", _p(patches), _p(class_emb.contiguous()), _p(pos_emb.contiguous()), _p(gamma), _p(beta), float(eps), N, T, Cc,
              _p(out), _stream())
    return out


def clip_scores(img: torch.Tensor, txt: torch.Tensor, clip_frames: Sequence[int], pairs: Sequence[Sequence[int]], scale: float) -> dict:
    """img [N, D] / txt [P, D] fp32 features; clip_frames [K]; pairs [K] x (source row, target row) -> dict of fp32 device tensors
    (success int32): img_norm, txt_norm, logits [N, 2], probs [N, 2], success, margin, cosine [N], clip_mean [K]."""
    _chk(img, torch.float32, "clip_scores"); _chk(txt, torch.float32, "clip_scores")
    N, D = img.shape
    P = txt.shape[0]
    assert txt.shape[1] == D and img.is_contiguous() and txt.is_contiguous()
    K = len(clip_frames)
    dev = img.device
    o = dict(img_norm=torch.empty(N, device=dev), txt_norm=torch.empty(P, device=dev), logits=torch.empty(N, 2, device=dev),
             probs=torch.empty(N, 2, device=dev), success=torch.empty(N, dtype=torch.int32, device=dev), margin=torch.empty(N, device=dev),
             cosine=torch.empty(N, device=dev), clip_mean=torch.empty(max(K, 1), device=dev))
    fr = (C.c_int * max(K, 1))(*[int(f) for f in clip_frames])
    pr = (C.c_int * max(2 * K, 1))(*[int(v) for pq in pairs for v in pq])
    _lib.call("fz_clip_scores", _p(img), _p(txt), N, P, D, fr, pr, K, float(scale), *(_p(o[k]) for k in
              ("img_norm", "txt_norm", "logits", "probs", "success", "margin", "cosine", "clip_mean")), _stream())
    return o


def cross_heatmaps(maps: Sequence[torch.Tensor], ntok: int) -> torch.Tensor:
    """maps: cross-attention running sums [F, heads, r*r, ld] (fp16 or fp32) of ONE resolution -> uint8 [F, ntok, r, r] heat maps."""
    m0 = maps[0]
    Fm, heads, rr, _ = m0.shape
    _same_map_geometry(maps, "cross_heatmaps")
    r = int(round(rr ** 0.5))
    arr = (C.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
    out = torch.empty((Fm, ntok, r, r), dtype=torch.uint8, device=m0.device)
    _lib.call("fz_cross_heatmaps", arr, len(maps), int(m0.dtype == torch.float32), Fm, heads, r, m0.stride(2), int(ntok), _p(out), _stream())
    return out


def attention(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, out: torch.Tensor, *, S_q: int, keys_per_slot: int, n_src: int, d: int,
              heads: int, F: int, BF: int, scale: float, src_index: Sequence[Sequence[int]], edit_bf_start: int = 0,
              row_mode: int = _lib.ATTN_NONE, store=None, base=None, cache_ld: int = 0, acc=None, xedit=None, mask=None, dbg=None,
              causal: bool = False, groups: Optional[Sequence[dict]] = None):
    """q/k: strided 2-D views (rows, ld) whose column h*d starts head h; vt [n_src, heads, d, vt_ld]; out [BF*S_q, ldo].
    groups (batched edits and inversions): one dict(row_mode=, mask=, acc=, xedit=, store=, base=) per row group of F rows after
    edit_bf_start; a group without `store` / `base` uses the slab given here.  row_mode / acc / xedit / mask must then be left at their
    defaults."""
    a = AttnArgs()
    a.q, a.ldq = _p(q), q.stride(0)
    a.k, a.ldk = _p(k), k.stride(0)
    a.vt, a.vt_ld = _p(vt), vt.stride(2)
    a.out, a.ldo = _p(out), out.stride(0)
    a.S_q, a.keys_per_slot, a.n_slots, a.n_src = S_q, keys_per_slot, len(src_index), n_src
    a.d, a.heads, a.F, a.BF = d, heads, F, BF
    a.scale = float(scale)
    flat = [int(v) for row in src_index for v in row]
    arr = (C.c_int * len(flat))(*flat)
    a.src_index = arr
    a.edit_bf_start, a.row_mode = edit_bf_start, row_mode
    a.store, a.base, a.cache_ld = _p(store), _p(base), cache_ld
    a.acc, a.acc_ld = _p(acc), (acc.stride(2) if acc is not None else 0)
    a.xedit, a.mask = _p(xedit), _p(mask)
    a.dbg = _p(dbg)
    a.causal = int(causal)
    if groups is None:
        _lib.call("fz_attention_f16", C.byref(a), _stream())
        return out
    if row_mode != _lib.ATTN_NONE or acc is not None or xedit is not None or mask is not None:
        raise ValueError("fatezero_b200.ops.attention: with groups=, the hook arguments belong to the groups")
    if not 1 <= len(groups) <= _lib.MAX_ATTN_GROUPS:
        raise ValueError(f"fatezero_b200.ops.attention: {len(groups)} groups (1..{_lib.MAX_ATTN_GROUPS})")
    gs = _lib.AttnGroups()
    gs.n_groups = len(groups)
    for i, g in enumerate(groups):
        gs.g[i].row_mode = int(g.get("row_mode", _lib.ATTN_NONE))
        gs.g[i].xedit, gs.g[i].mask, gs.g[i].acc = _p(g.get("xedit")), _p(g.get("mask")), _p(g.get("acc"))
        if g.get("acc") is not None:
            a.acc_ld = g["acc"].stride(2)
    if all(g.get("store") is None and g.get("base") is None for g in groups):
        _lib.call("fz_attention_grouped_f16", C.byref(a), C.byref(gs), _stream())
        return out
    sl = _lib.AttnSlabs()
    for i, g in enumerate(groups):
        sl.store[i], sl.base[i] = _p(g.get("store")), _p(g.get("base"))
    _lib.call("fz_attention_grouped_slabs_f16", C.byref(a), C.byref(gs), C.byref(sl), _stream())
    return out
