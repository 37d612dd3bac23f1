"""VAE encode / decode on the sm_90a kernels (SURVEY.md §8(f) rank 1): the `AutoencoderKL` the reference brackets its hot path with
(`pipelines/p2p_ddim_spatial_temporal.py:88-96`: `vae.encode(image).latent_dist.sample(generator)`; `pipelines/stable_diffusion.py:297-319`:
`vae.decode(latents).sample` in chunks of 16 frames).

`VaeEngine` executes the SD-1.x VAE (diffusers 0.11.1 `AutoencoderKL`: DownEncoderBlock2D / UNetMidBlock2D with a single-head 512-wide
AttentionBlock / UpDecoderBlock2D, GroupNorm(32, eps 1e-6) + SiLU, no time embedding) with the kernels of libfatezero_b200.so:
  * every 3x3 conv is the tap-GEMM (`fz_conv3x3_nhwc_f16`; images wider than 128 pixels are tiled in row segments whose width is the
    largest divisor of the output width up to 128: 128 at 256 / 512 / 640 / 768, 96 at 192 / 288 / 576, 80 at 160 / 320, 72 at 144;
    the encoder's downsample is the right/bottom-padded stride-2 variant `fz_conv3x3_down_asym_nhwc_f16`), 1x1 shortcuts and attention projections are
    `fz_gemm_f16`, the RGB / latent input convs go through the im2col GEMM like the UNet's conv_in;
  * GroupNorm(+SiLU), nearest upsampling: the UNet's HBM-bound kernels;
  * the mid-block attention (one head of width 512: more than the fused attention kernel holds in registers) runs per image as
    GEMM (Q K^T) -> `fz_softmax_rows_f16` -> GEMM (P V^T with V^T produced directly by a GEMM with swapped operands; the value bias is
    added after P V, exact because the probabilities of a row sum to one).
fp16 storage / fp32 accumulation, fp32 in and out.  `AutoencoderKL` below is a parameter container with the diffusers state-dict names and
the `encode(...).latent_dist.sample(generator)` / `decode(...).sample` surface, so it can be handed to the pipeline as `vae`; the pipeline
also wraps a foreign AutoencoderKL-shaped module (diffusers) that lives on the GPU (`pipeline._vae()`).
Numerics are checked against an fp32 torch restatement (oracle/vae_oracle.py, tests/test_gpu_vae.py), every kernel call of encode / decode
against fp64 at 512 and 768 pixels and every block against an independent fp64 restatement (tests/test_gpu_vae_blocks.py); neither
restatement is pinned to the real diffusers package (absent offline) — see DESIGN.md §5."""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict, Optional

import torch
from torch import nn

from . import ops

f16, f32 = torch.float16, torch.float32

SD14_VAE_CONFIG = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4,
                       norm_num_groups=32, sample_size=512)
_ATTN_ALIASES = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}  # newer diffusers releases renamed these


def vae_param_spec(cfg: dict) -> "OrderedDict[str, tuple]":
    """name -> shape for every tensor of the AutoencoderKL state dict (diffusers 0.11.1 names)."""
    ch = list(cfg["block_out_channels"])
    lpb, lat = cfg["layers_per_block"], cfg["latent_channels"]
    spec: "OrderedDict[str, tuple]" = OrderedDict()

    def conv(n, ci, co, k=3):
        spec[n + ".weight"], spec[n + ".bias"] = (co, ci, k, k), (co,)

    def vec(n, c):
        spec[n + ".weight"], spec[n + ".bias"] = (c,), (c,)

    def resnet(n, ci, co):
        vec(n + ".norm1", ci); conv(n + ".conv1", ci, co); vec(n + ".norm2", co); conv(n + ".conv2", co, co)
        if ci != co:
            conv(n + ".conv_shortcut", ci, co, 1)

    def mid(n, c):
        resnet(n + ".resnets.0", c, c)
        vec(n + ".attentions.0.group_norm", c)
        for q in ("query", "key", "value", "proj_attn"):
            spec[f"{n}.attentions.0.{q}.weight"], spec[f"{n}.attentions.0.{q}.bias"] = (c, c), (c,)
        resnet(n + ".resnets.1", c, c)

    conv("encoder.conv_in", cfg["in_channels"], ch[0])
    co = ch[0]
    for i, c in enumerate(ch):
        ci, co = co, c
        for j in range(lpb):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", ci if j == 0 else co, co)
        if i != len(ch) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", co, co)
    mid("encoder.mid_block", ch[-1])
    vec("encoder.conv_norm_out", ch[-1])
    conv("encoder.conv_out", ch[-1], 2 * lat)
    conv("quant_conv", 2 * lat, 2 * lat, 1)
    conv("post_quant_conv", lat, lat, 1)
    rev = list(reversed(ch))
    conv("decoder.conv_in", lat, rev[0])
    mid("decoder.mid_block", rev[0])
    co = rev[0]
    for i, c in enumerate(rev):
        ci, co = co, c
        for j in range(lpb + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", ci if j == 0 else co, co)
        if i != len(ch) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", co, co)
    vec("decoder.conv_norm_out", rev[-1])
    conv("decoder.conv_out", rev[-1], cfg["out_channels"])
    return spec


class DiagonalGaussianDistribution:
    """diffusers models/vae.py DiagonalGaussianDistribution (mean | logvar moments, logvar clamped to [-30, 20])."""

    def __init__(self, moments: torch.Tensor):
        self.parameters = moments
        self.mean, self.logvar = torch.chunk(moments, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        dev = self.parameters.device
        gdev = generator.device if generator is not None else dev
        noise = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.mean.dtype).to(dev)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class _Out(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class VaeEngine:
    def __init__(self, state_dict: Dict[str, torch.Tensor], cfg: dict, device: torch.device):
        if torch.device(device).type != "cuda":
            raise RuntimeError("VaeEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.dev = torch.device(device)
        self.cfg = dict(cfg)
        self.ch = list(cfg["block_out_channels"])
        self.lpb = int(cfg["layers_per_block"])
        self.lat = int(cfg["latent_channels"])
        self.groups = int(cfg["norm_num_groups"])
        if any(c % 8 or c % self.groups for c in self.ch):
            raise NotImplementedError(f"VAE channel counts {self.ch} must be multiples of 8 and of the group count")
        sd = {}
        for k, v in state_dict.items():
            for new, old in _ATTN_ALIASES.items():
                k = k.replace(f".attentions.0.{new}.", f".attentions.0.{old}.")
            sd[k] = v.detach()
        missing = [k for k in vae_param_spec(self.cfg) if k not in sd]
        if missing:
            raise KeyError(f"VAE state dict lacks {len(missing)} tensors (first: {missing[0]})")
        w: Dict[str, torch.Tensor] = {}
        dev = self.dev

        def h(t):
            return t.to(dev, f16).contiguous()

        def f(t):
            return t.to(dev, f32).contiguous()

        def im2col_w(t):  # [Cout, Cin, 3, 3] with Cin*9 <= 64 -> [Cout, 64], column = tap * Cin + c (the layout fz_im2col_latents_f16 writes)
            co, ci = t.shape[:2]
            m = torch.zeros(co, 64)
            m[:, : 9 * ci] = t.float().permute(0, 2, 3, 1).reshape(co, 9 * ci)
            return h(m)

        def pad16(t9, b):  # a conv with a handful of output channels runs as one 16-wide MMA tile
            co = t9.shape[1]
            w9 = torch.zeros(9, 16, t9.shape[2])
            w9[:, :co] = t9
            return h(w9), f(torch.nn.functional.pad(b.float(), (0, 16 - co)))

        for name, t in sd.items():
            if name in ("encoder.conv_in.weight", "decoder.conv_in.weight"):
                w[name] = im2col_w(t)
            elif name == "decoder.conv_out.weight":
                w[name], w["decoder.conv_out.bias"] = pad16(t.float().permute(2, 3, 0, 1).reshape(9, t.shape[0], t.shape[1]), sd["decoder.conv_out.bias"])
            elif name == "encoder.conv_out.weight":
                # quant_conv (1x1) composed into conv_out: both are linear and the 1x1 follows the 3x3, so W' = Wq W, b' = Wq b + bq exactly
                wq, bq = sd["quant_conv.weight"].float().reshape(2 * self.lat, 2 * self.lat), sd["quant_conv.bias"].float()
                t2 = torch.einsum("om,mikl->oikl", wq, t.float())
                b2 = wq @ sd["encoder.conv_out.bias"].float() + bq
                w[name], w["encoder.conv_out.bias"] = pad16(t2.permute(2, 3, 0, 1).reshape(9, t2.shape[0], t2.shape[1]), b2)
            elif name in ("decoder.conv_out.bias", "encoder.conv_out.bias", "quant_conv.weight", "quant_conv.bias"):
                continue
            elif name.endswith(".weight") and t.dim() == 4 and t.shape[-1] == 3:
                w[name] = h(t.permute(2, 3, 0, 1).reshape(9, t.shape[0], t.shape[1]))
            elif name.endswith(".weight") and t.dim() == 4:
                w[name] = h(t.reshape(t.shape[0], t.shape[1])) if not name.startswith("post_quant") else f(t.reshape(t.shape[0], t.shape[1]))
            elif name.endswith(".weight") and t.dim() == 2:
                w[name] = h(t)
            else:
                w[name] = f(t)
        # fused q|k projection of the two mid-block attentions
        for side in ("encoder", "decoder"):
            a = f"{side}.mid_block.attentions.0."
            w[a + "qk.weight"] = h(torch.cat([sd[a + "query.weight"], sd[a + "key.weight"]], 0))
            w[a + "qk.bias"] = f(torch.cat([sd[a + "query.bias"], sd[a + "key.bias"]], 0))
        self.w = w

    # ---- blocks ---------------------------------------------------------------------------------------------------------
    def _gn(self, n: str, x: torch.Tensor, silu: bool) -> torch.Tensor:
        NB, H, W, C = x.shape
        return ops.groupnorm(x.view(NB, H * W, C), self.w[n + ".weight"], self.w[n + ".bias"], 1e-6, self.groups, 1, silu).view(NB, H, W, C)

    def _resnet(self, n: str, x: torch.Tensor) -> torch.Tensor:
        w = self.w
        NB, H, W, Cin = x.shape
        hcur = ops.conv3x3(self._gn(n + ".norm1", x, True), w[n + ".conv1.weight"], bias=w[n + ".conv1.bias"])
        Cout = hcur.shape[-1]
        sc = x
        if n + ".conv_shortcut.weight" in w:
            sc = ops.gemm(x.view(-1, Cin), w[n + ".conv_shortcut.weight"], bias=w[n + ".conv_shortcut.bias"]).view(NB, H, W, Cout)
        return ops.conv3x3(self._gn(n + ".norm2", hcur, True), w[n + ".conv2.weight"], bias=w[n + ".conv2.bias"], residual=sc)

    def _attn(self, n: str, x: torch.Tensor) -> torch.Tensor:
        w = self.w
        NB, H, W, C = x.shape
        S = H * W
        xn = self._gn(n + ".group_norm", x, False).view(NB * S, C)
        qk = ops.gemm(xn, w[n + ".qk.weight"], bias=w[n + ".qk.bias"])                       # [NB*S, 2C]
        o = torch.empty((NB * S, C), dtype=f16, device=self.dev)
        for i in range(NB):
            rows = slice(i * S, (i + 1) * S)
            s = ops.gemm(qk[rows, :C], qk[rows, C:])                                          # Q K^T  [S, S]
            ops.softmax_rows_(s, 1.0 / math.sqrt(C))                                          # (q c)(k c)^T with c = C^-1/4 each
            vt = ops.gemm(w[n + ".value.weight"], xn[rows])                                   # V^T (bias-free) [C, S]: operands swapped
            ops.gemm(s, vt, bias=w[n + ".value.bias"], out=o[rows])                           # P V + b_v (rows of P sum to one)
        return ops.gemm(o, w[n + ".proj_attn.weight"], bias=w[n + ".proj_attn.bias"], residual=x.view(NB * S, C)).view(NB, H, W, C)

    def _mid(self, n: str, x: torch.Tensor) -> torch.Tensor:
        return self._resnet(n + ".resnets.1", self._attn(n + ".attentions.0", self._resnet(n + ".resnets.0", x)))

    def _conv_in(self, name: str, x_nchw: torch.Tensor) -> torch.Tensor:
        N, Cc, H, W = x_nchw.shape
        cols = ops.im2col_latents(x_nchw.to(f32).permute(1, 0, 2, 3)[None].contiguous())    # [N*H*W, 64]
        return ops.gemm(cols, self.w[name + ".weight"], bias=self.w[name + ".bias"]).view(N, H, W, -1)

    def _down(self, n: str, x: torch.Tensor) -> torch.Tensor:  # Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)), 3x3 conv stride 2
        return ops.conv3x3(x, self.w[n + ".conv.weight"], bias=self.w[n + ".conv.bias"], stride=2, asym_pad=True)

    def _up(self, n: str, x: torch.Tensor) -> torch.Tensor:  # Upsample2D: nearest 2x, 3x3 conv
        return ops.conv3x3(ops.upsample2x(x), self.w[n + ".conv.weight"], bias=self.w[n + ".conv.bias"])

    def _encoder_out(self, x: torch.Tensor) -> torch.Tensor:
        """conv_norm_out + SiLU + conv_out with quant_conv folded in -> moments [N, 2*latent, H, W] fp32."""
        w = self.w
        y = ops.conv3x3(self._gn("encoder.conv_norm_out", x, True), w["encoder.conv_out.weight"], bias=w["encoder.conv_out.bias"])
        return y[..., : 2 * self.lat].permute(0, 3, 1, 2).float().contiguous()

    def _decoder_in(self, z: torch.Tensor) -> torch.Tensor:
        """post_quant_conv (4x4 per pixel, fp32) + decoder conv_in: latents [N, latent, h, w] -> [N, h, w, C] fp16."""
        w = self.w
        z = torch.einsum("oc,nchw->nohw", w["post_quant_conv.weight"], z.to(self.dev, f32)) + w["post_quant_conv.bias"][None, :, None, None]
        return self._conv_in("decoder.conv_in", z)

    def _decoder_out(self, x: torch.Tensor) -> torch.Tensor:
        """conv_norm_out + SiLU + conv_out -> images [N, 3, H, W] fp32."""
        w = self.w
        y = ops.conv3x3(self._gn("decoder.conv_norm_out", x, True), w["decoder.conv_out.weight"], bias=w["decoder.conv_out.bias"])
        return y[..., : self.cfg["out_channels"]].permute(0, 3, 1, 2).float().contiguous()

    # ---- public ---------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode_moments(self, images: torch.Tensor) -> torch.Tensor:
        """images [N, 3, H, W] (CUDA, any float dtype, values in [-1, 1]) -> moments [N, 2*latent, H/8, W/8] fp32 (mean | logvar)."""
        with torch.cuda.device(self.dev):
            x = self._conv_in("encoder.conv_in", images.to(self.dev))
            for i in range(len(self.ch)):
                for j in range(self.lpb):
                    x = self._resnet(f"encoder.down_blocks.{i}.resnets.{j}", x)
                if i != len(self.ch) - 1:
                    x = self._down(f"encoder.down_blocks.{i}.downsamplers.0", x)
            return self._encoder_out(self._mid("encoder.mid_block", x))

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """latents [N, latent, h, w] (already divided by the 0.18215 scaling factor by the caller) -> images [N, 3, 8h, 8w] fp32."""
        with torch.cuda.device(self.dev):
            x = self._mid("decoder.mid_block", self._decoder_in(z))
            for i in range(len(self.ch)):
                for j in range(self.lpb + 1):
                    x = self._resnet(f"decoder.up_blocks.{i}.resnets.{j}", x)
                if i != len(self.ch) - 1:
                    x = self._up(f"decoder.up_blocks.{i}.upsamplers.0", x)
            return self._decoder_out(x)


class _Config(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class AutoencoderKL(nn.Module):
    """Parameter container with diffusers' AutoencoderKL state-dict names and call surface; encode / decode run on `VaeEngine`."""

    def __init__(self, **kwargs):
        super().__init__()
        cfg = dict(SD14_VAE_CONFIG)
        cfg.update(kwargs)
        cfg["block_out_channels"] = tuple(cfg["block_out_channels"])
        self._internal_dict = _Config(cfg)
        for name, shape in vae_param_spec(cfg).items():
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            t = torch.ones(shape) if (len(shape) == 1 and "norm" in name and name.endswith("weight")) else (
                torch.zeros(shape) if len(shape) == 1 else torch.empty(shape).uniform_(-fan_in ** -0.5, fan_in ** -0.5))
            mod = self
            parts = name.split(".")
            for part in parts[:-1]:
                if part not in mod._modules:
                    mod.add_module(part, nn.Module())
                mod = mod._modules[part]
            mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))
        self._engine = None

    @property
    def config(self):
        return self._internal_dict

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        self._engine = None
        renamed = {}
        for k, v in state_dict.items():
            for new, old in _ATTN_ALIASES.items():
                k = k.replace(f".attentions.0.{new}.", f".attentions.0.{old}.")
            renamed[k] = v
        return super().load_state_dict(renamed, strict=strict, **kw)

    def engine(self) -> VaeEngine:
        if self._engine is None:
            self._engine = VaeEngine(self.state_dict(), dict(self.config), self.device)
        return self._engine

    def encode(self, x: torch.Tensor, return_dict: bool = True):
        dist = DiagonalGaussianDistribution(self.engine().encode_moments(x).to(x.dtype if x.is_floating_point() else f32))
        return _Out(latent_dist=dist) if return_dict else (dist,)

    def decode(self, z: torch.Tensor, return_dict: bool = True):
        img = self.engine().decode(z).to(z.dtype)
        return _Out(sample=img) if return_dict else (img,)

    def forward(self, sample, sample_posterior: bool = False, generator=None):
        post = self.encode(sample).latent_dist
        return self.decode(post.sample(generator) if sample_posterior else post.mode())


def engine_for(vae) -> Optional[VaeEngine]:
    """A VaeEngine for a foreign AutoencoderKL-shaped module living on the GPU (e.g. diffusers'), or None when `vae` is not one."""
    if isinstance(vae, AutoencoderKL):
        return vae.engine()
    if not isinstance(vae, nn.Module):
        return None
    try:
        p = next(vae.parameters())
    except StopIteration:
        return None
    sd = vae.state_dict()
    if not p.is_cuda or "encoder.conv_in.weight" not in sd or "decoder.conv_out.weight" not in sd:
        return None
    cfg = dict(SD14_VAE_CONFIG)
    src = getattr(vae, "config", {})
    for k in ("in_channels", "out_channels", "block_out_channels", "layers_per_block", "latent_channels", "norm_num_groups"):
        v = src.get(k) if isinstance(src, dict) else getattr(src, k, None)
        if v is not None:
            cfg[k] = v
    try:
        return VaeEngine(sd, cfg, p.device)
    except (KeyError, NotImplementedError):
        return None
