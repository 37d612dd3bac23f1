"""UNetPseudo3DConditionModel — drop-in parameter container + forward entry of the reference UNet
(video_diffusion/models/unet_3d_condition.py:37-501, unet_3d_blocks.py, resnet.py, attention.py, lora.py).

The module owns fp32 parameters under EXACTLY the reference's state-dict names / shapes (SURVEY.md App. E3), so
`from_2d_model` / `load_2d_state_dict` / `load_state_dict` accept Stable-Diffusion-1.x and Tune-A-Video checkpoints
unchanged, and so do Stable-Diffusion-2.x base configurations (per-block `attention_head_dim`, `use_linear_projection`,
`upcast_attention`, 1024-wide text).  `forward` does not run PyTorch layers: it hands the tensors to `engine.UNetEngine`, which executes the
step with the sm_90a kernels of libfatezero_b200.so (there is no CPU / eager fallback).
"""
from __future__ import annotations

import glob
import json
import math
import os
from collections import OrderedDict
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn


class _Config(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class UNetPseudo3DConditionOutput(dict):
    """Supports both `.sample` and `["sample"]` (the reference uses both: p2p_ddim_spatial_temporal.py:142 / :397)."""

    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


def lora_rank(requested: int, channels: int) -> int:
    """lora.py:26-28: rank falls back to min(in,out)//2 when larger than the channel count."""
    return requested if requested <= channels else channels // 2


def level_heads(cfg: dict) -> List[int]:
    """Attention heads of the transformers at each resolution level.  `attention_head_dim` is the head COUNT per block (diffusers 0.11.1
    semantics, unet_3d_condition.py:115-116,164,195,217 -> unet_3d_blocks.py:177-179): one int for every block (SD-1.x: 8) or one entry
    per down block (SD-2.x: 5 / 10 / 20 / 20, head dim 64).  Down block i uses entry i, the mid block the last entry and up block i the
    reversed list's entry i, so every block at level l runs entry l."""
    ch = list(cfg["block_out_channels"])
    hd = cfg["attention_head_dim"]
    heads = [int(hd)] * len(ch) if isinstance(hd, int) else [int(h) for h in hd]
    if len(heads) != len(ch) or any(h < 1 or c % h for h, c in zip(heads, ch)):
        raise ValueError(f"attention_head_dim {hd!r} does not give a head count dividing each of block_out_channels {tuple(ch)}")
    return heads


def transformer_heads(cfg: dict) -> "OrderedDict[str, int]":
    """State-dict prefix of every transformer of the UNet (forward order) -> its head count (level_heads)."""
    heads = level_heads(cfg)
    nblk = len(heads)
    lpb = int(cfg["layers_per_block"])
    out: "OrderedDict[str, int]" = OrderedDict()
    for i, t in enumerate(cfg["down_block_types"]):
        if t.startswith("CrossAttn"):
            for j in range(lpb):
                out[f"down_blocks.{i}.attentions.{j}"] = heads[i]
    out["mid_block.attentions.0"] = heads[-1]
    for i, t in enumerate(cfg["up_block_types"]):
        if t.startswith("CrossAttn"):
            for j in range(lpb + 1):
                out[f"up_blocks.{i}.attentions.{j}"] = heads[nblk - 1 - i]
    return out


def unet_param_spec(cfg: dict, model_config: dict) -> "OrderedDict[str, Tuple[tuple, str]]":
    """name -> (shape, init kind) for every tensor of the reference state dict (902 tensors for SD-1.4 + lora:160)."""
    spec: "OrderedDict[str, Tuple[tuple, str]]" = OrderedDict()
    ch = list(cfg["block_out_channels"])
    c0 = ch[0]
    temb = 4 * c0
    dtext = cfg["cross_attention_dim"]
    linear_proj = bool(cfg.get("use_linear_projection", False))
    lpb = cfg["layers_per_block"]
    mc = model_config or {}

    def conv(name, cin, cout, k):
        spec[f"{name}.weight"] = ((cout, cin, k, k), "fan_in")
        spec[f"{name}.bias"] = ((cout,), f"bias:{cin * k * k}")
        if k > 1:
            if "lora" in mc:
                r = lora_rank(int(mc["lora"]), cout)
                spec[f"{name}.conv_temporal.down.weight"] = ((r, cout, 3), f"normal:{1.0 / r}")
                spec[f"{name}.conv_temporal.up.weight"] = ((cout, r, 3), "zeros")
            else:
                spec[f"{name}.conv_temporal.weight"] = ((cout, cout, k), "dirac")
                spec[f"{name}.conv_temporal.bias"] = ((cout,), "zeros")

    def linear(name, cin, cout, bias=True):
        spec[f"{name}.weight"] = ((cout, cin), "fan_in")
        if bias:
            spec[f"{name}.bias"] = ((cout,), f"bias:{cin}")

    def norm(name, c):
        spec[f"{name}.weight"] = ((c,), "ones")
        spec[f"{name}.bias"] = ((c,), "zeros")

    def resnet(name, cin, cout):
        norm(f"{name}.norm1", cin)
        conv(f"{name}.conv1", cin, cout, 3)
        linear(f"{name}.time_emb_proj", temb, cout)
        norm(f"{name}.norm2", cout)
        conv(f"{name}.conv2", cout, cout, 3)
        if cin != cout:
            conv(f"{name}.conv_shortcut", cin, cout, 1)

    def transformer(name, c):
        norm(f"{name}.norm", c)
        # use_linear_projection (SD-2.x): proj_in / proj_out are nn.Linear [C, C] instead of 1x1 convs (models/attention.py:63-66,90-93)
        if linear_proj:
            linear(f"{name}.proj_in", c, c)
        else:
            conv(f"{name}.proj_in", c, c, 1)
        b = f"{name}.transformer_blocks.0"
        for proj in ("to_q", "to_k", "to_v"):
            linear(f"{b}.attn1.{proj}", c, c, bias=False)
        linear(f"{b}.attn1.to_out.0", c, c)
        norm(f"{b}.norm1", c)
        linear(f"{b}.attn2.to_q", c, c, bias=False)
        linear(f"{b}.attn2.to_k", dtext, c, bias=False)
        linear(f"{b}.attn2.to_v", dtext, c, bias=False)
        linear(f"{b}.attn2.to_out.0", c, c)
        norm(f"{b}.norm2", c)
        for proj in ("to_q", "to_k", "to_v"):
            linear(f"{b}.attn_temporal.{proj}", c, c, bias=False)
        spec[f"{b}.attn_temporal.to_out.0.weight"] = ((c, c), "zeros")  # models/attention.py:224
        spec[f"{b}.attn_temporal.to_out.0.bias"] = ((c,), f"bias:{c}")
        norm(f"{b}.norm_temporal", c)
        linear(f"{b}.ff.net.0.proj", c, 8 * c)
        linear(f"{b}.ff.net.2", 4 * c, c)
        norm(f"{b}.norm3", c)
        if linear_proj:
            linear(f"{name}.proj_out", c, c)
        else:
            conv(f"{name}.proj_out", c, c, 1)

    conv("conv_in", cfg["in_channels"], c0, 3)
    linear("time_embedding.linear_1", c0, temb)
    linear("time_embedding.linear_2", temb, temb)
    out_c = c0
    for i, btype in enumerate(cfg["down_block_types"]):
        in_c, out_c = out_c, ch[i]
        for j in range(lpb):
            resnet(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c)
        if btype.startswith("CrossAttn"):
            for j in range(lpb):
                transformer(f"down_blocks.{i}.attentions.{j}", out_c)
        if i != len(ch) - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", out_c, out_c, 3)
    resnet("mid_block.resnets.0", ch[-1], ch[-1])
    transformer("mid_block.attentions.0", ch[-1])
    resnet("mid_block.resnets.1", ch[-1], ch[-1])
    rev = list(reversed(ch))
    out_c = rev[0]
    for i, btype in enumerate(cfg["up_block_types"]):
        prev_c, out_c = out_c, rev[i]
        in_c = rev[min(i + 1, len(ch) - 1)]
        for j in range(lpb + 1):
            skip_c = in_c if j == lpb else out_c
            r_in = prev_c if j == 0 else out_c
            resnet(f"up_blocks.{i}.resnets.{j}", r_in + skip_c, out_c)
        if btype.startswith("CrossAttn"):
            for j in range(lpb + 1):
                transformer(f"up_blocks.{i}.attentions.{j}", out_c)
        if i != len(ch) - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", out_c, out_c, 3)
    norm("conv_norm_out", c0)
    conv("conv_out", c0, cfg["out_channels"], 3)
    return spec


def _init_tensor(shape, kind: str) -> torch.Tensor:
    if kind == "ones":
        return torch.ones(shape)
    if kind == "zeros":
        return torch.zeros(shape)
    if kind == "dirac":
        t = torch.zeros(shape)
        nn.init.dirac_(t)
        return t
    if kind == "fan_in":
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        bound = 1.0 / math.sqrt(fan_in)
        return torch.empty(shape).uniform_(-bound, bound)
    if kind.startswith("bias:"):
        bound = 1.0 / math.sqrt(int(kind.split(":")[1]))
        return torch.empty(shape).uniform_(-bound, bound)
    if kind.startswith("normal:"):
        return torch.randn(shape) * float(kind.split(":")[1])
    raise ValueError(kind)


def _attach(root: nn.Module, dotted: str, value: nn.Parameter):
    mod = root
    parts = dotted.split(".")
    for part in parts[:-1]:
        if part not in mod._modules:
            mod.add_module(part, nn.Module())
        mod = mod._modules[part]
    mod.register_parameter(parts[-1], value)


_SD_DEFAULTS = dict(
    sample_size=None, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True, freq_shift=0,
    down_block_types=("CrossAttnDownBlockPseudo3D", "CrossAttnDownBlockPseudo3D", "CrossAttnDownBlockPseudo3D", "DownBlockPseudo3D"),
    mid_block_type="UNetMidBlockPseudo3DCrossAttn",
    up_block_types=("UpBlockPseudo3D", "CrossAttnUpBlockPseudo3D", "CrossAttnUpBlockPseudo3D", "CrossAttnUpBlockPseudo3D"),
    only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2, downsample_padding=1,
    mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5, cross_attention_dim=1280, attention_head_dim=8,
    dual_cross_attention=False, use_linear_projection=False, class_embed_type=None, num_class_embeds=None, upcast_attention=False,
    resnet_time_scale_shift="default",
)
_MODEL_CONFIG_KEYS = ("lora", "SparseCausalAttention_index", "least_sc_channel", "temporal_downsample", "temporal_downsample_time")


class UNetPseudo3DConditionModel(nn.Module):
    """Drop-in for the reference's UNetPseudo3DConditionModel (SD-1.x and SD-2.x base configurations).

    `upcast_attention=True` is accepted and changes nothing: every attention kernel forms Q.K^T from fp16 operands with fp32
    accumulation and runs the softmax in fp32, which is what upcasting asks of an fp16 model.  Only epsilon-prediction checkpoints are
    meaningful (the reference's DDIM inversion assumes epsilon); v-prediction (SD-2.x 768-v) checkpoints load but are not converted."""

    def __init__(self, **kwargs):
        super().__init__()
        cfg = dict(_SD_DEFAULTS)
        cfg.update(kwargs)
        self._internal_dict = _Config(cfg)
        self.model_config = {k: cfg[k] for k in _MODEL_CONFIG_KEYS if k in cfg}
        self._check_supported(cfg)
        self.sample_size = cfg["sample_size"]
        self._spec = unet_param_spec(cfg, self.model_config)
        for name, (shape, kind) in self._spec.items():
            _attach(self, name, nn.Parameter(_init_tensor(shape, kind), requires_grad=False))
        self._engine = None
        self._controller = None
        self.num_upsamplers = len(cfg["block_out_channels"]) - 1

    @staticmethod
    def _check_supported(cfg):
        def bad(msg):
            raise NotImplementedError(f"fatezero_b200 UNet: {msg} is not on the FateZero SD-1.x hot path")
        if cfg["dual_cross_attention"]:
            bad("dual_cross_attention")
        if cfg["class_embed_type"] is not None or cfg["num_class_embeds"] is not None:
            bad("class embeddings")
        if cfg["resnet_time_scale_shift"] != "default":
            bad("resnet_time_scale_shift != 'default'")
        if cfg.get("temporal_downsample") or cfg.get("temporal_downsample_time"):
            bad("temporal_downsample (commented out in every shipped YAML)")
        if cfg["only_cross_attention"] not in (False, [False] * 4, (False,) * 4):
            bad("only_cross_attention")
        level_heads(cfg)
        if cfg["center_input_sample"]:
            bad("center_input_sample")
        if cfg["act_fn"] not in ("silu", "swish"):
            bad(f"act_fn {cfg['act_fn']}")

    # ---- diffusers-style surface ---------------------------------------------------------------------------------
    @property
    def config(self):
        return self._internal_dict

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def set_controller(self, controller):
        """Called by prompt_attention.register_attention_control (attention_register.py:14)."""
        self._controller = controller

    def invalidate_engine(self):
        self._engine = None

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        self._engine = None
        return super().load_state_dict(state_dict, strict=strict, **kw)

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def engine(self):
        if self._engine is None:
            from .engine import UNetEngine
            self._engine = UNetEngine(self)
        return self._engine

    def set_frame_shard(self, rank: int, world: int, group=None):
        """Split the frames of one clip over `world` GPUs (SURVEY.md §8(e)): every rank then calls forward with ITS frames
        [B, 4, F/world, H, W]; the engine all-gathers K/V and all-reduces the joint-frame GroupNorm statistics over `group`."""
        self.engine().set_frame_shard(rank, world, group)

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, attention_mask=None, return_dict: bool = True):
        if class_labels is not None or attention_mask is not None:
            raise NotImplementedError("class_labels / attention_mask are not supported (attention_register.py:146-151)")
        if not sample.is_cuda:
            raise RuntimeError("fatezero_b200.UNetPseudo3DConditionModel runs on CUDA (sm_90a) only; move the model and inputs to "
                               "the GPU — there is no CPU fallback")
        t = float(timestep.item()) if torch.is_tensor(timestep) else float(timestep)
        if sample.device != self.device:
            raise RuntimeError(f"sample lives on {sample.device} but the UNet parameters on {self.device}")
        # every launch, workspace and controller slab of the forward belongs to the UNet's device, whatever the caller's current device is
        with torch.cuda.device(self.device):
            eps = self.engine().forward(sample, t, encoder_hidden_states, self._controller)
        eps = eps.to(sample.dtype) if sample.dtype != torch.float32 else eps
        if not return_dict:
            return (eps,)
        return UNetPseudo3DConditionOutput(eps)

    # ---- checkpoints (unet_3d_condition.py:448-501) -----------------------------------------------------------------
    @classmethod
    def from_2d_model(cls, model_path, model_config):
        config_path = os.path.join(model_path, "config.json")
        if not os.path.isfile(config_path):
            raise RuntimeError(f"{config_path} does not exist")
        with open(config_path, "r") as f:
            config = json.load(f)
        config.pop("_class_name", None)
        config.pop("_diffusers_version", None)
        rename = {"CrossAttnDownBlock2D": "CrossAttnDownBlockPseudo3D", "DownBlock2D": "DownBlockPseudo3D",
                  "UpBlock2D": "UpBlockPseudo3D", "CrossAttnUpBlock2D": "CrossAttnUpBlockPseudo3D"}
        config["down_block_types"] = [rename.get(b, b) for b in config["down_block_types"]]
        config["up_block_types"] = [rename.get(b, b) for b in config["up_block_types"]]
        if model_config is not None:
            config.update(model_config)
        model = cls(**config)
        candidates = glob.glob(os.path.join(model_path, "*.bin"))
        if candidates:
            state_dict = torch.load(candidates[0], map_location="cpu")
            model.load_2d_state_dict(state_dict=state_dict)
        return model

    def load_2d_state_dict(self, state_dict, **kwargs):
        own = self.state_dict()
        for k, v in state_dict.items():
            if k not in own:
                raise KeyError(f"2d state_dict key {k} does not exist in 3d model")
            if v.shape != own[k].shape:
                raise ValueError(f"state_dict shape mismatch, 2d {v.shape}, 3d {own[k].shape}")
        for k in own:
            if "_temporal" in k:
                continue
            if k not in state_dict:
                raise KeyError(f"3d state_dict key {k} does not exist in 2d model")
        own.update(state_dict)
        self.load_state_dict(own, **kwargs)
