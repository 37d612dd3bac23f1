"""Stable Diffusion 2.x base geometry for the parity tests: the cases, the oracle's SD-2 restatement and the compact golden format.

SD-2.x UNets differ from SD-1.x in three ways the oracle has to follow (diffusers 0.11.1 semantics, as in the reference):
  * `attention_head_dim` is the head COUNT per block, one entry per down block (5 / 10 / 20 / 20: head dim 64 at every level); down
    block i uses entry i, the mid block the last entry, up block i the reversed list's entry i (unet_3d_condition.py:115-116,164,195,217),
    so every transformer runs the entry of its resolution level;
  * `use_linear_projection`: proj_in / proj_out are nn.Linear [C, C] on the (h w) tokens (models/attention.py:63-66,90-93,112-114,130-132);
  * 1024-wide text (cross_attention_dim).
OracleUNetSD2 restates both on top of fz_oracle.OracleUNet: a Linear over the channel axis of every pixel is the 1x1 convolution with
the same [C, C] matrix, so the linear weights are handed to the conv path as [C, C, 1, 1]; the head count is set per transformer.

Golden files (oracle/make_sd2_golden.py) are kept small: every latent of a trajectory is kept as a fixed strided sample (every
LAT_STRIDE-th element of the flattened tensor) plus float64 sums and sums of squares; the single-forward epsilon as every
EPS_STRIDE-th element; stored maps as sums / sums of squares plus a few (frame 0, first two heads, first 32 query rows, first 128 keys)
slices; blend masks as uint8.
The SD-2-base case also keeps, in full, the reference latents a teacher-forced run starts its steps from; the samples of those
steps are not stored twice (tests/_sd2_golden.py takes them from the full tensors)."""
from __future__ import annotations

from typing import Dict

import torch

from oracle import fz_oracle as fo
from oracle.cases import SRC

SD2_CASES = {
    # config #1-like: Refine + Reweight with ['mid'] K/V frames at the mini SD-2 geometry (heads 1 / 2 / 4 / 4, d = 64)
    "sd2mini_refine": dict(
        unet="sd2mini", model_config=dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128),
        frames=3, size=32, steps=4, source=SRC, target="watercolor painting of " + SRC,
        p2p=dict(is_replace_controller=False, cross_replace_steps={"default_": 0.8}, self_replace_steps=0.8,
                 eq_params={"words": ["watercolor"], "values": [10, 10]})),
    # Replace + self-attention mask blend + latent blend at 64x64 latents (the blender's 16x16 maps: 4 heads at the mini geometry)
    "sd2mini_replace_blend": dict(
        unet="sd2mini", model_config=dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128),
        frames=2, size=64, steps=5, source=SRC, target="a Porsche car driving down a curvy road in the countryside",
        p2p=dict(is_replace_controller=True, cross_replace_steps={"default_": 0.5}, self_replace_steps=0.6,
                 blend_words=[["silver", "jeep"], ["Porsche", "car"]], blend_self_attention=True, blend_latents=True,
                 blend_th=[0.985, 0.985])),
    # SD-2-base geometry (heads 5 / 10 / 20 / 20): Replace + self-attention mask blend, 2 frames of 64x64 latents, 2 + 2 steps (at 2 steps
    # the latent blend's window int(0.2 N) < counter < int(0.8 N) is empty: its masks are computed and compared, the blend itself is
    # covered by sd2mini_replace_blend).  big=True: the GPU test compares the product with this golden directly
    "sd2_replace_blend": dict(
        big=True, unet="sd2", model_config=dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=640),
        frames=2, size=64, steps=2, source=SRC, target="a Porsche car driving down a curvy road in the countryside",
        p2p=dict(is_replace_controller=True, cross_replace_steps={"default_": 0.7}, self_replace_steps=0.7,
                 blend_words=[["silver", "jeep"], ["Porsche", "car"]], blend_self_attention=True, blend_latents=True,
                 blend_th=[0.985, 0.985])),
}
SD2_MINI_CASES = [k for k, v in SD2_CASES.items() if not v.get("big")]

LAT_STRIDE = 8
EPS_STRIDE = 8
MAP_SLICES = 3  # maps of step 0 kept as [frame 0, heads 0..1, query rows 0..31, keys 0..127] slices


def sample(t: torch.Tensor, stride: int) -> torch.Tensor:
    return t.detach().float().cpu().reshape(-1)[::stride].clone()


def fwd_inputs(case: dict, x0: torch.Tensor):
    """The single-forward pin: a CFG batch of two 2-frame clips at 481, 1024-wide text from seed 2."""
    x2 = torch.cat([x0, 0.7 * x0])[:, :, :2]
    emb = torch.randn(2, 77, 1024, generator=torch.Generator().manual_seed(2))
    return x2, 481, emb


def map_slice(t: torch.Tensor) -> torch.Tensor:
    return t[0, :2, :32, :128]


def level_of(prefix: str, nblk: int) -> int:
    """Resolution level of a transformer from its state-dict prefix."""
    if prefix.startswith("down_blocks."):
        return int(prefix.split(".")[1])
    if prefix.startswith("up_blocks."):
        return nblk - 1 - int(prefix.split(".")[1])
    return nblk - 1


class OracleUNetSD2(fo.OracleUNet):
    """fz_oracle.OracleUNet with per-level heads and linear projections (see the module docstring)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], unet_config: dict, model_config: dict):
        super().__init__(state_dict, unet_config, model_config)
        hd = self.cfg["attention_head_dim"]
        self.level_heads = [int(hd)] * len(self.ch) if isinstance(hd, int) else [int(h) for h in hd]
        if self.cfg.get("use_linear_projection", False):
            for k in list(self.w):
                if k.endswith((".proj_in.weight", ".proj_out.weight")) and self.w[k].dim() == 2:
                    self.w[k] = self.w[k][:, :, None, None]

    def transformer(self, p, x, text, place):
        self.heads = self.level_heads[level_of(p, len(self.ch))]
        return super().transformer(p, x, text, place)
