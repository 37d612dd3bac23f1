"""Non-square clips for the parity tests: the cases and their single-forward inputs.  Kept apart from oracle/cases.py::CASES, which the
square-clip tests iterate over; the goldens use the compact format of oracle/sd2.py (strided latent samples, map sums and slices).

At the mini UNet geometry a 32x48 latent has levels 32x48, 16x24, 8x12 and 4x6: the first holds 1536 pixels and is not stored (the store
threshold S <= 32**2 of attention_store.py:82), so the stored down_cross list starts at the 16x24 level.

Reference goldens (NONSQUARE_REF_CASES) come from the unmodified reference without blend words: its SpatialBlender asserts square maps
(spatial_blend.py:94-96), and its heat maps (visualization.py:14-31) find no map of res**2 pixels on a non-square clip, so the harness
skips that call.  Blend cases on non-square clips (NONSQUARE_ORACLE_CASES) have no reference behaviour; they are checked against the
restatement below only: OracleEditNS is fz_oracle.OracleEdit whose blend masks are built on the rh x rw grid of each map, recovered from
the clip's latent size with level_hw, by the reference's steps (word-weighted mean over maps and heads, 3x3 max-pool, F.interpolate's
nearest resize, whose source index is taken per axis, per-frame max, threshold)."""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.nn.functional as F

from fatezero_b200 import synth
from oracle import fz_oracle as fo
from oracle.cases import SRC

_MC = dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128)

NONSQUARE_CASES = {
    # landscape: Refine + Reweight (config #1-like) on 32x48 latents (256x384 pixels)
    "ns_landscape_refine": dict(
        unet="mini", model_config=_MC, frames=3, h=32, w=48, steps=4, source=SRC, target="watercolor painting of " + SRC,
        p2p=dict(is_replace_controller=False, cross_replace_steps={"default_": 0.8}, self_replace_steps=0.8,
                 eq_params={"words": ["watercolor"], "values": [10, 10]})),
    # portrait: Replace on 48x32 latents
    "ns_portrait_replace": dict(
        unet="mini", model_config=_MC, frames=2, h=48, w=32, steps=3, source=SRC,
        target="a silver car driving down a curvy road in the countryside",
        p2p=dict(is_replace_controller=True, cross_replace_steps={"default_": 0.7}, self_replace_steps=0.6)),
    # oracle only: Replace + self-attention mask blend + latent blend on 64x96 latents (the blender's maps are the 16x24 level)
    "ns_replace_blend": dict(
        ref=False, unet="mini", model_config=_MC, frames=2, h=64, w=96, steps=5, source=SRC,
        target="a Porsche car driving down a curvy road in the countryside",
        p2p=dict(is_replace_controller=True, cross_replace_steps={"default_": 0.5}, self_replace_steps=0.6,
                 blend_words=[["silver", "jeep"], ["Porsche", "car"]], blend_self_attention=True, blend_latents=True,
                 blend_th=[0.985, 0.985])),
}
NONSQUARE_REF_CASES = [k for k, v in NONSQUARE_CASES.items() if v.get("ref", True)]
NONSQUARE_ORACLE_CASES = [k for k, v in NONSQUARE_CASES.items() if not v.get("ref", True)]


def case_inputs(case: dict) -> torch.Tensor:
    return synth.synth_latents(case["frames"], case["h"], case["w"]) * 0.5


def fwd_inputs(case: dict, x0: torch.Tensor):
    """The single-forward pin: a CFG batch of two 2-frame clips at 481, text from seed 2."""
    x2 = torch.cat([x0, 0.7 * x0])[:, :, :2]
    emb = torch.randn(2, 77, synth.UNET_CONFIGS[case["unet"]]["cross_attention_dim"], generator=torch.Generator().manual_seed(2))
    return x2, 481, emb


def level_hw(S: int, h: int, w: int) -> Tuple[int, int]:
    """(rh, rw) of the UNet level k with (h >> k) * (w >> k) == S in a clip of h x w latents."""
    for k in range(max(h, w).bit_length()):
        if min(h >> k, w >> k) >= 1 and (h >> k) * (w >> k) == S:
            return h >> k, w >> k
    raise ValueError(f"no level of a {h} x {w} latent holds {S} pixels")


def blend_mask(maps5: List[torch.Tensor], word_alpha: torch.Tensor, th: float, h: int, w: int, latent_hw: Tuple[int, int]) -> torch.Tensor:
    """fz_oracle.blend_mask (spatial_blend.py:24-39, use_pool=True, ONE prompt) on the maps' rh x rw grid.  Returns bool [F, h, w]."""
    stack = []
    for m in maps5:
        f, heads, rr, _ = m.shape
        rh, rw = level_hw(rr, *latent_hw)
        stack.append((m.float() * word_alpha[None, None, None, :]).sum(-1).reshape(f, heads, rh, rw).permute(1, 0, 2, 3))
    maps = torch.cat(stack, dim=0).mean(0)  # [F, rh, rw]   (mean over layers*heads)
    maps = F.max_pool2d(maps[None], (3, 3), (1, 1), padding=(1, 1))
    mask = F.interpolate(maps, size=(h, w))[0]
    mask = mask / mask.amax(dim=(-2, -1), keepdim=True)
    return mask.gt(th)


class OracleEditNS(fo.OracleEdit):
    """fz_oracle.OracleEdit on a clip of latent_hw latents: the self-attention blend mask is made on each layer's own grid, the latent blend
    mask at the latent size, both from maps whose grid level_hw recovers.  Everything else is OracleEdit's."""

    def __init__(self, plan: fo.EditPlan, inv: fo.OracleStore, latent_hw: Tuple[int, int]):
        super().__init__(plan, inv)
        self.latent_hw = (int(latent_hw[0]), int(latent_hw[1]))

    def forward(self, attn, is_cross, place):
        pl = self.plan
        if is_cross or not pl.blend_self or attn.shape[-2] > 32 ** 2 or not (pl.self_window[0] <= self.cur_step < pl.self_window[1]):
            return super().forward(attn, is_cross, place)
        # OracleEdit.forward's self-attention blend, on the layer's rh x rw grid
        self.store(attn, is_cross, place)
        key = f"{place}_self"
        pos = self.pos[key]
        self.pos[key] += 1
        step_in_store = len(self.inv.all_step) - self.cur_step - 1
        base = self.inv.all_step[step_in_store][key][pos]
        rr = attn.shape[-2]
        rh, rw = level_hw(rr, *self.latent_hw)
        m = blend_mask(self._blend_maps(self.inv.all_step[step_in_store]), pl.blend_src, pl.th[0], rh, rw, self.latent_hw)
        m = m.float().reshape(m.shape[0], 1, rr, 1)
        return m * attn + (1 - m) * base

    def step_callback(self, x_t):
        """OracleEdit.step_callback (attention_util.py:47-78) with the latent blend's masks made by blend_mask above."""
        pl = self.plan
        if not pl.blend_lat:
            return super().step_callback(x_t)
        self.cur_step += 1
        self.between_steps()
        self.latents_store.append(x_t.clone())
        step_in_store = len(self.inv.latents_store) - self.cur_step
        x_inv = self.inv.latents_store[step_in_store]
        src = self._blend_maps(self.inv.all_step[step_in_store])
        tgt = self._blend_maps(self.attention_store)  # running sums of the pre-edit target maps
        h, w = x_t.shape[-2:]
        m_src = blend_mask(src, pl.blend_src, pl.th[0], h, w, self.latent_hw)
        m_tgt = blend_mask(tgt, pl.blend_tgt, pl.th[0], h, w, self.latent_hw)
        m = (m_src | m_tgt).float()
        self.mask_list.append(m_src.float())
        self.lat_counter += 1
        if pl.lat_window[0] < self.lat_counter < pl.lat_window[1]:
            return x_inv + m[None, None] * (x_t - x_inv)
        return x_t
