"""SpatialBlender — binary blend masks from cached cross-attention maps (reference: prompt_attention/spatial_blend.py).

Same constructor / attributes as the reference class (`alpha_layers`, `th`, `start_blend`, `end_blend`, `counter`, `mask_list`,
`prompt_choose`).  The mask itself is produced on the GPU by fz_blend_mask_hw straight from the HBM map cache: mean over the five
16x16 cross maps x 8 heads of the blend-word probability, 3x3 max-pool, nearest resize, per-frame max normalisation, FIXED
threshold th[0] (spatial_blend.py:24-39 — no Otsu in the reference, see SURVEY.md App. B.1).

Non-square clips: the reference asserts square maps (spatial_blend.py:94-96).  Here a map's rh x rw grid is recovered from the clip's
latent size with level_hw, and the mask is built on that grid by the same steps (the max-pool and the nearest resize per axis)."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops, tables


def level_hw(S: int, h: int, w: int) -> Tuple[int, int]:
    """(rh, rw) of the UNet level that holds S pixels per frame in a clip of h x w latents: level k holds (h >> k) x (w >> k) pixels."""
    k = 0
    while (h >> k) >= 1 and (w >> k) >= 1:
        if (h >> k) * (w >> k) == S:
            return h >> k, w >> k
        k += 1
    raise ValueError(f"no UNet level of a {h} x {w} latent holds {S} pixels")


class SpatialBlender:
    def __init__(self, prompts: List[str], words, substruct_words=None, start_blend: float = 0.2, end_blend: float = 0.8,
                 th=(0.9, 0.9), tokenizer=None, NUM_DDIM_STEPS: Optional[int] = None, save_path: Optional[str] = None,
                 prompt_choose: str = "source"):
        if prompt_choose not in ("source", "both"):
            raise AssertionError("choose to generate the mask by only source prompt or both the source and target")
        if substruct_words is not None:
            raise NotImplementedError("substruct_words is never passed by make_controller (SURVEY.md App. E5)")
        self.count = 0
        self.MAX_NUM_WORDS = 77
        self.NUM_DDIM_STEPS = NUM_DDIM_STEPS
        self.save_path = save_path
        self.prompt_choose = prompt_choose
        alpha_layers = torch.zeros(len(prompts), 1, 1, 1, 1, self.MAX_NUM_WORDS)
        for i, (prompt, words_) in enumerate(zip(prompts, words)):
            if isinstance(words_, str):
                words_ = [words_]
            for word in words_:
                ind = tables.get_word_inds(prompt, word, tokenizer)
                alpha_layers[i, :, :, :, :, ind] = 1
        self.alpha_layers = alpha_layers  # host tensor: the one-hot rows are kernel arguments
        self.substruct_layers = None
        self.start_blend = int(start_blend * self.NUM_DDIM_STEPS)
        self.end_blend = int(end_blend * self.NUM_DDIM_STEPS)
        self.counter = 0
        self.th = th
        self.mask_list: List[torch.Tensor] = []

    def word_row(self, prompt_index: int) -> torch.Tensor:
        return self.alpha_layers[prompt_index].reshape(-1)

    @staticmethod
    def select_maps(attention_store: Dict[str, Sequence[torch.Tensor]]) -> List[torch.Tensor]:
        """spatial_blend.py:78 hard-codes the five 16x16 maps (three 24x24 maps at 768^2): down_cross[2:4] + up_cross[:3] of what was
        stored."""
        maps = list(attention_store["down_cross"][2:4]) + list(attention_store["up_cross"][:3])
        if len({m.shape[-2] for m in maps}) != 1:
            raise RuntimeError("SpatialBlender needs cross maps of one resolution (latent 64x64 or 96x96; SURVEY.md App. B.14)")
        return maps

    def mask_from(self, attention_store, prompt_index: int, h: int, w: int, latent_hw: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """[F, h, w] float {0,1} for one prompt's maps (each [F, heads, rh*rw, >=77]).  latent_hw: the clip's latent size, from which the
        maps' rh x rw grid is recovered (level_hw); None: square maps, as the reference asserts."""
        maps = self.select_maps(attention_store)
        hw = None if latent_hw is None else level_hw(maps[0].shape[-2], int(latent_hw[0]), int(latent_hw[1]))
        return ops.blend_mask(maps, self.word_row(prompt_index), float(self.th[0]), h, w, hw=hw)

    def __call__(self, attention_store, step_in_store: Optional[int] = None, target_h=None, target_w=None, x_t=None):
        """Reference-compatible entry (spatial_blend.py:58-124).  Maps may be 4-D ([F,h,s,77], one prompt) or 5-D ([P,F,h,s,77])."""
        if target_h is None and target_w is None and x_t is not None:
            target_h, target_w = x_t.shape[-2:]
        latent_hw = tuple(x_t.shape[-2:]) if x_t is not None else None
        self.counter += 1
        first = attention_store["down_cross"][0] if len(attention_store["down_cross"]) else attention_store["up_cross"][0]
        if first.dim() == 5:
            per_prompt = [{k: [m[i] for m in v] for k, v in attention_store.items()} for i in range(first.shape[0])]
        else:
            per_prompt = [attention_store]
        if self.prompt_choose == "source":
            mask = self.mask_from(per_prompt[0], 0, target_h, target_w, latent_hw)[None]
        else:
            if len(per_prompt) != 2:
                raise AssertionError("If using both source and target prompt")
            m0 = self.mask_from(per_prompt[0], 0, target_h, target_w, latent_hw)
            m1 = self.mask_from(per_prompt[1], 1, target_h, target_w, latent_hw)
            mask = torch.stack([m0, torch.maximum(m0, m1)], 0)  # mask[:1] + mask on booleans
        self.mask_list.append(mask[0][:, None, :, :].float())
        if x_t is not None:
            m = mask[:, None, ...] if x_t.dim() == 5 else mask
            if self.start_blend < self.counter < self.end_blend:
                x_t = x_t[:1] + m * (x_t - x_t[:1])
            return x_t
        return mask
