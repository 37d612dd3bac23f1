"""Cross-attention heat-map strips (reference: prompt_attention/visualization.py:14-72).  Off the timed path; reads the
controller's `get_average_attention()` exactly like the reference does, so the HBM cache keeps its Python-visible layout."""
from __future__ import annotations

import os
import time
from typing import List

import numpy as np
import torch


def aggregate_attention(prompts, attention_store, res: int, from_where: List[str], is_cross: bool, select: int) -> torch.Tensor:
    """Mean over all stored maps of resolution `res` (layers x heads) -> [frames, res, res, tokens] on the host."""
    picked = []
    maps = attention_store.get_average_attention()
    want = res * res
    kind = "cross" if is_cross else "self"
    for place in from_where:
        for item in maps.get(f"{place}_{kind}", []):
            if item.dim() == 4 and item.shape[2] == want:
                t, heads, _, tok = item.shape
                picked.append(item.float().reshape(len(prompts), t, heads, res, res, tok)[select])
            elif item.dim() == 3 and item.shape[1] == want:
                picked.append(item.float().reshape(len(prompts), -1, res, res, item.shape[-1])[select])
    if not picked:
        raise ValueError(f"no stored {kind}-attention map at resolution {res}")
    stacked = torch.cat(picked, dim=-4)
    return (stacked.sum(-4) / stacked.shape[-4]).cpu()


def _caption(image: np.ndarray, text: str) -> np.ndarray:
    h, w, c = image.shape
    pad = int(h * 0.2)
    canvas = np.full((h + pad, w, c), 255, dtype=np.uint8)
    canvas[:h] = image
    try:
        import cv2
        font = cv2.FONT_HERSHEY_SIMPLEX
        size = cv2.getTextSize(text, font, 1, 2)[0]
        cv2.putText(canvas, text, ((w - size[0]) // 2, h + pad - size[1] // 2), font, 1, (0, 0, 0), 2)
    except Exception:
        pass
    return canvas


def device_heatmaps(attention_store, res: int, from_where: List[str], ntok: int):
    """uint8 [frames, ntok, res, res] computed on the GPU straight from the controller's cross-attention running sums (fz_cross_heatmaps),
    or None when the store is not one of this package's controllers holding device slabs (then the reference's host path is used)."""
    acc = getattr(attention_store, "_acc", None)
    if not acc or len(getattr(attention_store, "attention_store_all_step", [])) == 0 and attention_store.cur_step == 0:
        return None
    picked = [t for place in from_where for t in acc.get(f"{place}_cross", []) if t is not None and t.is_cuda and t.dim() == 4
              and t.shape[2] == res * res]
    if not picked or len(picked) > 8:
        return None
    from . import ops
    with torch.cuda.device(picked[0].device):
        return ops.cross_heatmaps(picked, ntok)


def show_cross_attention(tokenizer, prompts, attention_store, res: int, from_where: List[str], select: int = 0, save_path=None):
    """Returns one H x (W*tokens) x 3 uint8 strip per frame (what p2p_validation_loop stacks into the attention GIF).  With this package's
    controllers the per-token heat maps are produced on the GPU from the running cross-attention sums (only frames x tokens x res^2 BYTES
    reach the host); any other store goes through the reference's get_average_attention() path."""
    from PIL import Image
    if isinstance(prompts, str):
        prompts = [prompts]
    tokens = tokenizer.encode(prompts[select])
    heat_u8 = device_heatmaps(attention_store, res, from_where, len(tokens)) if len(prompts) == 1 or select == 0 else None
    if heat_u8 is not None:
        maps = heat_u8.permute(0, 2, 3, 1).cpu()  # [frames, res, res, tokens] uint8
    else:
        maps = aggregate_attention(prompts, attention_store, res, from_where, True, select)
        if maps.dim() == 3:
            maps = maps[None]
    strips = []
    for frame in maps:
        tiles = []
        for i, tok in enumerate(tokens):
            heat = frame[:, :, i]
            if heat.dtype != torch.uint8:  # an all-zero map is black (0/0 would be NaN, whose uint8 cast is undefined)
                heat = (255 * heat / heat.max()).nan_to_num(0.0).clamp(0, 255)
            heat = heat.numpy().astype(np.uint8)
            tile = np.array(Image.fromarray(np.repeat(heat[:, :, None], 3, axis=2)).resize((256, 256)))
            tiles.append(_caption(tile, tokenizer.decode(int(tok))))
        strips.append(np.concatenate(tiles, axis=1))
    if save_path is not None:
        os.makedirs(save_path, exist_ok=True)
        stamp = time.strftime("%Y-%m-%dT%H-%M-%S")
        for j, strip in enumerate(strips):
            Image.fromarray(strip).save(os.path.join(save_path, f"{stamp}_{j:02d}.png"))
    return strips
