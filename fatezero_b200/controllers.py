"""Attention controllers with the reference's Python surface (prompt_attention/attention_store.py, attention_util.py) driving
the fused kernels instead of rewriting probability tensors in Python.

Reference mechanism: `register_attention_control` monkeypatches every attention `forward`; the closure materialises
softmax(QK^T) and calls `controller(attn, is_cross, place)` 32 times per UNet forward; AttentionStore deep-copies the maps
(32x32 ones to host RAM), AttentionControlEdit overwrites the cond half in place.
Here: the UNet engine asks the controller, per hooked layer, for *kernel arguments* (`self_attn_args` / `cross_attn_args`);
the maps live in an HBM cache owned by the controller (torch tensors, so `attention_store_all_step[i][key][j]`,
`attention_store` and `get_average_attention()` keep their Python-visible layout), and fz_attention_f16 performs the STORE /
REPLACE / mask-BLEND / cross-edit inline.  State machine semantics (cur_step bookkeeping in step_callback, per-key position
counters, mirrored step indexing, off-by-one latent index of the latent blend) follow SURVEY.md App. A / App. B exactly.
"""
from __future__ import annotations

import abc
import copy
import os
import time
import warnings
from typing import Dict, List, Optional, Tuple, Union

import torch

from . import _lib, tables
from .spatial_blend import SpatialBlender

KEYS = ("down_cross", "mid_cross", "up_cross", "down_self", "mid_self", "up_self")
CROSS_LD = 80  # 77 text tokens padded so cache rows are 16-byte multiples (TMA store / vector access)
f16 = torch.float16


def _key(place: str, is_cross: bool) -> str:
    return f"{place}_{'cross' if is_cross else 'self'}"


class EmptyControl:
    """attention_util.py:26-37"""

    def step_callback(self, x_t):
        return x_t

    def between_steps(self):
        return

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        return attn


class AttentionControl(abc.ABC):
    """attention_store.py:12-61 — base state machine."""

    def __init__(self):
        self.LOW_RESOURCE = False  # False: CFG batch, only the cond half is controlled
        self.cur_step = 0
        self.num_att_layers = -1
        self.cur_att_layer = 0

    def step_callback(self, x_t):
        self.cur_att_layer = 0
        self.cur_step += 1
        self.between_steps()
        return x_t

    def between_steps(self):
        return

    @property
    def num_uncond_att_layers(self):
        return 0

    def __call__(self, attn, is_cross: bool, place_in_unet: str):
        raise NotImplementedError(
            "fatezero_b200 controllers are not called with materialised probability tensors: the UNet engine queries "
            "self_attn_args()/cross_attn_args() and the STORE / INJECT work happens inside fz_attention_f16")

    def reset(self):
        self.cur_step = 0
        self.cur_att_layer = 0

    # ---- fused-kernel protocol (called by engine.UNetEngine) ----------------------------------------------------
    def begin_forward(self, batch: int, frames: int):
        self._pos = {k: 0 for k in KEYS}

    def _edit_start(self, nb: int) -> int:
        return 0 if self.LOW_RESOURCE else nb // 2

    def self_attn_args(self, place: str, S: int, T: int, heads: int, nb: int, frames: int) -> Optional[dict]:
        return None

    def cross_attn_args(self, place: str, S: int, heads: int, nb: int, frames: int) -> Optional[dict]:
        return None


class HostStep:
    """One inversion step's maps parked in PINNED host memory (host_spill mode: clips whose map cache exceeds HBM, e.g. 24 frames with
    the default [-1, 'first'] K/V frames = 208 GiB).  The device->host copies run on a side stream behind the step that produced the maps;
    `fetch()` brings the step back (host->device on the side stream, the consumer waits on an event), normally one step ahead of its use.
    The reference does the equivalent with `.cpu()` + deepcopy on the critical path (attention_store.py:81-93) and `.to(device)` per layer
    in the edit pass (attention_util.py:83-84,216-218)."""

    def __init__(self, step_store: Dict[str, List[torch.Tensor]], stream: "torch.cuda.Stream"):
        self.stream = stream
        self.host: Dict[str, List[Tuple[torch.Tensor, int]]] = {}
        self.dev: Optional[Dict[str, List[torch.Tensor]]] = None
        self.ready = None
        cur = torch.cuda.current_stream()
        done = torch.cuda.Event()
        done.record(cur)
        stream.wait_event(done)
        with torch.cuda.stream(stream):
            for k, lst in step_store.items():
                out = []
                for t in lst:
                    raw = t._base if (t._base is not None and not t.is_contiguous()) else t   # cross maps are [..., :77] views of 80-wide slabs
                    h = torch.empty(raw.shape, dtype=raw.dtype, pin_memory=True)
                    h.copy_(raw, non_blocking=True)
                    raw.record_stream(stream)  # the slab may be freed by Python now: the allocator keeps it until the copy has run
                    out.append((h, t.shape[-1]))
                self.host[k] = out
        self.device = cur.device if hasattr(cur, "device") else torch.device("cuda", torch.cuda.current_device())

    def prefetch(self):
        if self.dev is not None:
            return
        with torch.cuda.stream(self.stream):
            dev = {}
            for k, lst in self.host.items():
                dev[k] = []
                for h, width in lst:
                    d = torch.empty(h.shape, dtype=h.dtype, device=self.device)
                    d.copy_(h, non_blocking=True)
                    dev[k].append(d[..., :width] if width != h.shape[-1] else d)
            self.ready = torch.cuda.Event()
            self.ready.record(self.stream)
        self.dev = dev

    def fetch(self) -> Dict[str, List[torch.Tensor]]:
        self.prefetch()
        torch.cuda.current_stream().wait_event(self.ready)
        for lst in self.dev.values():
            for t in lst:
                (t._base if t._base is not None else t).record_stream(torch.cuda.current_stream())
        return self.dev

    def release(self):
        self.dev = None
        self.ready = None


class AttentionStore(AttentionControl):
    """attention_store.py:63-137 — inversion-time STORE into the HBM map cache."""

    def __init__(self, save_self_attention: bool = True, disk_store: bool = False, host_spill: Optional[bool] = None):
        super().__init__()
        self.disk_store = disk_store
        # host_spill (extension; default from $FZ_HOST_SPILL): park every finished step's maps in pinned host memory and free the HBM
        # slabs; the edit pass prefetches them back one step ahead.  For clips whose cache does not fit HBM; forces the eager loops.
        self.host_spill = bool(int(os.environ.get("FZ_HOST_SPILL", "0"))) if host_spill is None else bool(host_spill)
        self._spill_stream = None
        self.store_dir = None
        if disk_store:
            self.store_dir = f"./trash/attention_cache_{time.strftime('%Y%m%d-%H%M%S')}"
            os.makedirs(self.store_dir, exist_ok=True)
        self.step_store = self.get_empty_store()
        self._acc: Dict[str, List[torch.Tensor]] = {}  # fp16 running sums of the cross maps (80-wide slabs)
        self._self_sum_cache = None
        self.save_self_attention = save_self_attention
        self.latents_store: List[torch.Tensor] = []
        self.attention_store_all_step: List[Dict[str, List[torch.Tensor]]] = []
        self.attention_store_paths: List[str] = []
        self._pos = {k: 0 for k in KEYS}
        self._graph_plan_id = None  # set when the maps live in the memory pool of a captured inversion plan (graphs.py)

    @staticmethod
    def get_empty_store():
        return {k: [] for k in KEYS}

    @staticmethod
    def get_empty_cross_store():
        return {"down_cross": [], "mid_cross": [], "up_cross": []}

    # ---- fused protocol -------------------------------------------------------------------------------------------
    def _acc_slab(self, key: str, pos: int, shape, device) -> torch.Tensor:
        lst = self._acc.setdefault(key, [])
        while len(lst) <= pos:
            lst.append(None)
        if lst[pos] is None:
            lst[pos] = torch.zeros(shape, dtype=f16, device=device)
        return lst[pos]

    def _store_self(self, place, S, T, heads, nb) -> Optional[dict]:
        if S > 32 ** 2 or not self.save_self_attention:
            return None
        start = self._edit_start(nb)
        key = _key(place, False)
        slab = torch.empty((nb - start, heads, S, T), dtype=f16, device=torch.cuda.current_device())
        self.step_store[key].append(slab)
        self._pos[key] += 1
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=slab, cache_ld=T)

    def _store_cross(self, place, S, heads, nb) -> Optional[dict]:
        if S > 32 ** 2:
            return None
        start = self._edit_start(nb)
        key = _key(place, True)
        pos = self._pos[key]
        self._pos[key] += 1
        dev = torch.cuda.current_device()
        slab = torch.empty((nb - start, heads, S, CROSS_LD), dtype=f16, device=dev)
        self.step_store[key].append(slab[..., :77])
        acc = self._acc_slab(key, pos, (nb - start, heads, S, CROSS_LD), slab.device)
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=slab, cache_ld=CROSS_LD, acc=acc)

    def self_attn_args(self, place, S, T, heads, nb, frames):
        return self._store_self(place, S, T, heads, nb)

    def cross_attn_args(self, place, S, heads, nb, frames):
        return self._store_cross(place, S, heads, nb)

    # ---- reference surface ------------------------------------------------------------------------------------------
    def step_callback(self, x_t):
        x_t = super().step_callback(x_t)
        self.latents_store.append(x_t.detach().clone())  # stays in HBM (the reference parks it in host RAM)
        return x_t

    def between_steps(self):
        self._self_sum_cache = None
        if self.disk_store:
            # attention_store.py:103-106: the step dict goes to disk and the list holds its PATH; the HBM slabs are released here
            # (the running cross sums stay: they are what `attention_store` / the latent blend read)
            path = self.store_dir + f"/{self.cur_step:03d}.pt"
            torch.save({k: [t.cpu() for t in v] for k, v in self.step_store.items()}, path)
            self.attention_store_paths.append(path)
            self.attention_store_all_step.append(path)
        elif self.host_spill and any(len(v) for v in self.step_store.values()):
            if self._spill_stream is None:
                self._spill_stream = torch.cuda.Stream()
            self.attention_store_all_step.append(HostStep(self.step_store, self._spill_stream))
        else:
            self.attention_store_all_step.append(self.step_store)
        self.step_store = self.get_empty_store()

    @property
    def attention_store(self) -> Dict[str, List[torch.Tensor]]:
        """Running sums over the steps so far (attention_store.py:95-101).  Cross sums are maintained in-kernel in fp16 with
        the reference's summation order; self sums are only needed by visualisation, so they are rebuilt on demand."""
        out = {k: [] for k in KEYS}
        for k, lst in self._acc.items():
            out[k] = [a[..., :77] for a in lst if a is not None]
        if self.attention_store_all_step and self.save_self_attention:
            if self._self_sum_cache is None:
                sums = {}
                for k in ("down_self", "mid_self", "up_self"):
                    per_pos = None
                    for d in self.attention_store_all_step:
                        if isinstance(d, str):
                            d = torch.load(d)
                        elif isinstance(d, HostStep):
                            d = d.fetch()
                        cur = d.get(k, [])
                        per_pos = [t.clone() for t in cur] if per_pos is None else [a + b for a, b in zip(per_pos, cur)]
                    sums[k] = per_pos or []
                self._self_sum_cache = sums
            out.update(self._self_sum_cache)
        if all(len(v) == 0 for v in out.values()):
            return {}
        return out

    def get_average_attention(self):
        store = self.attention_store
        return {key: [item / self.cur_step for item in store[key]] for key in store}

    # ---- CUDA-graph replay support (graphs.py): the launch sequence of a loop depends on the controller only through this signature;
    # after a replay the captured controller's end-of-loop state (same slabs, refilled) is adopted by the caller's controller object ----
    _ADOPT = ("cur_step", "cur_att_layer", "step_store", "_acc", "_self_sum_cache", "latents_store", "attention_store_all_step",
              "attention_store_paths", "_pos")

    def graph_signature(self):
        if type(self) is not AttentionStore or self.disk_store or self.host_spill:
            return None
        return ("store", bool(self.save_self_attention), bool(self.LOW_RESOURCE))

    def is_pristine(self) -> bool:
        return self.cur_step == 0 and not self.attention_store_all_step and not self.latents_store and not self._acc

    def adopt_from(self, tmpl: "AttentionStore"):
        if tmpl is self:
            return
        for k in self._ADOPT:
            v = getattr(tmpl, k)
            if isinstance(v, list):
                v = list(v)
            elif isinstance(v, dict):
                v = {kk: (list(vv) if isinstance(vv, list) else vv) for kk, vv in v.items()}
            setattr(self, k, v)
        self._self_sum_cache = None  # the replay refilled the slabs: a sum the template computed before it is stale
        self._graph_plan_id = getattr(tmpl, "_graph_plan_id", None)

    def reset(self):
        super().reset()
        self.step_store = self.get_empty_store()
        self.attention_store_all_step = []
        self.attention_store_paths = []
        self.latents_store = []
        self._acc = {}
        self._self_sum_cache = None


class AttentionControlEdit(AttentionStore, abc.ABC):
    """attention_util.py:39-209 — edit-time INJECT / BLEND against the stored inversion maps."""

    def __init__(self, prompts, num_steps: int, cross_replace_steps: Union[float, Tuple[float, float], Dict[str, Tuple[float, float]]],
                 self_replace_steps: Union[float, Tuple[float, float]], latent_blend: Optional[SpatialBlender], tokenizer=None,
                 additional_attention_store: AttentionStore = None, use_inversion_attention: bool = False,
                 attention_blend: SpatialBlender = None, save_self_attention: bool = True, disk_store=False):
        super().__init__(save_self_attention=save_self_attention, disk_store=disk_store)
        self.additional_attention_store = additional_attention_store
        self.batch_size = len(prompts)
        self.attention_blend = attention_blend
        if self.additional_attention_store is not None:
            self.batch_size = len(prompts) // 2
            assert self.batch_size == 1, "Only support single video editing with additional attention_store"
        else:
            raise NotImplementedError("editing without an external inversion store (batch of prompts in one UNet call) is the "
                                      "prompt-to-prompt image mode; FateZero edits against additional_attention_store")
        self.num_steps = num_steps
        self.cross_replace_alpha = tables.get_time_words_attention_alpha(prompts, num_steps, cross_replace_steps, tokenizer)
        if type(self_replace_steps) is float:
            self_replace_steps = 0, self_replace_steps
        self.num_self_replace = int(num_steps * self_replace_steps[0]), int(num_steps * self_replace_steps[1])
        self.latent_blend = latent_blend
        self.prev_attention_key_name = 0
        self.use_inversion_attention = use_inversion_attention
        self.attention_position_counter_dict = {k: 0 for k in KEYS}
        self._xedit = None
        self._graph_plan_id = None
        self._mask_cache: Dict[Tuple[int, int], torch.Tensor] = {}
        if save_self_attention:
            warnings.warn("AttentionControlEdit(save_self_attention=True): pre-edit self-attention maps of the edit pass are not "
                          "kept by the fused path (only the reference's visualisation helpers read them)")
        self.save_self_attention = False

    # ---- tables for FZ_ATTN_CROSSEDIT -------------------------------------------------------------------------------
    def _cross_tables(self) -> Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]:
        """(mode, mapper[77], alphas[77], M[77,77], equalizer[77])"""
        raise NotImplementedError

    def _build_xedit(self, device) -> torch.Tensor:
        mode, mapper, a, M, eq = self._cross_tables()
        n_t = self.num_steps + 1
        tab = torch.zeros(n_t, _lib.XEDIT_FLOATS)
        tab[:, 0] = mode
        tab[:, 8:8 + 77] = self.cross_replace_alpha[:, 0, 0, 0, :]
        tab[:, 88:88 + 80] = 1.0
        if eq is not None:
            tab[:, 88:88 + 77] = eq.reshape(-1)[:77]
        if a is not None:
            tab[:, 168:168 + 77] = a.reshape(-1)[:77]
        if mapper is not None:
            tab[:, 248:248 + 77] = mapper.reshape(-1)[:77].float()
        if M is not None:
            mm = torch.zeros(80, 80)
            mm[:77, :77] = M.reshape(77, 77)
            tab[:, 328:] = mm.reshape(-1)
        return tab.to(device).contiguous()

    def prepare_tables(self, device):
        """Build the device-side edit tables now (a graph capture must not contain the pageable host-to-device copy)."""
        if self._xedit is None:
            self._xedit = self._build_xedit(device)

    def load_tables_from(self, other: "AttentionControlEdit"):
        """Refresh this (captured) controller's device tables with the content of `other` (same structure, new prompts)."""
        self.prepare_tables(other._xedit.device if other._xedit is not None else self._xedit.device)
        if other is not self:
            self._xedit.copy_(other._build_xedit("cpu"), non_blocking=False)

    _ADOPT_EDIT = AttentionStore._ADOPT + ("attention_position_counter_dict", "_mask_cache", "_xedit")

    def graph_signature(self):
        """Everything that shapes the launch sequence of the edit loop (table CONTENT is refreshed per replay, see load_tables_from)."""
        if self.disk_store or self.additional_attention_store is None or getattr(self.additional_attention_store, "host_spill", False):
            return None

        def blender(b):
            if b is None:
                return None
            return (b.prompt_choose, tuple(float(t) for t in b.th), b.start_blend, b.end_blend,
                    tuple(b.alpha_layers.reshape(-1).tolist()))
        return ("edit", self.num_steps, tuple(self.num_self_replace), bool(self.use_inversion_attention), bool(self.LOW_RESOURCE),
                blender(self.latent_blend), blender(self.attention_blend),
                getattr(self.additional_attention_store, "_graph_plan_id", None))

    def adopt_from(self, tmpl: "AttentionControlEdit"):
        if tmpl is self:
            return
        for k in self._ADOPT_EDIT:
            v = getattr(tmpl, k)
            if isinstance(v, list):
                v = list(v)
            elif isinstance(v, dict):
                v = {kk: (list(vv) if isinstance(vv, list) else vv) for kk, vv in v.items()}
            setattr(self, k, v)
        for name in ("latent_blend", "attention_blend"):
            mine, theirs = getattr(self, name), getattr(tmpl, name)
            if mine is not None and theirs is not None:
                mine.counter = theirs.counter
                mine.mask_list = list(theirs.mask_list)

    def _step_in_store(self) -> int:
        if self.use_inversion_attention:
            return len(self.additional_attention_store.attention_store_all_step) - self.cur_step - 1
        return self.cur_step

    def _source_maps(self, step_in_store: int) -> Dict[str, List[torch.Tensor]]:
        steps = self.additional_attention_store.attention_store_all_step
        d = steps[step_in_store]
        if isinstance(d, str):
            d = torch.load(d)
        elif isinstance(d, HostStep):
            # host-spilled inversion maps: this step was prefetched while the previous one was in use; start the next transfer now and
            # drop the steps that are behind us (at most two steps' maps are resident)
            nxt = step_in_store - 1 if self.use_inversion_attention else step_in_store + 1
            if 0 <= nxt < len(steps) and isinstance(steps[nxt], HostStep):
                steps[nxt].prefetch()
            for j, other in enumerate(steps):
                if isinstance(other, HostStep) and j not in (step_in_store, nxt) and other.dev is not None:
                    other.release()
            d = d.fetch()
        return d

    # ---- fused protocol -------------------------------------------------------------------------------------------------
    def begin_forward(self, batch, frames):
        super().begin_forward(batch, frames)
        if self.LOW_RESOURCE or batch != 2:
            raise RuntimeError("the edit controller expects a classifier-free-guidance batch (uncond, cond); LOW_RESOURCE is the "
                               "inversion mode (attention_store.py:40-46)")

    def self_attn_args(self, place, S, T, heads, nb, frames):
        if S > 32 ** 2:
            return None
        key = _key(place, False)
        pos = self.attention_position_counter_dict[key]
        self.attention_position_counter_dict[key] += 1
        lo, hi = self.num_self_replace
        if not (lo <= self.cur_step < hi):
            return None
        step_in_store = self._step_in_store()
        base = self._source_maps(step_in_store)[key][pos]
        if base.device.type != "cuda":
            base = base.to(torch.cuda.current_device(), f16)
        start = self._edit_start(nb)
        if self.attention_blend is not None:
            r = int(round(S ** 0.5))
            ck = (step_in_store, r)
            if ck not in self._mask_cache:
                # prompt_choose == 'source': only the stored source maps enter, so the mask is shared by all layers of a step at
                # one resolution (the reference recomputes it per layer: SURVEY.md K18)
                self._mask_cache = {k: v for k, v in self._mask_cache.items() if k[0] == step_in_store}
                m = self.attention_blend.mask_from(self._source_maps(step_in_store), 0, r, r)
                self._mask_cache[ck] = m.reshape(m.shape[0], S).contiguous()
            self.attention_blend.counter += 1
            return dict(edit_bf_start=start, row_mode=_lib.ATTN_BLEND, base=base, cache_ld=T, mask=self._mask_cache[ck])
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_REPLACE, base=base, cache_ld=T)

    def cross_attn_args(self, place, S, heads, nb, frames):
        if S > 32 ** 2:
            return None
        key = _key(place, True)
        pos = self.attention_position_counter_dict[key]
        self.attention_position_counter_dict[key] += 1
        base = self._source_maps(self._step_in_store())[key][pos]
        if base.stride(2) != CROSS_LD or base.device.type != "cuda":
            slab = torch.zeros((*base.shape[:3], CROSS_LD), dtype=f16, device=torch.cuda.current_device())
            slab[..., :77] = base
            base = slab
        start = self._edit_start(nb)
        if self._xedit is None:
            self._xedit = self._build_xedit(base.device)
        # pre-edit target maps accumulate in this controller's attention_store (attention_util.py:103; App. B quirk 4)
        acc = self._acc_slab(key, pos, (nb - start, heads, S, CROSS_LD), base.device)
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_CROSSEDIT, base=base, cache_ld=CROSS_LD, acc=acc,
                    xedit=self._xedit[self.cur_step])

    # ---- reference surface --------------------------------------------------------------------------------------------
    def latent_blend_args(self, h: int, w: int) -> Optional[dict]:
        """Arguments that fuse the latent blend (attention_util.py:47-78, spatial_blend.py:116-122) into fz_cfg_ddim_step.
        Must be called AFTER the UNet forward of the step and BEFORE step_callback (cur_step not yet incremented)."""
        if self.latent_blend is None:
            return None
        inv = self.additional_attention_store
        cur_next = self.cur_step + 1
        step_in_store = (len(inv.latents_store) - cur_next) if self.use_inversion_attention else cur_next
        x_inv = inv.latents_store[step_in_store]
        lb = self.latent_blend
        src = self._source_maps(step_in_store)
        tgt = self.attention_store  # running sums including this step's pre-edit maps (updated in-kernel)
        m_src = lb.mask_from(src, 0, h, w)
        m_tgt = lb.mask_from(tgt, 1, h, w)
        lb.mask_list.append(m_src[:, None, :, :].float())
        lb.counter += 1
        apply = lb.start_blend < lb.counter < lb.end_blend
        return dict(x_inv=x_inv.to(torch.float32), mask_a=m_src, mask_b=m_tgt, apply_blend=apply)

    def step_callback(self, x_t, blend_fused: bool = False):
        x_t = AttentionStore.step_callback(self, x_t)
        if self.latent_blend is None or blend_fused:
            return x_t
        raise NotImplementedError("the latent blend is fused into fz_cfg_ddim_step: call latent_blend_args() before the DDIM step "
                                  "and step_callback(x_t, blend_fused=True) after it (see pipeline.sd_ddim_pipeline)")

    def between_steps(self):
        super().between_steps()
        self.attention_position_counter_dict = {k: 0 for k in KEYS}

    def replace_self_attention(self, attn_base, att_replace, reshaped_mask=None):
        raise NotImplementedError("fused into fz_attention_f16 (FZ_ATTN_REPLACE / FZ_ATTN_BLEND)")

    def replace_cross_attention(self, attn_base, att_replace):
        raise NotImplementedError("fused into fz_attention_f16 (FZ_ATTN_CROSSEDIT)")


class AttentionReplace(AttentionControlEdit):
    """attention_util.py:211-239: word-swap edits, cross maps projected through the 77x77 replacement matrix."""

    def __init__(self, prompts, num_steps: int, cross_replace_steps, self_replace_steps, latent_blend=None, tokenizer=None,
                 additional_attention_store=None, use_inversion_attention=False, attention_blend=None, save_self_attention: bool = True,
                 disk_store=False):
        super().__init__(prompts, num_steps, cross_replace_steps, self_replace_steps, latent_blend, tokenizer=tokenizer,
                         additional_attention_store=additional_attention_store, use_inversion_attention=use_inversion_attention,
                         attention_blend=attention_blend, save_self_attention=save_self_attention, disk_store=disk_store)
        self.mapper = tables.get_replacement_mapper(prompts, tokenizer)

    def _cross_tables(self):
        return 1, None, None, self.mapper[0], None


class AttentionRefine(AttentionControlEdit):
    """attention_util.py:241-273: prompt refinement, cross maps gathered through the token alignment."""

    def __init__(self, prompts, num_steps: int, cross_replace_steps, self_replace_steps, latent_blend=None, tokenizer=None,
                 additional_attention_store=None, use_inversion_attention=False, attention_blend=None, save_self_attention: bool = True,
                 disk_store=False):
        super().__init__(prompts, num_steps, cross_replace_steps, self_replace_steps, latent_blend, tokenizer=tokenizer,
                         additional_attention_store=additional_attention_store, use_inversion_attention=use_inversion_attention,
                         attention_blend=attention_blend, save_self_attention=save_self_attention, disk_store=disk_store)
        self.mapper, alphas = tables.get_refinement_mapper(prompts, tokenizer)
        self.alphas = alphas.reshape(alphas.shape[0], 1, 1, alphas.shape[1])

    def _cross_tables(self):
        return 0, self.mapper[0], self.alphas.reshape(-1, 77)[0], None, None


class AttentionReweight(AttentionControlEdit):
    """attention_util.py:275-305: multiplies the (replaced / refined) cross maps by the equalizer."""

    def __init__(self, prompts, num_steps: int, cross_replace_steps, self_replace_steps, equalizer, latent_blend=None,
                 controller: Optional[AttentionControlEdit] = None, tokenizer=None, additional_attention_store=None,
                 use_inversion_attention=False, attention_blend=None, save_self_attention: bool = True, disk_store=False):
        super().__init__(prompts, num_steps, cross_replace_steps, self_replace_steps, latent_blend, tokenizer=tokenizer,
                         additional_attention_store=additional_attention_store, use_inversion_attention=use_inversion_attention,
                         attention_blend=attention_blend, save_self_attention=save_self_attention, disk_store=disk_store)
        self.equalizer = equalizer
        self.prev_controller = controller

    def _cross_tables(self):
        if self.prev_controller is not None:
            mode, mapper, a, M, _ = self.prev_controller._cross_tables()
        else:
            # no previous controller: R = base * eq  == Replace with the identity matrix
            mode, mapper, a, M = 1, None, None, torch.eye(77)
        return mode, mapper, a, M, self.equalizer.reshape(-1)


class AttentionControlEditBatch:
    """K edit controllers of ONE inverted clip driven through one batched edit pass (CFG batch [uncond_1..K ; cond_1..K]).

    Every child is asked exactly what it would be asked in its own single-prompt pass (a CFG batch of 2 at `frames` frames), so its
    position counters, tables, masks and running sums evolve as in that pass; the answers are merged into one grouped attention launch
    (fz_attention_grouped_f16: child k owns rows [(K + k) F, (K + k + 1) F)), and a child that answers None becomes a NONE group.  The
    children must edit against the same inversion store with the same step count and store indexing."""

    def __init__(self, edits: List[AttentionControlEdit]):
        edits = list(edits)
        if not edits or len(edits) > _lib.MAX_ATTN_GROUPS:
            raise ValueError(f"AttentionControlEditBatch: 1..{_lib.MAX_ATTN_GROUPS} edit controllers, got {len(edits)}")
        c0 = edits[0]
        for e in edits[1:]:
            if e.additional_attention_store is not c0.additional_attention_store:
                raise ValueError("AttentionControlEditBatch: every edit must read the same additional_attention_store")
            if e.num_steps != c0.num_steps or bool(e.use_inversion_attention) != bool(c0.use_inversion_attention):
                raise ValueError("AttentionControlEditBatch: every edit must share num_steps and use_inversion_attention")
        store = c0.additional_attention_store
        if any(getattr(e, "disk_store", False) for e in edits) or getattr(store, "disk_store", False) or getattr(store, "host_spill", False):
            raise NotImplementedError("AttentionControlEditBatch: disk_store / host_spill stores are edited one prompt at a time")
        self.edits = edits
        self.prompt_groups = len(edits)
        self.LOW_RESOURCE = False
        self.num_att_layers = -1
        self._frames = None

    # ---- state shared with the children --------------------------------------------------------------------------------
    @property
    def cur_step(self) -> int:
        return self.edits[0].cur_step

    @property
    def additional_attention_store(self):
        return self.edits[0].additional_attention_store

    def __setattr__(self, name, value):
        object.__setattr__(self, name, value)
        if name == "num_att_layers":  # register_attention_control sets it on whatever object it is given: pass it on
            for e in self.__dict__.get("edits", []):
                e.num_att_layers = value

    # ---- fused-kernel protocol ------------------------------------------------------------------------------------------
    def begin_forward(self, batch, frames):
        if batch != 2 * self.prompt_groups:
            raise RuntimeError(f"AttentionControlEditBatch: expected a CFG batch of 2 x {self.prompt_groups} prompts, got {batch}")
        self._frames = frames
        for e in self.edits:
            e.begin_forward(2, frames)

    def _merge(self, answers: List[Optional[dict]], frames: int) -> Optional[dict]:
        if self.prompt_groups == 1:
            return answers[0]
        live = [a for a in answers if a is not None]
        if not live:
            return None
        base, cache_ld = live[0]["base"], live[0]["cache_ld"]
        for a in live[1:]:
            if a["base"].data_ptr() != base.data_ptr() or a["cache_ld"] != cache_ld or a["base"].shape != base.shape:
                raise RuntimeError("AttentionControlEditBatch: the edits disagree on the cached inversion map of this layer")
        for a in live:
            if a["edit_bf_start"] != frames:
                raise RuntimeError("AttentionControlEditBatch: an edit asked for rows outside its conditional half")
        groups = [dict(row_mode=_lib.ATTN_NONE) if a is None else
                  dict(row_mode=a["row_mode"], mask=a.get("mask"), acc=a.get("acc"), xedit=a.get("xedit")) for a in answers]
        return dict(edit_bf_start=self.prompt_groups * frames, base=base, cache_ld=cache_ld, groups=groups)

    def self_attn_args(self, place, S, T, heads, nb, frames):
        return self._merge([e.self_attn_args(place, S, T, heads, 2 * frames, frames) for e in self.edits], frames)

    def cross_attn_args(self, place, S, heads, nb, frames):
        return self._merge([e.cross_attn_args(place, S, heads, 2 * frames, frames) for e in self.edits], frames)

    def latent_blend_args(self, h: int, w: int) -> List[Optional[dict]]:
        return [e.latent_blend_args(h, w) for e in self.edits]

    def step_callback(self, x_t, blend_fused: bool = False):
        for k, e in enumerate(self.edits):
            e.step_callback(x_t[k:k + 1], blend_fused=blend_fused)
        return x_t

    def reset(self):
        for e in self.edits:
            e.reset()

    # ---- CUDA-graph replay support: composed from the children's --------------------------------------------------------------
    def graph_signature(self):
        sigs = [e.graph_signature() for e in self.edits]
        if any(s is None for s in sigs):
            return None
        # the last element is the inversion store's plan id (shared by the children), as for a single edit
        return ("edit_batch", tuple(s[:-1] for s in sigs), sigs[0][-1])

    def prepare_tables(self, device):
        for e in self.edits:
            e.prepare_tables(device)

    def load_tables_from(self, other: "AttentionControlEditBatch"):
        for mine, theirs in zip(self.edits, other.edits):
            mine.load_tables_from(theirs)

    def adopt_from(self, tmpl: "AttentionControlEditBatch"):
        if tmpl is self:
            return
        for mine, theirs in zip(self.edits, tmpl.edits):
            mine.adopt_from(theirs)


class AttentionStoreBatch:
    """K inversion stores, one per source clip, filled by ONE batched inversion (UNet batch [clip_1..K], F frames each).

    Every store is asked exactly what it is asked in its own batch-1 inversion (a LOW_RESOURCE batch of 1 at `frames` frames), so its slabs,
    running sums, latents and step counter end up as `prepare_latents_ddim_inverted` leaves `pipe.store_controller`; the answers are merged
    into one grouped launch (fz_attention_grouped_slabs_f16: clip k owns rows [k F, (k + 1) F) and writes its own slabs).
    store_maps=False: no maps are stored (prepare_latents_ddim_inverted with store_attention=False); the stores still record the latents,
    and the batch still makes the UNet plan its GroupNorm statistics per clip."""

    def __init__(self, stores: List[AttentionStore], store_maps: bool = True):
        stores = list(stores)
        if not stores or len(stores) > _lib.MAX_ATTN_GROUPS:
            raise ValueError(f"AttentionStoreBatch: 1..{_lib.MAX_ATTN_GROUPS} stores, got {len(stores)}")
        if any(not isinstance(s, AttentionStore) or isinstance(s, AttentionControlEdit) for s in stores):
            raise TypeError("AttentionStoreBatch: every clip needs its own AttentionStore")
        if len({id(s) for s in stores}) != len(stores):
            raise ValueError("AttentionStoreBatch: a store appears twice (one store per clip)")
        if any(s.disk_store or s.host_spill for s in stores):
            raise NotImplementedError("AttentionStoreBatch: disk_store / host_spill stores are inverted one clip at a time")
        if len({bool(s.save_self_attention) for s in stores}) != 1:
            raise ValueError("AttentionStoreBatch: the stores disagree on save_self_attention")
        self.stores = stores
        self.store_maps = bool(store_maps)
        self.prompt_groups = len(stores)
        self.num_att_layers = -1

    def __setattr__(self, name, value):
        object.__setattr__(self, name, value)
        if name == "num_att_layers":
            for s in self.__dict__.get("stores", []):
                s.num_att_layers = value

    @property
    def cur_step(self) -> int:
        return self.stores[0].cur_step

    # ---- fused-kernel protocol ------------------------------------------------------------------------------------------
    def begin_forward(self, batch, frames):
        if batch != self.prompt_groups:
            raise RuntimeError(f"AttentionStoreBatch: expected a batch of {self.prompt_groups} clips, got {batch}")
        for s in self.stores:
            s.begin_forward(1, frames)

    def _merge(self, answers: List[Optional[dict]]) -> Optional[dict]:
        if self.prompt_groups == 1:
            return answers[0]
        if all(a is None for a in answers):
            return None
        if any(a is None or a["edit_bf_start"] != 0 for a in answers):
            raise RuntimeError("AttentionStoreBatch: every clip must store all of its rows (LOW_RESOURCE inversion)")
        return dict(edit_bf_start=0, cache_ld=answers[0]["cache_ld"],
                    groups=[dict(row_mode=_lib.ATTN_STORE, store=a["store"], acc=a.get("acc")) for a in answers])

    def self_attn_args(self, place, S, T, heads, nb, frames):
        if not self.store_maps:
            return None
        return self._merge([s.self_attn_args(place, S, T, heads, frames, frames) for s in self.stores])

    def cross_attn_args(self, place, S, heads, nb, frames):
        if not self.store_maps:
            return None
        return self._merge([s.cross_attn_args(place, S, heads, frames, frames) for s in self.stores])

    def step_callback(self, x_t):
        for k, s in enumerate(self.stores):
            s.step_callback(x_t[k:k + 1])
        return x_t

    def reset(self):
        for s in self.stores:
            s.reset()

    # ---- CUDA-graph replay support (graphs.py), composed from the stores' --------------------------------------------------
    def graph_signature(self):
        sigs = [s.graph_signature() for s in self.stores]
        if any(s is None for s in sigs):
            return None
        return ("store_batch", len(sigs), self.store_maps, sigs[0])

    def is_pristine(self) -> bool:
        return all(s.is_pristine() for s in self.stores)

    @property
    def _graph_plan_id(self):
        return tuple(s._graph_plan_id for s in self.stores)

    @_graph_plan_id.setter
    def _graph_plan_id(self, plan_id):
        # clip k's maps are its own slabs of the plan: (plan, k) tells them apart in the key of a captured edit that reads them
        for k, s in enumerate(self.stores):
            s._graph_plan_id = (plan_id, k)

    def adopt_from(self, tmpl: "AttentionStoreBatch"):
        if tmpl is self:
            return
        for mine, theirs in zip(self.stores, tmpl.stores):
            mine.adopt_from(theirs)


class AttentionControlEditClips(AttentionControlEditBatch):
    """K edit controllers of possibly DIFFERENT inverted clips driven through one batched edit pass (CFG batch [uncond_1..K ; cond_1..K]).

    As AttentionControlEditBatch, each child is asked what its own single-prompt pass asks, but every group reads the cached maps of its
    own child's additional_attention_store (fz_attention_grouped_slabs_f16), and the latent blend of each child uses its own store's
    inverted latents (fz_cfg_ddim_step_multi).  Several children may edit the same clip."""

    def __init__(self, edits: List[AttentionControlEdit]):
        edits = list(edits)
        if not edits or len(edits) > _lib.MAX_ATTN_GROUPS:
            raise ValueError(f"AttentionControlEditClips: 1..{_lib.MAX_ATTN_GROUPS} edit controllers, got {len(edits)}")
        c0 = edits[0]
        for e in edits[1:]:
            if e.num_steps != c0.num_steps or bool(e.use_inversion_attention) != bool(c0.use_inversion_attention):
                raise ValueError("AttentionControlEditClips: every edit must share num_steps and use_inversion_attention")
        for e in edits:
            st = e.additional_attention_store
            if getattr(e, "disk_store", False) or getattr(st, "disk_store", False) or getattr(st, "host_spill", False):
                raise NotImplementedError("AttentionControlEditClips: disk_store / host_spill stores are edited one clip at a time")
        self.edits = edits
        self.prompt_groups = len(edits)
        self.LOW_RESOURCE = False
        self.num_att_layers = -1
        self._frames = None

    @property
    def additional_attention_store(self):
        raise AttributeError("AttentionControlEditClips: every edit has its own additional_attention_store (see .edits)")

    def _merge(self, answers: List[Optional[dict]], frames: int) -> Optional[dict]:
        if self.prompt_groups == 1:
            return answers[0]
        live = [a for a in answers if a is not None]
        if not live:
            return None
        cache_ld = live[0]["cache_ld"]
        for a in live:
            if a["cache_ld"] != cache_ld or a["base"].shape != live[0]["base"].shape:
                raise RuntimeError("AttentionControlEditClips: the clips' cached inversion maps of this layer differ in geometry")
            if a["edit_bf_start"] != frames:
                raise RuntimeError("AttentionControlEditClips: an edit asked for rows outside its conditional half")
        groups = [dict(row_mode=_lib.ATTN_NONE) if a is None else
                  dict(row_mode=a["row_mode"], mask=a.get("mask"), acc=a.get("acc"), xedit=a.get("xedit"), base=a["base"]) for a in answers]
        return dict(edit_bf_start=self.prompt_groups * frames, cache_ld=cache_ld, groups=groups)

    def graph_signature(self):
        sigs = [e.graph_signature() for e in self.edits]
        if any(s is None for s in sigs):
            return None
        # which store each child reads is part of the launch sequence (the base slabs are baked into the captured kernels); the last
        # element lists the stores' plan ids, None when one of them does not live in a captured inversion plan
        plans = tuple(s[-1] for s in sigs)
        stores = [id(e.additional_attention_store) for e in self.edits]
        layout = tuple(stores.index(s) for s in stores)
        return ("edit_clips", tuple(s[:-1] for s in sigs), layout, None if any(p is None for p in plans) else plans)


def map_cache_bytes(unet_config: dict, model_config: dict, h: int, w: int, save_self_attention: bool = True) -> Tuple[int, int]:
    """HBM of one clip frame's inversion map cache at latent size h x w: (bytes per DDIM step, bytes held once: the cross running sums).
    Restates the slab shapes AttentionStore allocates for the UNet's transformer layers (self maps [heads, S, n_slots S], cross maps
    [heads, S, 80] and their sums, for S <= 32^2) so that a batch can be admitted before any of it is allocated."""
    from .unet import level_heads
    ch = list(unet_config["block_out_channels"])
    lh = level_heads(unet_config)  # SD-2.x stores 5 / 10 / 20 heads at the 64 / 32 / 16-pixel levels of a 512^2 clip, SD-1.x 8 everywhere
    lpb = int(unet_config["layers_per_block"])
    nblk = len(ch)
    layers = []  # (channels, heads, S)
    for i, t in enumerate(unet_config["down_block_types"]):
        if t.startswith("CrossAttn"):
            layers += [(ch[i], lh[i], (h >> i) * (w >> i))] * lpb
    layers.append((ch[-1], lh[-1], (h >> (nblk - 1)) * (w >> (nblk - 1))))
    for i, t in enumerate(unet_config["up_block_types"]):
        if t.startswith("CrossAttn"):
            s = nblk - 1 - i
            layers += [(ch[s], lh[s], (h >> s) * (w >> s))] * (lpb + 1)
    index_list = list(model_config.get("SparseCausalAttention_index", [-1, "first"]))
    per_step = once = 0
    for c, heads, S in layers:
        if S > 32 ** 2:
            continue
        slots = len(index_list) if index_list and not ("least_sc_channel" in model_config and c < model_config["least_sc_channel"]) else 1
        if save_self_attention:
            per_step += heads * S * slots * S * 2
        per_step += heads * S * CROSS_LD * 2
        once += heads * S * CROSS_LD * 2
    return per_step, once


def get_equalizer(text: str, word_select, values, tokenizer=None):
    return tables.get_equalizer(text, word_select, values, tokenizer)


def make_controller(tokenizer, prompts: List[str], is_replace_controller: bool, cross_replace_steps: Dict[str, float],
                    self_replace_steps: float = 0.0, blend_words=None, equilizer_params=None, additional_attention_store=None,
                    use_inversion_attention=False, blend_th=(0.3, 0.3), NUM_DDIM_STEPS=None, blend_latents=False,
                    blend_self_attention=False, save_path=None, save_self_attention=True, disk_store=False) -> AttentionControlEdit:
    """attention_util.py:320-387 (same argument names, including the reference's `equilizer_params` spelling)."""
    if (blend_words is None) or (blend_words == "None"):
        latent_blend = None
        attention_blend = None
    else:
        if save_path is None:
            raise TypeError("blend_words requires save_path (attention_util.py:339,348 concatenate it)")
        latent_blend = None
        if blend_latents:
            latent_blend = SpatialBlender(prompts, blend_words, start_blend=0.2, end_blend=0.8, tokenizer=tokenizer, th=blend_th,
                                          NUM_DDIM_STEPS=NUM_DDIM_STEPS, save_path=save_path + "/latent_blend_mask", prompt_choose="both")
        attention_blend = None
        if blend_self_attention:
            attention_blend = SpatialBlender(prompts, blend_words, start_blend=0.0, end_blend=2, tokenizer=tokenizer, th=blend_th,
                                             NUM_DDIM_STEPS=NUM_DDIM_STEPS, save_path=save_path + "/attention_blend_mask",
                                             prompt_choose="source")
    common = dict(cross_replace_steps=cross_replace_steps, self_replace_steps=self_replace_steps, latent_blend=latent_blend,
                  tokenizer=tokenizer, additional_attention_store=additional_attention_store,
                  use_inversion_attention=use_inversion_attention, attention_blend=attention_blend,
                  save_self_attention=save_self_attention, disk_store=disk_store)
    cls = AttentionReplace if is_replace_controller else AttentionRefine
    controller = cls(prompts, NUM_DDIM_STEPS, **common)
    if equilizer_params is not None:
        eq = get_equalizer(prompts[1], equilizer_params["words"], equilizer_params["values"], tokenizer=tokenizer)
        controller = AttentionReweight(prompts, NUM_DDIM_STEPS, equalizer=eq, controller=controller, **common)
    return controller


def register_attention_control(model, controller):
    """attention_register.py:14-258: connect a pipeline (anything with `.unet`) with a controller.  Nothing is monkeypatched:
    the UNet keeps a reference and its engine asks the controller for kernel arguments layer by layer."""
    unet = model.unet
    if not hasattr(unet, "set_controller"):
        raise TypeError("register_attention_control needs a fatezero_b200 UNetPseudo3DConditionModel")
    unet.set_controller(controller)
    n = 2 * sum(1 for k in unet.state_dict() if k.endswith("attn1.to_q.weight"))
    if controller is not None:
        try:
            controller.num_att_layers = n  # attention_register.py:257 sets it on whatever object it is given
        except AttributeError:
            pass
    return n
