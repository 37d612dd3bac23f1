"""CPU checks of the batched multi-prompt edit: the argument merging of controllers.AttentionControlEditBatch (with stub children),
the input refusals of P2pDDIMSpatioTemporalPipeline.p2preplace_edit_batch (all raised before any GPU work) and the new C-ABI symbols."""
import types

import pytest
import torch

from fatezero_b200 import _lib, controllers


class StubEdit:
    """Answers like an AttentionControlEdit: fixed per-layer answers, records what it was asked."""

    def __init__(self, store, self_answer, cross_answer, num_steps=5, use_inversion_attention=True, blend=None):
        self.additional_attention_store = store
        self.num_steps = num_steps
        self.use_inversion_attention = use_inversion_attention
        self.disk_store = False
        self.cur_step = 0
        self.self_answer, self.cross_answer, self.blend = self_answer, cross_answer, blend
        self.asked = []
        self.stepped = []

    def begin_forward(self, batch, frames):
        self.asked.append(("begin", batch, frames))

    def self_attn_args(self, place, S, T, heads, nb, frames):
        self.asked.append(("self", place, S, T, heads, nb, frames))
        return self.self_answer

    def cross_attn_args(self, place, S, heads, nb, frames):
        self.asked.append(("cross", place, S, heads, nb, frames))
        return self.cross_answer

    def latent_blend_args(self, h, w):
        return self.blend

    def step_callback(self, x, blend_fused=False):
        self.stepped.append(x)
        self.cur_step += 1
        return x

    def graph_signature(self):
        return ("edit", self.num_steps, "plan-7")


def _store():
    return types.SimpleNamespace(disk_store=False, host_spill=False)


def test_merge_self_and_cross_args():
    store, F = _store(), 3
    base = torch.zeros(F, 2, 16, 32, dtype=torch.float16)
    m1, m3 = torch.ones(F, 16), torch.zeros(F, 16)
    a_rep = dict(edit_bf_start=F, row_mode=_lib.ATTN_REPLACE, base=base, cache_ld=32)
    a_bl1 = dict(edit_bf_start=F, row_mode=_lib.ATTN_BLEND, base=base, cache_ld=32, mask=m1)
    a_bl3 = dict(edit_bf_start=F, row_mode=_lib.ATTN_BLEND, base=base, cache_ld=32, mask=m3)
    xb = torch.zeros(F, 2, 16, 80, dtype=torch.float16)
    acc = [torch.zeros(F, 2, 16, 80, dtype=torch.float16) for _ in range(4)]
    xe = [torch.full((8,), float(k)) for k in range(4)]
    cross = [dict(edit_bf_start=F, row_mode=_lib.ATTN_CROSSEDIT, base=xb, cache_ld=80, acc=acc[k], xedit=xe[k]) for k in range(4)]
    kids = [StubEdit(store, a_rep, cross[0]), StubEdit(store, None, cross[1]), StubEdit(store, a_bl1, cross[2]), StubEdit(store, a_bl3, cross[3])]
    b = controllers.AttentionControlEditBatch(kids)
    assert b.prompt_groups == 4 and b.cur_step == 0
    b.begin_forward(8, F)
    got = b.self_attn_args("down", 16, 32, 2, 8 * F, F)
    assert got["edit_bf_start"] == 4 * F and got["base"] is base and got["cache_ld"] == 32
    modes = [g["row_mode"] for g in got["groups"]]
    assert modes == [_lib.ATTN_REPLACE, _lib.ATTN_NONE, _lib.ATTN_BLEND, _lib.ATTN_BLEND]
    assert got["groups"][2]["mask"] is m1 and got["groups"][3]["mask"] is m3 and got["groups"][0].get("mask") is None
    x = b.cross_attn_args("up", 16, 2, 8 * F, F)
    assert [g["acc"] for g in x["groups"]] == acc and [g["xedit"] for g in x["groups"]] == xe
    # every child is asked exactly what its own single-prompt pass asks: a CFG batch of 2 at F frames
    for k in kids:
        assert k.asked == [("begin", 2, F), ("self", "down", 16, 32, 2, 2 * F, F), ("cross", "up", 16, 2, 2 * F, F)]
    # all children un-hooked -> a plain launch
    quiet = controllers.AttentionControlEditBatch([StubEdit(store, None, None), StubEdit(store, None, None)])
    quiet.begin_forward(4, F)
    assert quiet.self_attn_args("mid", 16, 32, 2, 4 * F, F) is None
    # one child -> its own answer, unchanged
    one = controllers.AttentionControlEditBatch([StubEdit(store, a_rep, None)])
    one.begin_forward(2, F)
    assert one.self_attn_args("mid", 16, 32, 2, 2 * F, F) is a_rep


def test_merge_refuses_different_bases_and_batches():
    store, F = _store(), 2
    b1 = dict(edit_bf_start=F, row_mode=_lib.ATTN_REPLACE, base=torch.zeros(F, 1, 4, 8, dtype=torch.float16), cache_ld=8)
    b2 = dict(b1, base=torch.zeros(F, 1, 4, 8, dtype=torch.float16))
    b = controllers.AttentionControlEditBatch([StubEdit(store, b1, None), StubEdit(store, b2, None)])
    with pytest.raises(RuntimeError, match="CFG batch"):
        b.begin_forward(2, F)
    b.begin_forward(4, F)
    with pytest.raises(RuntimeError, match="disagree"):
        b.self_attn_args("mid", 4, 8, 1, 4 * F, F)


def test_construction_refusals():
    s1, s2 = _store(), _store()
    with pytest.raises(ValueError, match="same additional_attention_store"):
        controllers.AttentionControlEditBatch([StubEdit(s1, None, None), StubEdit(s2, None, None)])
    with pytest.raises(ValueError, match="num_steps"):
        controllers.AttentionControlEditBatch([StubEdit(s1, None, None), StubEdit(s1, None, None, num_steps=6)])
    with pytest.raises(ValueError, match="num_steps and use_inversion_attention"):
        controllers.AttentionControlEditBatch([StubEdit(s1, None, None), StubEdit(s1, None, None, use_inversion_attention=False)])
    with pytest.raises(ValueError, match="1..8"):
        controllers.AttentionControlEditBatch([StubEdit(s1, None, None) for _ in range(9)])
    spilled = types.SimpleNamespace(disk_store=False, host_spill=True)
    with pytest.raises(NotImplementedError, match="host_spill"):
        controllers.AttentionControlEditBatch([StubEdit(spilled, None, None)])


def test_step_blend_and_graph_composition():
    store = _store()
    kids = [StubEdit(store, None, None, blend=dict(apply_blend=True)), StubEdit(store, None, None), StubEdit(store, None, None)]
    b = controllers.AttentionControlEditBatch(kids)
    b.num_att_layers = 32
    assert all(k.num_att_layers == 32 for k in kids)
    assert b.latent_blend_args(8, 8) == [dict(apply_blend=True), None, None]
    x = torch.arange(3 * 4 * 2 * 2 * 2, dtype=torch.float32).view(3, 4, 2, 2, 2)
    b.step_callback(x, blend_fused=True)
    for k, kid in enumerate(kids):
        assert kid.stepped[0].shape == (1, 4, 2, 2, 2) and torch.equal(kid.stepped[0], x[k:k + 1])
    assert b.cur_step == 1
    sig = b.graph_signature()
    assert sig[0] == "edit_batch" and sig[-1] == "plan-7" and len(sig[1]) == 3


def _cpu_pipe():
    from _helpers import build_product
    return build_product("mini", dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128), device="cpu")


def test_batch_api_refusals_before_gpu_work():
    pipe = _cpu_pipe()
    p2p = dict(is_replace_controller=True, cross_replace_steps={"default_": 0.5}, self_replace_steps=0.5, use_inversion_attention=True)
    src = "a silver jeep driving down a curvy road"
    kw = dict(source_prompt=src, num_inference_steps=5, guidance_scale=7.5)
    x = torch.zeros(1, 4, 2, 8, 8)
    with pytest.raises(ValueError, match="128"):
        pipe.p2preplace_edit_batch([src] * 5, [p2p] * 5, latents=torch.zeros(1, 4, 16, 8, 8), **kw)
    with pytest.raises(ValueError, match="at most 8"):
        pipe.p2preplace_edit_batch([src] * 9, [p2p] * 9, latents=x, **kw)
    with pytest.raises(ValueError, match="num_inference_steps"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p, dict(p2p, num_inference_steps=10)], latents=x, **kw)
    with pytest.raises(ValueError, match="guidance_scale"):
        pipe.p2preplace_edit_batch([src] * 2, [dict(p2p, guidance_scale=5.0), p2p], latents=x, **kw)
    with pytest.raises(NotImplementedError, match="eta"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p, dict(p2p, eta=0.5)], latents=x, **kw)
    with pytest.raises(ValueError, match="p2p configs"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p], latents=x, **kw)
    with pytest.raises(ValueError, match=r"\[1, 4, F, h, w\]"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p] * 2, latents=torch.zeros(2, 4, 2, 8, 8), **kw)
    pipe.store_controller.host_spill = True
    with pytest.raises(NotImplementedError, match="host_spill"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p] * 2, latents=x, **kw)
    pipe.store_controller.host_spill = False
    pipe.unet._engine = types.SimpleNamespace(shard=(0, 2, None))
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        pipe.p2preplace_edit_batch([src] * 2, [p2p] * 2, latents=x, **kw)


def test_new_c_abi_symbols_exported():
    lib = _lib.load()
    for name in ("fz_attention_grouped_f16", "fz_cfg_ddim_step_batched", "fz_groupnorm_batched_nhwc_f16"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert _lib.MAX_ATTN_GROUPS == 8
    import ctypes
    # fz_attn_groups_t: int n_groups + 8 x {int, 3 pointers}
    assert ctypes.sizeof(_lib.AttnGroups) == 8 + 8 * 32
