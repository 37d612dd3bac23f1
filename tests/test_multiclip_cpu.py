"""CPU checks of the multi-clip inversion and edit: the group tables of controllers.AttentionStoreBatch / AttentionControlEditClips (with
stub children), the input refusals of prepare_latents_ddim_inverted_batch / p2preplace_edit_clips (all raised before any GPU work), the
HBM admission arithmetic and the new C-ABI symbols and structures."""
import ctypes
import os
import re
import types

import pytest
import torch

from fatezero_b200 import _lib, controllers
from test_edit_batch_cpu import StubEdit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class StubStore(controllers.AttentionStore):
    """A real AttentionStore whose slabs are allocated on the CPU."""

    def __init__(self):
        super().__init__(host_spill=False)

    def _store_self(self, place, S, T, heads, nb):
        start = self._edit_start(nb)
        slab = torch.empty((nb - start, heads, S, T), dtype=torch.float16)
        self.step_store[controllers._key(place, False)].append(slab)
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=slab, cache_ld=T)

    def _store_cross(self, place, S, heads, nb):
        start = self._edit_start(nb)
        key = controllers._key(place, True)
        pos = self._pos[key]
        self._pos[key] += 1
        slab = torch.empty((nb - start, heads, S, controllers.CROSS_LD), dtype=torch.float16)
        self.step_store[key].append(slab[..., :77])
        acc = self._acc.setdefault(key, [])
        if len(acc) <= pos:
            acc.append(torch.zeros_like(slab))
        return dict(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=slab, cache_ld=controllers.CROSS_LD, acc=acc[pos])


def _stores(K):
    out = []
    for _ in range(K):
        s = StubStore()
        s.LOW_RESOURCE = True
        out.append(s)
    return out


@pytest.mark.parametrize("kind,T", [("mid", 16), ("prev_first", 32)])
@pytest.mark.parametrize("K", [1, 2, 3])
def test_store_batch_groups(K, kind, T):
    F, S, heads = 2, 16, 2
    stores = _stores(K)
    b = controllers.AttentionStoreBatch(stores)
    b.begin_forward(K, F)
    got = b.self_attn_args("down", S, T, heads, K * F, F)
    x = b.cross_attn_args("down", S, heads, K * F, F)
    for k, s in enumerate(stores):
        slab = s.step_store["down_self"][0]
        assert slab.shape == (F, heads, S, T)  # exactly the slab of a batch-1 inversion
        assert s.step_store["down_cross"][0].shape == (F, heads, S, 77)
    if K == 1:
        assert got["row_mode"] == _lib.ATTN_STORE and got["store"] is stores[0].step_store["down_self"][0]
        return
    assert got["edit_bf_start"] == 0 and got["cache_ld"] == T and "store" not in got
    assert [g["row_mode"] for g in got["groups"]] == [_lib.ATTN_STORE] * K
    assert [g["store"] for g in got["groups"]] == [s.step_store["down_self"][0] for s in stores]
    assert [g["acc"] for g in got["groups"]] == [None] * K
    assert x["cache_ld"] == controllers.CROSS_LD
    for k, (g, s) in enumerate(zip(x["groups"], stores)):
        assert g["store"][..., :77].data_ptr() == s.step_store["down_cross"][0].data_ptr()
        assert g["acc"] is s._acc["down_cross"][0]
    # latents split per clip, every store advances
    xt = torch.arange(K * 4 * F * 2 * 2, dtype=torch.float32).view(K, 4, F, 2, 2)
    b.step_callback(xt)
    for k, s in enumerate(stores):
        assert s.cur_step == 1 and torch.equal(s.latents_store[0], xt[k:k + 1]) and len(s.attention_store_all_step) == 1


def test_store_batch_construction_and_graph_ids():
    with pytest.raises(ValueError, match="1..8"):
        controllers.AttentionStoreBatch([controllers.AttentionStore(host_spill=False) for _ in range(9)])
    s = controllers.AttentionStore(host_spill=False)
    with pytest.raises(ValueError, match="twice"):
        controllers.AttentionStoreBatch([s, s])
    with pytest.raises(NotImplementedError, match="host_spill"):
        controllers.AttentionStoreBatch([s, controllers.AttentionStore(host_spill=True)])
    with pytest.raises(ValueError, match="save_self_attention"):
        controllers.AttentionStoreBatch([s, controllers.AttentionStore(save_self_attention=False, host_spill=False)])
    with pytest.raises(TypeError):
        controllers.AttentionStoreBatch([s, object()])
    stores = [controllers.AttentionStore(host_spill=False) for _ in range(3)]
    b = controllers.AttentionStoreBatch(stores)
    with pytest.raises(RuntimeError, match="batch of 3"):
        b.begin_forward(6, 2)
    b.num_att_layers = 32
    assert all(x.num_att_layers == 32 for x in stores)
    assert b.is_pristine() and b.graph_signature() == ("store_batch", 3, True, stores[0].graph_signature())
    assert controllers.AttentionStoreBatch(stores, store_maps=False).graph_signature()[2] is False
    b._graph_plan_id = 77
    assert [x._graph_plan_id for x in stores] == [(77, 0), (77, 1), (77, 2)]


def _cross(F, acc, xe, base):
    return dict(edit_bf_start=F, row_mode=_lib.ATTN_CROSSEDIT, base=base, cache_ld=80, acc=acc, xedit=xe)


def test_edit_clips_groups_mixed_jobs_per_clip():
    F = 2
    sA, sB = types.SimpleNamespace(disk_store=False, host_spill=False), types.SimpleNamespace(disk_store=False, host_spill=False)
    baseA, baseB = torch.zeros(F, 2, 16, 32, dtype=torch.float16), torch.zeros(F, 2, 16, 32, dtype=torch.float16)
    xA, xB = torch.zeros(F, 2, 16, 80, dtype=torch.float16), torch.zeros(F, 2, 16, 80, dtype=torch.float16)
    m = torch.ones(F, 16)
    acc = [torch.zeros(F, 2, 16, 80, dtype=torch.float16) for _ in range(3)]
    kids = [StubEdit(sA, dict(edit_bf_start=F, row_mode=_lib.ATTN_REPLACE, base=baseA, cache_ld=32), _cross(F, acc[0], "t0", xA)),
            StubEdit(sB, dict(edit_bf_start=F, row_mode=_lib.ATTN_BLEND, base=baseB, cache_ld=32, mask=m), _cross(F, acc[1], "t1", xB)),
            StubEdit(sA, None, _cross(F, acc[2], "t2", xA))]
    b = controllers.AttentionControlEditClips(kids)
    b.begin_forward(6, F)
    got = b.self_attn_args("up", 16, 32, 2, 6 * F, F)
    assert got["edit_bf_start"] == 3 * F and "base" not in got and got["cache_ld"] == 32
    assert [g["row_mode"] for g in got["groups"]] == [_lib.ATTN_REPLACE, _lib.ATTN_BLEND, _lib.ATTN_NONE]
    assert got["groups"][0]["base"] is baseA and got["groups"][1]["base"] is baseB and got["groups"][1]["mask"] is m
    x = b.cross_attn_args("up", 16, 2, 6 * F, F)
    assert [g["base"] for g in x["groups"]] == [xA, xB, xA] and [g["acc"] for g in x["groups"]] == acc
    for k in kids:
        assert k.asked == [("begin", 2, F), ("self", "up", 16, 32, 2, 2 * F, F), ("cross", "up", 16, 2, 2 * F, F)]
    # the plan key records which clip each job reads
    sig = b.graph_signature()
    assert sig[0] == "edit_clips" and sig[2] == (0, 1, 0) and sig[-1] == ("plan-7",) * 3
    with pytest.raises(AttributeError):
        b.additional_attention_store  # noqa: B018
    bad = controllers.AttentionControlEditClips([StubEdit(sA, dict(edit_bf_start=F, row_mode=_lib.ATTN_REPLACE, base=baseA, cache_ld=32), None),
                                                 StubEdit(sB, dict(edit_bf_start=F, row_mode=_lib.ATTN_REPLACE, base=baseA[:1], cache_ld=32), None)])
    bad.begin_forward(4, F)
    with pytest.raises(RuntimeError, match="geometry"):
        bad.self_attn_args("up", 16, 32, 2, 4 * F, F)
    with pytest.raises(ValueError, match="num_steps"):
        controllers.AttentionControlEditClips([StubEdit(sA, None, None), StubEdit(sB, None, None, num_steps=6)])
    with pytest.raises(NotImplementedError, match="host_spill"):
        controllers.AttentionControlEditClips([StubEdit(sA, None, None), StubEdit(types.SimpleNamespace(disk_store=False, host_spill=True), None, None)])
    # the single-clip batch keeps refusing stores of different clips
    with pytest.raises(ValueError, match="same additional_attention_store"):
        controllers.AttentionControlEditBatch([StubEdit(sA, None, None), StubEdit(sB, None, None)])


def test_map_cache_bytes_sd14():
    """SD-1.4 at 512x512 (64x64 latents), 8 heads: maps are stored at the 32x32, 16x16 and 8x8 levels (5 + 5 + 1 layers)."""
    from fatezero_b200 import synth
    cfg = synth.UNET_CONFIGS["sd14"]
    per_step, once = controllers.map_cache_bytes(cfg, dict(SparseCausalAttention_index=["mid"]), 64, 64)
    heads = cfg["attention_head_dim"]
    want = sum(n * heads * S * (S + 80) * 2 for n, S in ((5, 1024), (5, 256), (1, 64)))
    assert per_step == want
    assert once == sum(n * heads * S * 80 * 2 for n, S in ((5, 1024), (5, 256), (1, 64)))
    two, _ = controllers.map_cache_bytes(cfg, dict(SparseCausalAttention_index=[-1, "first"]), 64, 64)
    assert two - per_step == sum(n * heads * S * S * 2 for n, S in ((5, 1024), (5, 256), (1, 64)))
    # least_sc_channel: the layers below it (the 640-channel 32x32 level) attend to their own frame only (one K/V slot)
    narrow, _ = controllers.map_cache_bytes(cfg, dict(SparseCausalAttention_index=[-1, "first"], least_sc_channel=1280), 64, 64)
    assert narrow == per_step + sum(n * heads * S * S * 2 for n, S in ((5, 256), (1, 64)))
    no_self, _ = controllers.map_cache_bytes(cfg, dict(SparseCausalAttention_index=["mid"]), 64, 64, save_self_attention=False)
    assert no_self == once


def _cpu_pipe():
    from _helpers import build_product
    return build_product("mini", dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128), device="cpu")


def test_map_cache_admission():
    pipe = _cpu_pipe()
    per_step, once = controllers.map_cache_bytes(dict(pipe.unet.config), dict(pipe.unet.model_config), 8, 8)
    need = 3 * 2 * (5 * per_step + once)
    assert pipe.map_cache_admission(3, 2, 8, 8, 5, free_bytes=need) == need
    with pytest.raises(ValueError, match=r"3 clips x 2 frames x 5 steps need .* GiB.*smaller batches"):
        pipe.map_cache_admission(3, 2, 8, 8, 5, free_bytes=need - 1)


def test_inversion_batch_refusals_before_gpu_work():
    pipe = _cpu_pipe()
    src = "a silver jeep driving down a curvy road"
    z = torch.zeros(1, 4, 2, 8, 8)
    inv = pipe.prepare_latents_ddim_inverted_batch
    with pytest.raises(ValueError, match="either images or latents"):
        inv([src])
    with pytest.raises(ValueError, match="2 source prompts and 1 clips"):
        inv([src, src], latents=[z])
    with pytest.raises(ValueError, match="at most 8"):
        inv([src] * 9, latents=[z] * 9)
    with pytest.raises(ValueError, match="differ in"):
        inv([src] * 2, latents=[z, torch.zeros(1, 4, 3, 8, 8)])
    with pytest.raises(ValueError, match="differ in"):
        inv([src] * 2, latents=[z, torch.zeros(1, 4, 2, 8, 16)])
    with pytest.raises(ValueError, match=r"\[1, 4, F, h, w\]"):
        inv([src], latents=[torch.zeros(2, 4, 2, 8, 8)])
    with pytest.raises(ValueError, match=r"\[F, 3, H, W\]"):
        inv([src], images=[torch.zeros(1, 2, 3, 64, 64)])
    with pytest.raises(ValueError, match="8 clips x 24 frames = 192 rows exceed 128"):
        inv([src] * 8, latents=[torch.zeros(1, 4, 24, 8, 8)] * 8)
    with pytest.raises(ValueError, match="generators"):
        inv([src] * 2, latents=[z, z], generator=[torch.Generator()])
    pipe.store_controller.disk_store = True
    with pytest.raises(NotImplementedError, match="disk_store"):
        inv([src] * 2, latents=[z, z])
    pipe.store_controller.disk_store = False
    pipe.unet._engine = types.SimpleNamespace(shard=(0, 2, None))
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        inv([src] * 2, latents=[z, z])


def test_edit_clips_refusals_before_gpu_work():
    pipe = _cpu_pipe()
    src = "a silver jeep driving down a curvy road"
    p2p = dict(is_replace_controller=True, cross_replace_steps={"default_": 0.5}, self_replace_steps=0.5, use_inversion_attention=True)

    def store(n=5, **kw):
        s = controllers.AttentionStore(host_spill=False, **kw)
        s.attention_store_all_step = [{}] * n
        return s

    A, B = store(), store()
    z = torch.zeros(1, 4, 2, 8, 8)

    def job(st=A, lat=z, **kw):
        return dict(store=st, latents=lat, prompt=src, source_prompt=src, **p2p, **kw)

    ed = lambda jobs: pipe.p2preplace_edit_clips(jobs, 5, 7.5)  # noqa: E731
    with pytest.raises(ValueError, match="no jobs"):
        ed([])
    with pytest.raises(ValueError, match="at most 8"):
        ed([job()] * 9)
    with pytest.raises(ValueError, match="lacks"):
        ed([dict(job(), store=None)])
    with pytest.raises(ValueError, match="differ in shape"):
        ed([job(), job(B, torch.zeros(1, 4, 2, 8, 16))])
    with pytest.raises(ValueError, match="differ in shape"):
        ed([job(), job(B, torch.zeros(1, 4, 3, 8, 8))])
    with pytest.raises(ValueError, match=r"2 x 5 jobs x 16 frames = 160 CFG rows exceed 128"):
        ed([job(lat=torch.zeros(1, 4, 16, 8, 8))] * 5)
    with pytest.raises(ValueError, match="inversion steps"):
        ed([job(), job(store(n=10))])
    with pytest.raises(ValueError, match="num_inference_steps"):
        ed([job(), job(B, num_inference_steps=10)])
    with pytest.raises(ValueError, match="guidance_scale"):
        ed([job(), job(B, guidance_scale=5.0)])
    with pytest.raises(NotImplementedError, match="eta"):
        ed([job(), job(B, eta=0.5)])
    spilled = store()
    spilled.host_spill = True
    with pytest.raises(NotImplementedError, match="host_spill"):
        ed([job(), job(spilled)])
    A._graph_plan_id, B._graph_plan_id = 5, 5
    with pytest.raises(ValueError, match="same captured inversion slot"):
        ed([job(A), job(B)])
    A._graph_plan_id, B._graph_plan_id = (5, 0), (5, 1)
    pipe.unet._engine = types.SimpleNamespace(shard=(0, 2, None))
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        ed([job(A), job(B)])


def _header_struct(name):
    hdr = open(os.path.join(ROOT, "include", "fatezero_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s_t;" % (name, name), hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [re.sub(r"\[.*\]", "", d.split()[-1]).lstrip("*") for d in body.split(";") if d.strip()]


def test_c_abi_structs_and_symbols():
    assert [f[0] for f in _lib.AttnGroup._fields_] == _header_struct("fz_attn_group")
    assert [f[0] for f in _lib.AttnSlabs._fields_] == _header_struct("fz_attn_slabs")
    assert ctypes.sizeof(_lib.AttnSlabs) == 2 * 8 * _lib.MAX_ATTN_GROUPS
    lib = _lib.load()
    for name in ("fz_attention_grouped_slabs_f16", "fz_cfg_ddim_step_multi"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    hdr = open(os.path.join(ROOT, "include", "fatezero_b200.h")).read()
    assert set(re.findall(r"\b(fz_[a-z0-9_]+)\s*\(", hdr)) - {"fz_last_error"} <= set(_lib.SIGNATURES)


def test_batch_inversion_releases_previous_stores_and_skips_admission_on_replay(monkeypatch):
    """The previous batch's stores are dropped before the admission counts free HBM, and a batch that will replay a captured inversion
    (which refills that plan's caches) is not admitted a second time."""
    pipe = _cpu_pipe()
    pipe.scheduler.set_timesteps(5)
    src = "a silver jeep driving down a curvy road"
    admitted, held = [], []
    monkeypatch.setattr(pipe, "map_cache_admission", lambda *a, **k: admitted.append(a))

    def loop(lat, text, ctrl):
        held.append(pipe.store_controllers)
        return [lat] * 6
    monkeypatch.setattr(pipe, "ddim_clean2noisy_loop", loop)
    z = torch.zeros(1, 4, 2, 8, 8)
    pipe.store_controllers = ["the previous batch's stores"]
    lats = pipe.prepare_latents_ddim_inverted_batch([src, src], latents=[z, z])
    assert held == [None] and len(admitted) == 1 and len(pipe.store_controllers) == 2 and len(lats[1]) == 6
    stores = [controllers.AttentionStore(host_spill=False) for _ in range(2)]
    for st in stores:
        st.LOW_RESOURCE = True  # as the stores of a captured inversion are
    sig = controllers.AttentionStoreBatch(stores).graph_signature()
    ts = tuple(int(t) for t in pipe.scheduler.timesteps)
    pipe._plans[("inv", (2, 4, 2, 8, 8), "torch.float32", ts, (2, 77, 32), sig, 0, None)] = object()
    pipe.prepare_latents_ddim_inverted_batch([src, src], latents=[z, z])
    assert len(admitted) == 1
    pipe.prepare_latents_ddim_inverted_batch([src, src, src], latents=[z, z, z])  # another batch size: no plan to replay
    assert len(admitted) == 2
    pipe.graph_mode = "off"
    pipe.prepare_latents_ddim_inverted_batch([src, src], latents=[z, z])
    assert len(admitted) == 3
