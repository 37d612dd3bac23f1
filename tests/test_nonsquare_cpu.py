"""Non-square clips without a GPU: the fp32 oracle against the reference goldens of a landscape (32x48 latents) and a portrait (48x32)
clip, the map levels (level_hw) at SD-1.4 / SD-2 geometries, the size refusals, the map-cache size at 512x768, the heat-map level
choice and tile shape on the host path, and the new C-ABI entry points."""
import os
import re

import numpy as np
import pytest
import torch

import _nonsquare as nsr
from _helpers import ROOT
from fatezero_b200 import _lib, controllers, synth, visualization
from fatezero_b200.spatial_blend import level_hw
from oracle import fz_oracle as fo
from oracle import nonsquare as ns
from oracle import sd2


# ------------------------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("name", ns.NONSQUARE_REF_CASES)
def test_oracle_matches_reference_golden_nonsquare(name):
    """test_sd2_cpu.py::test_oracle_matches_reference_golden_sd2's bounds on the compact golden: single forward 5e-5, inversion 1e-4,
    edit 1e-3 of max(1, |x|max) per step; stored maps: the same keys and shapes, slices 1e-3 (fp16 fixture), sums 1e-3 relative."""
    g = nsr.load(name)
    case = ns.NONSQUARE_CASES[name]
    ou = nsr.build_oracle(case["unet"], case["model_config"])
    x2, t, emb = ns.fwd_inputs(case, ns.case_inputs(case))
    eps = sd2.sample(ou.forward(x2, t, emb), g["eps_stride"])
    assert (eps - g["fwd_eps_sample"]).abs().max().item() < 5e-5
    out = nsr.run_oracle(case, ou)
    inv = torch.stack([sd2.sample(v, g["lat_stride"]) for v in out["inv_latents"]])
    assert inv.shape == g["inv_sample"].shape
    assert (inv - g["inv_sample"]).abs().max().item() < 1e-4
    ed = torch.stack([sd2.sample(v, g["lat_stride"]) for v in out["edit_latents"]])
    assert ed.shape == g["edit_sample"].shape
    d = (ed - g["edit_sample"]).abs().amax(dim=1)
    scale = g["edit_sample"].abs().amax(dim=1)
    assert bool((d <= 1e-3 * scale.clamp(min=1.0)).all()), (d.tolist(), scale.tolist())
    mine = {f"{s}/{k}/{p}": t for s, dct in enumerate(out["store"].all_step) for k, lst in dct.items() for p, t in enumerate(lst)}
    assert {k: list(v.shape) for k, v in mine.items()} == g["map_shapes"]
    # the first level (h x w latents, more than 32**2 pixels) is not stored: the largest stored map is the half-size level
    assert max(v[2] for v in g["map_shapes"].values()) == (case["h"] // 2) * (case["w"] // 2)
    for k, v in g["maps"].items():
        assert (sd2.map_slice(mine[k]) - v.float()).abs().max().item() < 1e-3
    for k, s in g["map_sums"].items():
        t = mine[k].double()
        assert abs(float(t.sum()) - s) <= 1e-3 * max(1.0, abs(s))
        assert abs(float((t ** 2).sum()) - g["map_sqsums"][k]) <= 1e-3 * abs(g["map_sqsums"][k])


def test_oracle_blend_restatement_reduces_to_square():
    """oracle/nonsquare.py's blend_mask on a square clip equals fz_oracle.blend_mask (the reference's square rule), and OracleEditNS on a
    square case gives fz_oracle.OracleEdit's latents and masks."""
    g = torch.Generator().manual_seed(3)
    maps = [torch.softmax(torch.randn(2, 4, 256, 77, generator=g) * 2, -1) for _ in range(5)]
    alpha = torch.zeros(77)
    alpha[[2, 5]] = 1
    for h, w, lat in ((64, 64, (64, 64)), (16, 16, (64, 64)), (82, 94, (32, 32))):
        assert torch.equal(fo.blend_mask(maps, alpha, 0.4, h, w), ns.blend_mask(maps, alpha, 0.4, h, w, lat))
    # one inversion, two edits: 1 frame of 64x64 latents (the blender's maps are then all 16x16), 2 + 2 steps
    case = dict(ns.NONSQUARE_CASES["ns_replace_blend"], frames=1, h=64, w=64, steps=2)
    p = case["p2p"]
    ou = nsr.build_oracle(case["unet"], case["model_config"])
    tok, te = synth.ToyTokenizer(), synth.ToyTextEncoder(synth.UNET_CONFIGS["mini"]["cross_attention_dim"])
    store = fo.OracleStore()
    inv = fo.invert(ou, ns.case_inputs(case), fo.encode_prompts(tok, te, case["source"])[1:], 2, store)
    plan = fo.EditPlan(tok, case["source"], case["target"], 2, p["cross_replace_steps"], p["self_replace_steps"], True, None,
                       p["blend_words"], True, True, p["blend_th"])
    emb = fo.encode_prompts(tok, te, case["target"])
    got, ref = ns.OracleEditNS(plan, store, (64, 64)), fo.OracleEdit(plan, store)
    assert torch.equal(torch.stack(fo.edit(ou, inv[-1], emb, 2, got)), torch.stack(fo.edit(ou, inv[-1], emb, 2, ref)))
    assert len(got.mask_list) == 2 and all(torch.equal(a, b) for a, b in zip(got.mask_list, ref.mask_list))


# ------------------------------------------------------------------------------------------------------------------ levels
def _stored_levels(cfg: dict, h: int, w: int):
    """place -> levels k of the stored cross-attention layers ((h >> k) * (w >> k) <= 32**2) of the UNet at latent h x w, in run order."""
    nblk = len(cfg["block_out_channels"])
    lpb = cfg["layers_per_block"]
    down = [i for i, t in enumerate(cfg["down_block_types"]) if t.startswith("CrossAttn") for _ in range(lpb)]
    up = [nblk - 1 - i for i, t in enumerate(cfg["up_block_types"]) if t.startswith("CrossAttn") for _ in range(lpb + 1)]
    keep = lambda ks: [k for k in ks if (h >> k) * (w >> k) <= 32 ** 2]  # noqa: E731
    return dict(down=keep(down), mid=keep([nblk - 1]), up=keep(up))


@pytest.mark.parametrize("unet", ["sd14", "sd2"])
@pytest.mark.parametrize("px", [(512, 768), (768, 512), (512, 896), (384, 512)], ids=str)
def test_level_hw(unet, px):
    H, W = px
    h, w = H // 8, W // 8
    levels = [k for ks in _stored_levels(synth.UNET_CONFIGS[unet], h, w).values() for k in ks]
    for k in levels:
        S = (h >> k) * (w >> k)
        assert level_hw(S, h, w) == (h >> k, w >> k) == ns.level_hw(S, h, w)
    expect = {(512, 768): [(16, 24), (8, 12)], (768, 512): [(24, 16), (12, 8)], (512, 896): [(16, 28), (8, 14)],
              (384, 512): [(24, 32), (12, 16), (6, 8)]}[px]
    assert sorted({(h >> k, w >> k) for k in levels}, reverse=True) == expect
    with pytest.raises(ValueError):
        level_hw(256, h, w)  # no 16x16 level in these clips
    assert level_hw(64 * 64, 64, 64) == (64, 64) and level_hw(16 * 16, 64, 64) == (16, 16)


def test_blend_maps_share_one_level_at_512x768():
    """down_cross[2:4] + up_cross[:3] of what is stored: at 512x768 the 32x48 level is not stored, so down_cross holds only the two 16x24
    maps of down block 2 and the blender reads the three 16x24 maps of up block 1."""
    for unet in ("sd14", "sd2"):
        lv = _stored_levels(synth.UNET_CONFIGS[unet], 64, 96)
        assert lv == dict(down=[2, 2], mid=[3], up=[2, 2, 2])
        picked = lv["down"][2:4] + lv["up"][:3]
        assert picked == [2, 2, 2] and level_hw((64 >> 2) * (96 >> 2), 64, 96) == (16, 24)


# ------------------------------------------------------------------------------------------------------------------ refusals
def _cpu_pipe():
    return nsr.build_product("mini", dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128), device="cpu")


def test_size_refusals_before_gpu_work():
    pipe = _cpu_pipe()
    src = "a silver jeep driving down a curvy road"
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.sd_ddim_pipeline(prompt=src, height=512, width=600)
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.sd_ddim_pipeline(prompt=src, latents=torch.zeros(1, 4, 2, 64, 75), height=512, width=512)
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.prepare_latents_ddim_inverted(torch.zeros(2, 3, 512, 600), 1, 1, None)
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.prepare_latents_ddim_inverted_batch([src], latents=[torch.zeros(1, 4, 2, 64, 75)])
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.prepare_latents_ddim_inverted_batch([src], images=[torch.zeros(2, 3, 512, 600)])
    st = controllers.AttentionStore(host_spill=False)
    st.attention_store_all_step = [{}] * 5
    job = dict(store=st, latents=torch.zeros(1, 4, 2, 60, 96), prompt=src, source_prompt=src, is_replace_controller=True,
               cross_replace_steps={"default_": 0.5}, self_replace_steps=0.5, use_inversion_attention=True)
    with pytest.raises(ValueError, match="multiples of 64"):
        pipe.p2preplace_edit_clips([job], 5, 7.5)
    # accepted: square sizes keep the multiple-of-8 rule, non-square multiples of 64
    for hw in ((520, 520), (512, 768), (768, 512), (512, 896), (384, 512), (64, 128)):
        pipe.check_frame_size(*hw, "test")


# ------------------------------------------------------------------------------------------------------------------ map cache
def test_map_cache_bytes_512x768():
    """SD-1.4 at 512x768 (64x96 latents), ['mid'] K/V frames from 640 channels on: the stored layers are down block 2 (2 x 16x24), the mid
    block (8x12) and up block 1 (3 x 16x24), 8 heads, one K/V slot; the 32x48 level (1536 pixels) is not stored."""
    mc = dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=640)
    per_step, once = controllers.map_cache_bytes(synth.SD14_UNET_CONFIG, mc, 64, 96)
    # by hand: 5 layers of 8 x 384 x (384 + 80) fp16 and one of 8 x 96 x (96 + 80); the running sums are 8 x S x 80 fp16
    assert per_step == 5 * 8 * 384 * 464 * 2 + 8 * 96 * 176 * 2 == 14524416
    assert once == 5 * 8 * 384 * 80 * 2 + 8 * 96 * 80 * 2 == 2580480


# ------------------------------------------------------------------------------------------------------------------ heat maps
class _ForeignStore:
    """A store that is not one of this package's controllers: show_cross_attention takes the host path."""

    def __init__(self, maps, latent_hw=None):
        self._maps = maps
        if latent_hw is not None:
            self._latent_hw = latent_hw

    def get_average_attention(self):
        return self._maps


def test_heatmap_level_by_shorter_side_and_tile_shape():
    g = torch.Generator().manual_seed(5)
    F, heads = 2, 2
    m16 = torch.rand(F, heads, 16 * 24, 77, generator=g)
    m8 = torch.rand(F, heads, 8 * 12, 77, generator=g)
    store = _ForeignStore({"down_cross": [m16, m16], "mid_cross": [m8], "up_cross": [m8, m16]}, (64, 96))
    agg = visualization.aggregate_attention(["a b"], store, 16, ["up", "down"], True, 0)
    assert agg.shape == (F, 16, 24, 77)
    ref = torch.stack([m16.reshape(F, heads, 16, 24, 77)] * 3, 0).mean(0).mean(1)
    assert torch.allclose(agg, ref, atol=1e-6)
    assert visualization.aggregate_attention(["a b"], store, 8, ["mid"], True, 0).shape == (F, 8, 12, 77)
    tok = synth.ToyTokenizer()
    strips = visualization.show_cross_attention(tok, "a silver jeep", store, 16, ["up", "down"])
    ntok = len(tok.encode("a silver jeep"))
    assert len(strips) == F and strips[0].shape == (256 + int(256 * 0.2), ntok * 384, 3) and strips[0].dtype == np.uint8
    portrait = _ForeignStore({"down_cross": [torch.rand(F, heads, 24 * 16, 77, generator=g)]}, (96, 64))
    assert visualization.show_cross_attention(tok, "a jeep", portrait, 16, ["down"])[0].shape[1] == len(tok.encode("a jeep")) * 170
    with pytest.raises(ValueError, match="resolution 32"):
        visualization.show_cross_attention(tok, "a jeep", store, 32, ["up", "down"])
    # a store without a latent size: square maps of exactly res**2 pixels, as the reference picks them
    with pytest.raises(ValueError, match="resolution 16"):
        visualization.aggregate_attention(["a b"], _ForeignStore(store._maps), 16, ["up", "down"], True, 0)
    sq = _ForeignStore({"up_cross": [torch.rand(F, heads, 256, 77, generator=g)]})
    assert visualization.show_cross_attention(tok, "a jeep", sq, 16, ["up"])[0].shape[:2] == (256 + 51, len(tok.encode("a jeep")) * 256)


def test_controllers_record_latent_size():
    store = controllers.AttentionStore(host_spill=False)
    store.begin_forward(1, 2)
    assert store._latent_hw is None
    store.begin_forward(1, 2, (32, 48))
    assert store._latent_hw == (32, 48) and "_latent_hw" in controllers.AttentionStore._ADOPT
    batch = controllers.AttentionStoreBatch([controllers.AttentionStore(host_spill=False) for _ in range(2)])
    batch.begin_forward(2, 3, (48, 32))
    assert [s._latent_hw for s in batch.stores] == [(48, 32)] * 2
    assert controllers.level_hw is level_hw


# ------------------------------------------------------------------------------------------------------------------ C ABI
def test_c_abi_hw_entry_points():
    hdr = open(os.path.join(ROOT, "include", "fatezero_b200.h")).read()
    lib = _lib.load()
    for name in ("fz_blend_mask_hw", "fz_cross_heatmaps_hw"):
        assert re.search(r"\b%s\s*\(" % name, hdr) and hasattr(lib, name) and name in _lib.SIGNATURES
    # the per-axis entry points take one more int (rw) than the square ones, right after rh
    assert len(_lib.SIGNATURES["fz_blend_mask_hw"]) == len(_lib.SIGNATURES["fz_blend_mask"]) + 1
    assert len(_lib.SIGNATURES["fz_cross_heatmaps_hw"]) == len(_lib.SIGNATURES["fz_cross_heatmaps"]) + 1
