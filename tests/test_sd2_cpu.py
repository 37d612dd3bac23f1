"""Stable Diffusion 2.x base configurations without a GPU: the UNet container's parameter layout against the unmodified reference, the
per-level head counts, the map-cache admission figure, the CPU oracle against the reference goldens of SD2_CASES and the self-check of
the exact-GELU bound (tests/_gelu_ref.py)."""
import gzip
import json
import os

import pytest
import torch

import _sd2_golden as sg
from _gelu_ref import all_finite_f16, gelu_ref
from _helpers import GOLDEN_DIR, case_inputs, run_oracle_case
from fatezero_b200 import controllers, synth
from fatezero_b200.unet import UNetPseudo3DConditionModel, level_heads, transformer_heads, unet_param_spec
from oracle import sd2
from oracle.sd2 import SD2_CASES, SD2_MINI_CASES


def test_spec_equals_reference_state_dict_sd2():
    """Names and shapes of the reference UNet built from the SD-2-base config with lora: 160 (recorded by
    `python -m oracle.make_sd2_golden sd2_shapes`) equal unet_param_spec's: linear [C, C] proj_in / proj_out, [C, 1024] text K / V."""
    rec = json.load(gzip.open(os.path.join(GOLDEN_DIR, "ref_unet_sd2_state_dict_shapes.json.gz")))
    assert rec["model_config"] == dict(lora=160)
    spec = unet_param_spec(dict(synth.SD2_UNET_CONFIG), rec["model_config"])
    ref = rec["shapes"]
    assert set(ref) == set(spec), set(ref) ^ set(spec)
    for k, v in ref.items():
        assert tuple(v) == tuple(spec[k][0]), k
    assert spec["down_blocks.0.attentions.0.proj_in.weight"][0] == (320, 320)
    assert spec["up_blocks.3.attentions.2.proj_out.weight"][0] == (320, 320)
    assert spec["mid_block.attentions.0.transformer_blocks.0.attn2.to_k.weight"][0] == (1280, 1024)


def test_level_heads_follow_the_reference_block_order():
    cfg = synth.SD2_UNET_CONFIG
    assert level_heads(cfg) == [5, 10, 20, 20]
    th = transformer_heads(cfg)
    assert len(th) == 16
    assert th["down_blocks.0.attentions.1"] == 5 and th["down_blocks.2.attentions.0"] == 20
    assert th["mid_block.attentions.0"] == 20
    # up block i takes the REVERSED list's entry i: up_blocks.1 runs at the 1280-channel level, up_blocks.3 at 320 channels
    assert th["up_blocks.1.attentions.0"] == 20 and th["up_blocks.2.attentions.2"] == 10 and th["up_blocks.3.attentions.0"] == 5
    assert all(c // h == 64 for c, h in zip(cfg["block_out_channels"], level_heads(cfg)))
    assert set(transformer_heads(synth.SD14_UNET_CONFIG).values()) == {8}
    with pytest.raises(ValueError):
        level_heads(dict(cfg, attention_head_dim=(5, 10, 20)))
    with pytest.raises(ValueError):
        level_heads(dict(cfg, attention_head_dim=(3, 10, 20, 20)))  # 320 channels do not split into 3 heads


def test_container_accepts_sd2_options_and_keeps_the_other_refusals():
    m = UNetPseudo3DConditionModel(**dict(synth.SD2_MINI_UNET_CONFIG, upcast_attention=True), lora=160)
    assert m.state_dict()["down_blocks.0.attentions.0.proj_in.weight"].shape == (64, 64)
    assert m.state_dict()["down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_v.weight"].shape == (64, 1024)
    for bad in (dict(only_cross_attention=True), dict(dual_cross_attention=True), dict(class_embed_type="timestep"),
                dict(num_class_embeds=10), dict(resnet_time_scale_shift="scale_shift"), dict(center_input_sample=True),
                dict(temporal_downsample=True)):
        with pytest.raises(NotImplementedError):
            UNetPseudo3DConditionModel(**dict(synth.SD2_MINI_UNET_CONFIG, **bad))


def test_map_cache_bytes_per_level():
    """SD-2-base at 512x512 (64x64 latents) with ['mid'] K/V frames from 640 channels on: per frame and DDIM step 130 621 440 B
    (124.57 MiB; SD-1.4: 97 468 416 B = 92.95 MiB), because the 32x32 and 16x16 levels store 10 and 20 heads instead of 8."""
    mc = dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=640)
    assert controllers.map_cache_bytes(synth.SD14_UNET_CONFIG, mc, 64, 64) == (97468416, 8273920)
    per_step, once = controllers.map_cache_bytes(synth.SD2_UNET_CONFIG, mc, 64, 64)
    assert (per_step, once) == (130621440, 12492800)
    # restated layer by layer: (heads, S, K/V slots) of the stored layers (S <= 32^2); 80-wide cross rows
    stored = [(10, 1024, 1)] * 2 + [(20, 256, 1)] * 2 + [(20, 64, 1)] + [(20, 256, 1)] * 3 + [(10, 1024, 1)] * 3
    assert per_step == sum(h * S * (k * S + 80) * 2 for h, S, k in stored)
    assert once == sum(h * S * 80 * 2 for h, S, k in stored)


def test_gelu_bound_selfcheck():
    """The bound of the fz_gelu_f16 parity test accepts an fp32 erf evaluation rounded to fp16 and rejects the tanh approximation and
    quick_gelu (both are what a wrong activation would compute), over every finite fp16 input."""
    x = all_finite_f16()
    ref, bound = gelu_ref(x)
    v = x.float()
    fp32_erf = (0.5 * v * (1.0 + torch.special.erf(v * 0.70710678118654752))).half().double()
    assert bool(((fp32_erf - ref).abs() <= bound).all())
    tanh = torch.nn.functional.gelu(v, approximate="tanh").half().double()
    assert int(((tanh - ref).abs() > bound).sum()) > 100
    quick = (v * torch.sigmoid(1.702 * v)).half().double()
    assert int(((quick - ref).abs() > bound).sum()) > 100


@pytest.mark.parametrize("name", SD2_MINI_CASES)
def test_oracle_matches_reference_golden_sd2(name):
    """The bounds of test_oracle_golden.py::test_oracle_matches_reference_golden at the mini SD-2 geometry, on the golden's strided
    samples of every latent (oracle/sd2.py): single forward 5e-5, inversion 1e-4, edit 1e-3 of max(1, |x|max) per step; stored maps:
    slices 1e-3 (fp16 fixture), sums 1e-3 relative; blend masks < 0.1% mismatched pixels."""
    g = sg.load(name)
    case = SD2_CASES[name]
    ou = sg.build_oracle(case)
    x0 = case_inputs(case)
    x2, t, emb = sd2.fwd_inputs(case, x0)
    eps = sd2.sample(ou.forward(x2, t, emb), g["eps_stride"])
    assert (eps - g["fwd_eps_sample"]).abs().max().item() < 5e-5
    out = run_oracle_case(case, ou)
    inv = sg.samples(out["inv_latents"], g["lat_stride"])
    assert inv.shape == g["inv_sample"].shape
    assert (inv - g["inv_sample"]).abs().max().item() < 1e-4
    sq = sg.sq_sums(out["inv_latents"])
    assert bool(((sq - g["inv_sums"][:, 1]).abs() <= 2e-4 * g["inv_sums"][:, 1].abs()).all())
    ed = sg.samples(out["edit_latents"], g["lat_stride"])
    assert ed.shape == g["edit_sample"].shape
    d = (ed - g["edit_sample"]).abs().amax(dim=1)
    scale = g["edit_sample"].abs().amax(dim=1)
    assert bool((d <= 1e-3 * scale.clamp(min=1.0)).all()), (d.tolist(), scale.tolist())
    for k, v in g["maps"].items():
        step, key, pos = k.split("/")
        mine = sd2.map_slice(out["store"].all_step[int(step)][key][int(pos)])
        assert mine.shape == v.shape and (mine - v.float()).abs().max().item() < 1e-3
    for k, s in g["map_sums"].items():
        step, key, pos = k.split("/")
        t = out["store"].all_step[int(step)][key][int(pos)].double()
        assert abs(float(t.sum()) - s) <= 1e-3 * max(1.0, abs(s))
        assert abs(float((t ** 2).sum()) - g["map_sqsums"][k]) <= 1e-3 * abs(g["map_sqsums"][k])
    if "mask_list" in g:
        assert sg.mask_mismatch(out["ctrl"].mask_list, g["mask_list"]) < 1e-3


def test_oracle_single_forward_sd2_base():
    """SD-2-base geometry: one CFG-batch forward (2 frames) of the oracle against the reference's epsilon of the big golden."""
    name = "sd2_replace_blend"
    g = sg.load(name)
    case = SD2_CASES[name]
    ou = sg.build_oracle(case)
    x2, t, emb = sd2.fwd_inputs(case, case_inputs(case))
    eps = sd2.sample(ou.forward(x2, t, emb), g["eps_stride"])
    assert (eps - g["fwd_eps_sample"]).abs().max().item() < 5e-5
