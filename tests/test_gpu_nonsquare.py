"""Non-square clips on the sm_90a kernels (landscape 32x48 and portrait 48x32 latents at the mini UNet geometry, oracle/nonsquare.py).

  * fz_blend_mask_hw / fz_cross_heatmaps_hw against an fp64 restatement (below) on rh x rw grids; with rh == rw bitwise equal to
    fz_blend_mask / fz_cross_heatmaps.
  * the product against the reference goldens, teacher-forced and free-running, with the mini goldens' bounds (test_gpu_pipeline.py).
  * Replace + self-attention blend + latent blend on 64x96 latents against the fp32 oracle (the reference has no non-square blend).
  * bitwise: a batched edit and a batched inversion equal the single-clip calls; graph replay equals eager.
  * output_type="pil" through the VAE, with heat-map strips of 256 x (256 * rw // rh) tiles.
  * the frame-sharded run at 2 GPUs (tools/shard_check_nonsquare.py; skipped with fewer GPUs)."""
import json
import os
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import _nonsquare as nsr  # noqa: E402
import _sd2_golden as sg  # noqa: E402
from _ref64 import check_heatmaps, check_mask, nearest_index  # noqa: E402
from fatezero_b200 import _lib, controllers, ops, synth, visualization  # noqa: E402
from oracle import nonsquare as ns  # noqa: E402

dev = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRIDS = [(16, 24), (24, 16), (8, 14), (12, 16), (1, 32)]


def rnd(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dev)


def attn_maps(Fr, heads, rh, rw, ldm, seed, dtype=torch.float16):
    return torch.softmax(rnd(Fr, heads, rh * rw, ldm, seed=seed) * 2, -1).to(dtype)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def robust_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return torch.quantile((a - b).abs().reshape(-1), 0.99).item() / (b.abs().max().item() + 1e-12)


# ------------------------------------------------------------------------------------------------------------------ fp64 restatement
def blend_ratio64(maps, word_w, rh, rw, h, w, ntok=77):
    """spatial_blend.py get_mask in fp64 on an rh x rw grid: (sum_n map w_n).mean(layers, heads), 3x3 max-pool (stride 1, pad 1), nearest
    resize to (h, w) with F.interpolate's fp32 source index taken per axis, divided by the per-frame max (NaN where it is 0)."""
    Fr = maps[0].shape[0]
    ww = word_w.double()[:ntok].to(maps[0].device)
    st = torch.stack([(m[..., :ntok].double() * ww).sum(-1) for m in maps]).mean((0, 2)).reshape(Fr, 1, rh, rw)
    pooled = F.max_pool2d(st, 3, 1, 1)[:, 0]
    mk = pooled[:, nearest_index(rh, h).to(dev)][:, :, nearest_index(rw, w).to(dev)]
    return mk / mk.amax((-2, -1), keepdim=True)


def heat64(maps, ntok, rh, rw):
    """fz_cross_heatmaps_hw in fp64: 255 a / max over the rh x rw pixels, a = sum over maps and heads -> [F, ntok, rh, rw]."""
    a = torch.stack([m[..., :ntok].double() for m in maps]).sum((0, 2)).transpose(1, 2)
    mx = a.amax(-1, keepdim=True)
    v = torch.where(mx > 0, 255 * a / mx.clamp(min=1e-300), torch.zeros_like(a))
    return v.reshape(a.shape[0], ntok, rh, rw)


# ------------------------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("grid", GRIDS, ids=str)
def test_blend_mask_hw_vs_fp64(grid, report):
    rh, rw = grid
    Fr, heads = 2, 8
    ww = torch.zeros(77)
    ww[[2, 5, 76]] = 1
    for n_maps, dtype, th in [(1, torch.float16, 0.3), (5, torch.float16, 0.6), (8, torch.float32, 0.5)]:
        maps = [attn_maps(Fr, heads, rh, rw, 80, 200 + i + rh, dtype) * (n_maps if dtype == torch.float32 else 1) for i in range(n_maps)]
        for h, w in [(4 * rh, 4 * rw), (rh, rw), (82, 94), (48, 32)]:
            got = ops.blend_mask(maps, ww, th, h, w, hw=(rh, rw))
            assert got.shape == (Fr, h, w)
            check_mask(got, blend_ratio64(maps, ww, rh, rw, h, w), torch.tensor(th, dtype=torch.float32).item(), report,
                       f"mask_{rh}x{rw}_{h}x{w}_L{n_maps}_{str(dtype)[6:]}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["f16", "f32"])
@pytest.mark.parametrize("grid", GRIDS, ids=str)
def test_cross_heatmaps_hw_vs_fp64(grid, dtype, report):
    rh, rw = grid
    Fr, heads, ntok = 2, 8, 77
    maps = [attn_maps(Fr, heads, rh, rw, 80, 300 + i + rw, dtype) * (3 if dtype == torch.float32 else 1) for i in range(3)]
    for m in maps:
        m[..., 40] = 0  # an all-zero token column: black
    got = ops.cross_heatmaps(maps, ntok, hw=(rh, rw))
    assert got.shape == (Fr, ntok, rh, rw) and torch.all(got[:, 40] == 0)
    check_heatmaps(got.reshape(Fr, ntok, -1), heat64(maps, ntok, rh, rw).reshape(Fr, ntok, -1), report, f"heat_{rh}x{rw}_{str(dtype)[6:]}")


@pytest.mark.parametrize("r", [8, 16, 32])
def test_hw_entry_points_equal_square_ones(r):
    """fz_blend_mask_hw / fz_cross_heatmaps_hw at rh == rw == r are bitwise fz_blend_mask / fz_cross_heatmaps."""
    import ctypes as C
    Fr, heads = 2, 8
    maps = [attn_maps(Fr, heads, r, r, 80, 400 + i) for i in range(5)]
    arr = (C.c_void_p * 5)(*[m.data_ptr() for m in maps])
    ww = torch.zeros(77)
    ww[[3, 4]] = 1
    wv = (C.c_float * 77)(*ww.tolist())
    st = torch.cuda.current_stream().cuda_stream
    for h, w in [(64, 64), (82, 94), (r, r)]:
        old = torch.empty(Fr, h, w, device=dev)
        _lib.call("fz_blend_mask", arr, 5, 0, Fr, heads, r, 80, 77, wv, 0.4, h, w, old.data_ptr(), st)
        assert torch.equal(ops.blend_mask(maps, ww, 0.4, h, w, hw=(r, r)), old)
        assert torch.equal(ops.blend_mask(maps, ww, 0.4, h, w), old)
    old = torch.empty(Fr, 77, r, r, dtype=torch.uint8, device=dev)
    _lib.call("fz_cross_heatmaps", arr, 5, 0, Fr, heads, r, 80, 77, old.data_ptr(), st)
    assert torch.equal(ops.cross_heatmaps(maps, 77, hw=(r, r)), old) and torch.equal(ops.cross_heatmaps(maps, 77), old)


def test_hw_argument_checks():
    maps = [attn_maps(1, 2, 16, 24, 80, 7)]
    with pytest.raises(ValueError, match="not a 24 x 24 grid"):
        ops.blend_mask(maps, torch.ones(77), 0.3, 32, 48, hw=(24, 24))
    with pytest.raises(RuntimeError, match="bad args"):
        ops.cross_heatmaps([attn_maps(1, 2, 33, 32, 80, 8)], 77, hw=(33, 32))  # more than 1024 pixels: not a stored level


# ------------------------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("name", ns.NONSQUARE_REF_CASES)
def test_free_running_vs_oracle_and_golden(name, report):
    """test_gpu_pipeline.py::test_case_vs_oracle_and_golden's bounds: inversion 2e-2 relative, final edit 8e-2 relative, stored maps of
    step 0 3e-3 absolute; against the golden on its strided samples."""
    case = ns.NONSQUARE_CASES[name]
    prod = nsr.run_product(case)
    orc = nsr.run_oracle(case)
    r_inv, r_ed = rel(prod["inv_latents"], orc["inv_latents"]), rel(prod["edit_latents"][-1], orc["edit_latents"][-1])
    store = prod["pipe"].store_controller
    assert store._latent_hw == (case["h"], case["w"])
    worst = 0.0
    for key, lst in store.attention_store_all_step[0].items():
        assert len(lst) == len(orc["store"].all_step[0][key]), key
        for pos, t in enumerate(lst):
            o = orc["store"].all_step[0][key][pos]
            assert t.shape == o.shape, (key, pos)
            worst = max(worst, (t.float().cpu() - o).abs().max().item())
    g = nsr.load(name)
    rg_inv = rel(sg.samples(prod["inv_latents"], g["lat_stride"]), g["inv_sample"])
    rg_ed = rel(sg.samples(prod["edit_latents"], g["lat_stride"])[-1], g["edit_sample"][-1])
    report[name] = dict(inv_rel=r_inv, edit_rel=r_ed, maps_max_abs=worst, golden_inv_rel=rg_inv, golden_edit_rel=rg_ed)
    assert worst < 3e-3
    assert r_inv < 2e-2 and r_ed < 8e-2
    assert rg_inv < 2e-2 and rg_ed < 8e-2


@pytest.mark.parametrize("name", ns.NONSQUARE_REF_CASES)
def test_teacher_forced_vs_golden(name, report):
    """Every forward starts from the reference's latent of that step: each compared latent carries one forward of kernel error, held to
    the free-running bounds (inversion 2e-2, edit 8e-2 relative) at every step."""
    case = ns.NONSQUARE_CASES[name]
    g = nsr.load(name)
    prod = nsr.run_product(case, teacher=sg.teacher(case, g, ns.case_inputs(case)))
    inv = sg.samples(prod["inv_latents"], g["lat_stride"])
    ed = sg.samples(prod["edit_latents"], g["lat_stride"])
    r_inv = [rel(a, b) for a, b in zip(inv[1:], g["inv_sample"][1:])]
    r_ed = [rel(a, b) for a, b in zip(ed, g["edit_sample"])]
    report[name] = dict(inv_rel=r_inv, edit_rel=r_ed)
    assert max(r_inv) < 2e-2 and max(r_ed) < 8e-2


def test_blend_case_vs_oracle(report):
    """Replace + self-attention blend + latent blend on 64x96 latents: no reference behaviour exists (its blender asserts square maps), so
    the fp32 oracle's restatement is the yardstick, with the mini blend case's bounds: inversion 2e-2 relative, final edit 8e-2 relative
    on the 99th percentile with < 2% outliers, latent-blend masks < 2% mismatched pixels."""
    case = ns.NONSQUARE_CASES["ns_replace_blend"]
    prod = nsr.run_product(case)
    orc = nsr.run_oracle(case)
    r_inv = rel(prod["inv_latents"], orc["inv_latents"])
    r_ed = robust_rel(prod["edit_latents"][-1], orc["edit_latents"][-1])
    outl = ((prod["edit_latents"][-1] - orc["edit_latents"][-1]).abs() > 0.05 * orc["edit_latents"][-1].abs().max()).float().mean().item()
    masks = prod["result"]["mask_list"]
    assert len(masks) == len(orc["ctrl"].mask_list) == case["steps"]
    assert masks[0].shape[-2:] == (case["h"], case["w"])
    mism = max((a.cpu().reshape(-1) != b.reshape(-1)).float().mean().item() for a, b in zip(masks, orc["ctrl"].mask_list))
    ones = [float(m.mean()) for m in masks]
    ctrl = prod["pipe"].last_edit_controller
    grids = sorted({k[1] for k in ctrl._mask_cache})
    report["ns_replace_blend"] = dict(inv_rel=r_inv, edit_rel=r_ed, outlier_frac=outl, mask_mismatch=mism, mask_ones=ones, self_grids=grids)
    assert 0.0 < max(ones) < 1.0  # the masks select part of the frame
    assert grids and all(rh * rw <= 32 ** 2 and rw * case["h"] == rh * case["w"] for rh, rw in grids)
    assert outl < 2e-2 and mism < 2e-2
    assert r_inv < 2e-2 and r_ed < 8e-2


# ------------------------------------------------------------------------------------------------------------------ bitwise
def _maps(store):
    return [(k, i, t.float().cpu().clone()) for d in store.attention_store_all_step for k, v in d.items() for i, t in enumerate(v)]


def test_graph_replay_equals_eager():
    case = ns.NONSQUARE_CASES["ns_replace_blend"]
    pipe = nsr.build_product(case["unet"], case["model_config"])
    eager = nsr.run_product(case, pipe=pipe)
    maps_eager = _maps(pipe.store_controller)
    nsr.run_product(case, pipe=pipe)                        # capture
    assert len(pipe._plans) == 2, list(pipe._plans)
    replayed = nsr.run_product(case, pipe=pipe)             # replay
    assert torch.equal(replayed["inv_latents"], eager["inv_latents"]) and torch.equal(replayed["edit_latents"], eager["edit_latents"])
    for (k, i, a), (k2, i2, b) in zip(maps_eager, _maps(pipe.store_controller)):
        assert (k, i) == (k2, i2) and torch.equal(a, b), (k, i)
    for a, b in zip(eager["result"]["mask_list"], replayed["result"]["mask_list"]):
        assert torch.equal(a.cpu(), b.cpu())
    assert pipe.last_edit_controller._latent_hw == (case["h"], case["w"])  # adopted from the captured controller


def test_batched_inversion_and_edit_equal_single_calls():
    """At 32x48: prepare_latents_ddim_inverted_batch over two clips == one inversion per clip, and p2preplace_edit_batch with two prompts
    == one p2preplace_edit per prompt, bit for bit (latents, stored maps, running sums)."""
    case = ns.NONSQUARE_CASES["ns_landscape_refine"]
    other = ns.NONSQUARE_CASES["ns_portrait_replace"]
    N = case["steps"]
    pipe = nsr.build_product(case["unet"], case["model_config"])
    pipe.graph_mode = "off"
    x0 = ns.case_inputs(case).to(dev)
    clips = [x0, -x0.flip(-1)]
    sources = [case["source"], "a red car driving down a curvy road in the countryside"]
    singles = []
    for x, src in zip(clips, sources):
        pipe.scheduler.set_timesteps(N)
        emb = pipe._encode_prompt(src, dev, 1, True, None)
        pipe.prepare_before_train_loop()
        store = controllers.AttentionStore()
        controllers.register_attention_control(pipe, store)
        store.LOW_RESOURCE = True
        inv = pipe.ddim_clean2noisy_loop(x, emb, store)
        store.LOW_RESOURCE = False
        controllers.register_attention_control(pipe, pipe.empty_controller)
        singles.append((inv, store))
    pipe.scheduler.set_timesteps(N)
    lats = pipe.prepare_latents_ddim_inverted_batch(sources, latents=clips)
    for k, ((inv, st), lat, bst) in enumerate(zip(singles, lats, pipe.store_controllers)):
        assert all(torch.equal(a, b) for a, b in zip(inv, lat)), k
        assert bst._latent_hw == st._latent_hw == (case["h"], case["w"])
        for (ka, ia, a), (kb, ib, b) in zip(_maps(st), _maps(bst)):
            assert (ka, ia) == (kb, ib) and torch.equal(a, b), (k, ka, ia)
    # batched edit of clip 0 with two prompts against the single edits
    pipe.store_controller = singles[0][1]
    xT = singles[0][0][-1]
    prompts = [(case["target"], case["p2p"]), ("a silver car driving down a curvy road in the countryside", other["p2p"])]
    save = tempfile.mkdtemp()
    single_runs = []
    for p, c in prompts:
        trace = []
        pipe(prompt=p, source_prompt=case["source"], edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5,
             output_type="latent", height=8 * case["h"], width=8 * case["w"], callback=lambda i, t, l: trace.append(l.detach().clone()),
             use_inversion_attention=True, save_self_attention=False, save_path=save, **c)
        single_runs.append((trace, pipe.last_edit_controller.attention_store))
    trace = []
    pipe.p2preplace_edit_batch([p for p, _ in prompts], [dict(c, use_inversion_attention=True, save_self_attention=False) for _, c in prompts],
                               case["source"], xT, N, 7.5, save_path=save, output_type="latent",
                               callback=lambda i, t, l: trace.append(l.detach().clone()))
    for k, (strace, sums) in enumerate(single_runs):
        for i, (a, b) in enumerate(zip(strace, trace)):
            assert torch.equal(a[0], b[k]), (k, i)
        mine = pipe.last_edit_controllers[k].attention_store
        for key in sums:
            for a, b in zip(sums[key], mine[key]):
                assert torch.equal(a, b), (k, key)


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_pil_output_and_heatmap_strips(report):
    """p2preplace_edit with output_type="pil" through a (small, random-init) VAE: 256x384 frames, and heat-map strips of the 16x24 level
    whose tiles are 256 tall and 384 wide.  The device heat maps agree with the host path to one grey level."""
    from fatezero_b200 import vae as fzvae
    case = ns.NONSQUARE_CASES["ns_landscape_refine"]
    pipe = nsr.build_product(case["unet"], case["model_config"])
    torch.manual_seed(0)
    pipe.vae = fzvae.AutoencoderKL(block_out_channels=(32, 64, 128, 128), layers_per_block=2, latent_channels=4, norm_num_groups=32).cuda()
    out = nsr.run_product(case, pipe=pipe, output_type="pil")
    frames = out["result"]["sdimage_output"].images
    assert len(frames) == 1 and len(frames[0]) == case["frames"]
    assert frames[0][0].size == (8 * case["w"], 8 * case["h"])  # PIL (width, height)
    strips = out["result"]["attention_output"]
    tok = synth.ToyTokenizer()
    n = len(tok.encode(case["target"]))
    assert len(strips) == case["frames"]
    assert strips[0].shape == (256 + int(256 * 0.2), n * 256 * 24 // 16, 3)
    ctrl = pipe.last_edit_controller
    dev_u8 = visualization.device_heatmaps(ctrl, 16, ["up", "down"], n)
    assert dev_u8 is not None and dev_u8.shape == (case["frames"], n, 16, 24)
    host = visualization.aggregate_attention([case["target"]], ctrl, 16, ["up", "down"], True, 0)  # [F, 16, 24, 77]
    want = torch.stack([(255 * host[..., i] / host[..., i].amax(dim=(1, 2), keepdim=True)).clamp(0, 255) for i in range(n)], 1)
    d = (dev_u8.cpu().float() - want.floor()).abs().max().item()
    report["heatmaps_16x24"] = dict(max_abs_lsb=d, tokens=n)
    assert d <= 1.0
    with pytest.raises(ValueError, match="resolution 32"):
        visualization.show_cross_attention(tok, case["target"], ctrl, 32, ["up", "down"])


# ------------------------------------------------------------------------------------------------------------------ frame sharding
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="frame sharding needs >= 2 GPUs")
def test_frame_sharded_nonsquare(report):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tools", "shard_check_nonsquare.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert line, r.stdout[-2000:] + r.stderr[-3000:]
    res = json.loads(line[-1])
    report["frame_shard_nonsquare_2gpu"] = res
    assert r.returncode == 0 and res["ok"], res
