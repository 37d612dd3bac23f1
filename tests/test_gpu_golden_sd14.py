"""Parity of the CUDA product at the REAL geometry (SD-1.4 UNet: head dims 40/80/160, C = 320/640/1280, 64x64 latents) against golden
vectors produced by the UNMODIFIED reference in the build container (oracle/make_golden.py, cases `sd14_config1` = BASELINE config #1 and
`sd14_replace_blend` = config #3 semantics).  The CPU oracle is NOT run here (35 min at this size): the goldens are the checker.

Three views per case, each with its own bound (fp16 storage / fp32 accumulation vs an fp32 reference):
  * teacher-forced: every CUDA forward starts from the reference's latent of that step, so the error of the post-step latent is ONE
    forward's kernel error (times the DDIM coefficient), not its amplification by 2N steps of the sampler.  This is the kernel-parity
    gate and carries the tight absolute bound.
  * free-running: the product's own trajectory (what a user gets) — inversion latents and every edit latent, reported per step.
  * stored maps: slices of the first and last inversion step's cache slabs and the square sum of every stored map of every step.
The measured values are printed and recorded by the `report` fixture (tests/conftest.py); the bounds and the values measured on
an H100 SXM (80 GB, 700 W power limit) are listed next to BOUNDS."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from _helpers import GOLDEN_DIR, build_product, run_product_case  # noqa: E402
from oracle.cases import BIG_CASES, CASES  # noqa: E402

# measured on an H100 SXM 80 GB at a 700 W power limit (`report` fixture); the asserted bounds leave 1.5-2.3x headroom over them
BOUNDS = {
    # measured (teacher-forced inv 1.9e-3 / edit 2.6e-2, free inv 5.7e-3 / edit 2.74e-1 on |x|max 15.8, slices 7.3e-4, square sums 1.0e-4)
    "sd14_config1": dict(tf_inv=4.4e-3, tf_edit=5e-2, free_inv=1.2e-2, free_edit=5.5e-1, map_abs=1.5e-3, sq_rel=1.8e-4),
    # measured (teacher-forced inv 3.2e-3 / edit q99 1.29e-2, free inv 4.5e-3 / edit q99 2.3e-2 on |x|max 5.2, slices 6.1e-4, square sums 1.0e-4)
    "sd14_replace_blend": dict(tf_inv=5.5e-3, tf_edit=2.7e-2, free_inv=9.2e-3, free_edit=4.7e-2, map_abs=1e-3, sq_rel=1.5e-4),
}


def _golden(name):
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    if not os.path.exists(path):
        pytest.skip(f"{path} not generated yet (python -m oracle.make_golden {name})")
    return torch.load(path)


def _per_step(a, b):
    d = (a.float().cpu() - b.float().cpu()).abs()
    return d.flatten(1).amax(1).tolist(), torch.quantile(d.flatten(1)[:, ::7], 0.99, dim=1).tolist()


def _check_maps(store, g, N, bounds, report, tag):
    worst = 0.0
    for k, v in g["maps"].items():
        name, _, sl = k.partition("@")
        step, key, pos = name.split("/")
        t = store.attention_store_all_step[int(step)][key][int(pos)]
        F = t.shape[0]
        if sl == "":
            mine = t[F // 2]
        elif sl == "f0h2":
            mine = t[0, 2]
        else:
            mine = t[min(1, F - 1), 5, :256]
        worst = max(worst, (mine.float().cpu() - v.float()).abs().max().item())
    sq_worst = 0.0
    for k, s in g["map_sqsums"].items():
        step, key, pos = k.split("/")
        t = store.attention_store_all_step[int(step)][key][int(pos)]
        mine = float((t.double() ** 2).sum())
        sq_worst = max(sq_worst, abs(mine - s) / abs(s))
    report[f"{tag}_maps"] = dict(slice_max_abs=worst, sqsum_max_rel=sq_worst, n_slices=len(g["maps"]), n_sqsums=len(g["map_sqsums"]))
    assert worst < bounds["map_abs"], f"stored map slices deviate by {worst:.3g}"
    assert sq_worst < bounds["sq_rel"], f"stored map square sums deviate by {sq_worst:.3g} (relative)"


@pytest.mark.parametrize("name", BIG_CASES)
def test_teacher_forced(name, report):
    """One forward of kernel error per compared latent: max|x_cuda - x_ref| after each inversion step and each CFG edit step."""
    g, case, b = _golden(name), CASES[name], BOUNDS[name]
    blend = bool(case["p2p"].get("blend_words"))
    pipe = build_product(case["unet"], case["model_config"])
    prod = run_product_case(case, pipe=pipe, teacher=g)
    inv_max, inv_q = _per_step(prod["inv_latents"][1:], g["inv_latents"][1:])
    ed_max, ed_q = _per_step(prod["edit_latents"], g["edit_latents"])
    scale = g["edit_latents"].abs().max().item()
    report[f"{name}_teacher_forced"] = dict(inv_max_abs=inv_max, inv_q99=inv_q, edit_max_abs=ed_max, edit_q99=ed_q, latent_abs_max=scale)
    print(f"\n{name} teacher-forced: inversion max|d| per step {['%.2e' % v for v in inv_max]}\n  edit max|d| per step {['%.2e' % v for v in ed_max]}"
          f"\n  edit q99 per step {['%.2e' % v for v in ed_q]} (|x|max {scale:.2f})")
    _check_maps(pipe.store_controller, g, case["steps"], b, report, f"{name}_tf")
    assert max(inv_max) < b["tf_inv"]
    # a thresholded blend mask can flip single pixels between an fp16 and an fp32 run: blend cases are judged on the 99th percentile
    assert max(ed_q if blend else ed_max) < b["tf_edit"]
    if "mask_list" in g and prod["result"]["mask_list"]:
        mism = max((a.cpu().reshape(-1) != m.reshape(-1)).float().mean().item() for a, m in zip(prod["result"]["mask_list"], g["mask_list"]))
        report[f"{name}_tf_mask_mismatch"] = mism
        assert mism < 1e-2


@pytest.mark.parametrize("name", BIG_CASES)
def test_free_running(name, report):
    """The product's own trajectory against the reference's (2N forwards of error propagation through the CFG x7.5 sampler)."""
    g, case, b = _golden(name), CASES[name], BOUNDS[name]
    blend = bool(case["p2p"].get("blend_words"))
    pipe = build_product(case["unet"], case["model_config"])
    prod = run_product_case(case, pipe=pipe)
    inv_max, inv_q = _per_step(prod["inv_latents"][1:], g["inv_latents"][1:])
    ed_max, ed_q = _per_step(prod["edit_latents"], g["edit_latents"])
    report[f"{name}_free"] = dict(inv_max_abs=inv_max, edit_max_abs=ed_max, edit_q99=ed_q, latent_abs_max=g["edit_latents"].abs().max().item())
    print(f"\n{name} free-running: inversion max|d| per step {['%.2e' % v for v in inv_max]}\n  edit max|d| per step {['%.2e' % v for v in ed_max]}")
    assert max(inv_max) < b["free_inv"]
    assert (ed_q if blend else ed_max)[-1] < b["free_edit"]


def test_single_forward_vs_reference(report):
    """One CFG-batch forward without a controller against the reference's epsilon (2 frames of the Replace/blend case's inputs)."""
    from fatezero_b200 import synth
    name = "sd14_replace_blend"
    g, case = _golden(name), CASES[name]
    pipe = build_product(case["unet"], case["model_config"])
    x0 = synth.synth_latents(case["frames"], case["size"], case["size"]) * 0.5
    x2 = torch.cat([x0, 0.7 * x0])[:, :, :2]
    emb = torch.randn(2, 77, 768, generator=torch.Generator().manual_seed(2))
    got = pipe.unet(x2.cuda(), 481, emb.cuda()).sample.float().cpu()
    d = (got - g["fwd_eps"]).abs().max().item()
    report["sd14_fwd_vs_reference"] = dict(max_abs=d, eps_abs_max=g["fwd_eps"].abs().max().item(), eps_std=g["fwd_eps"].std().item())
    assert d < 1e-2  # measured 4.9e-3 on max|eps| 3.0
