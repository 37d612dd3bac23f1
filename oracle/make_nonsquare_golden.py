"""Generate the non-square goldens (tests/golden/ns_*.pt, compact format of oracle/sd2.py) by running the UNMODIFIED reference
(/root/reference) through the tests-only shim.  Build container only (the reference does not travel).
The reference's heat-map call after the edit (p2p_ddim_spatial_temporal.py:211-213) concatenates the maps of exactly 16**2 pixels and
fails on a non-square clip, which has none: it is replaced at run time by a no-op (no reference source is edited).
Usage: python -m oracle.make_nonsquare_golden [case ...]"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fatezero_b200 import synth  # noqa: E402
from oracle import nonsquare as ns  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
from oracle import sd2  # noqa: E402


def run_case(name: str):
    c = ns.NONSQUARE_CASES[name]
    assert c.get("ref", True) and not c["p2p"].get("blend_words"), f"{name}: the reference asserts square maps in its blender"
    pipe = rh.build_reference_pipeline(synth.UNET_CONFIGS[c["unet"]], c["model_config"])
    from video_diffusion.prompt_attention import attention_util
    attention_util.show_cross_attention = lambda *a, **k: None
    x0 = ns.case_inputs(c)
    t = time.time()
    out = rh.run_reference(pipe, x0, c["source"], c["target"], c["steps"], c["p2p"])
    inv, ed = out["inv_latents"], out["edit_latents"]
    gold = dict(case=name, seconds=time.time() - t, torch=str(torch.__version__), lat_stride=sd2.LAT_STRIDE, eps_stride=sd2.EPS_STRIDE,
                inv_sample=torch.stack([sd2.sample(v, sd2.LAT_STRIDE) for v in inv]),
                edit_sample=torch.stack([sd2.sample(v, sd2.LAT_STRIDE) for v in ed]),
                inv_sums=torch.tensor([[v.double().sum(), (v.double() ** 2).sum()] for v in inv], dtype=torch.float64),
                edit_sums=torch.tensor([[v.double().sum(), (v.double() ** 2).sum()] for v in ed], dtype=torch.float64),
                edit_abs_max=float(ed.abs().max()),
                map_shapes={k: list(v.shape) for k, v in out["maps"].items()})
    # what a teacher-forced run starts its steps from, kept in full as for oracle/sd2.py's big case (the samples of those steps are then
    # taken from these tensors when the golden is read: tests/_sd2_golden.py)
    gold["teacher_inv"] = inv[1:].clone()
    gold["teacher_edit"] = ed[:-1].clone()
    gold["inv_sample"] = gold["inv_sample"][:1].clone()
    gold["edit_sample"] = gold["edit_sample"][-1:].clone()
    sums, sq, keep = {}, {}, {}
    for k, v in out["maps"].items():
        sums[k] = float(v.double().sum())
        sq[k] = float((v.double() ** 2).sum())
        step, key, pos = k.split("/")
        if step == "0" and pos == "0" and len(keep) < sd2.MAP_SLICES:
            keep[k] = sd2.map_slice(v).half().clone()
    gold.update(map_sums=sums, map_sqsums=sq, maps=keep)
    x2, tt, emb = ns.fwd_inputs(c, x0)
    gold["fwd_eps_sample"] = sd2.sample(rh.reference_unet_forward(pipe, x2, torch.tensor(tt), emb), sd2.EPS_STRIDE)
    path = os.path.join(ROOT, "tests", "golden", f"{name}.pt")
    torch.save(gold, path)
    print(name, "->", path, f"{os.path.getsize(path) / 1e3:.0f} kB", f"{gold['seconds']:.1f}s", len(sums), "maps")


if __name__ == "__main__":
    for n in (sys.argv[1:] or ns.NONSQUARE_REF_CASES):
        run_case(n)
