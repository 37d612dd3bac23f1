"""Generate the SD-2 goldens (tests/golden/sd2*.pt, compact format of oracle/sd2.py) and the reference's SD-2-base state-dict shapes by
running the UNMODIFIED reference (/root/reference) through the tests-only shim.  Build container only (the reference does not travel).
Usage: python -m oracle.make_sd2_golden [sd2_shapes | case ...]"""
import gzip
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fatezero_b200 import synth  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
from oracle import sd2  # noqa: E402


def run_case(name: str):
    c = sd2.SD2_CASES[name]
    cfg = synth.UNET_CONFIGS[c["unet"]]
    pipe = rh.build_reference_pipeline(cfg, c["model_config"])
    x0 = synth.synth_latents(c["frames"], c["size"], c["size"]) * 0.5
    save_path = tempfile.mkdtemp() if c["p2p"].get("blend_words") else None
    t = time.time()
    out = rh.run_reference(pipe, x0, c["source"], c["target"], c["steps"], c["p2p"], save_path=save_path)
    inv, ed = out["inv_latents"], out["edit_latents"]
    gold = dict(case=name, seconds=time.time() - t, torch=str(torch.__version__), lat_stride=sd2.LAT_STRIDE, eps_stride=sd2.EPS_STRIDE,
                inv_sample=torch.stack([sd2.sample(v, sd2.LAT_STRIDE) for v in inv]),
                edit_sample=torch.stack([sd2.sample(v, sd2.LAT_STRIDE) for v in ed]),
                inv_sums=torch.tensor([[v.double().sum(), (v.double() ** 2).sum()] for v in inv], dtype=torch.float64),
                edit_sums=torch.tensor([[v.double().sum(), (v.double() ** 2).sum()] for v in ed], dtype=torch.float64),
                edit_abs_max=float(ed.abs().max()))
    if c.get("big"):
        # what a teacher-forced run starts its steps from: inversion latents 1..N (0 is the seeded input), edit latents 0..N-2; their
        # samples are taken from these tensors when the golden is read
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
    if out["mask_list"] is not None:
        gold["mask_list"] = [m.to(torch.uint8).clone() for m in out["mask_list"]]
    x2, tt, emb = sd2.fwd_inputs(c, x0)
    gold["fwd_eps_sample"] = sd2.sample(rh.reference_unet_forward(pipe, x2, torch.tensor(tt), emb), sd2.EPS_STRIDE)
    path = os.path.join(ROOT, "tests", "golden", f"{name}.pt")
    torch.save(gold, path)
    print(name, "->", path, f"{os.path.getsize(path) / 1e3:.0f} kB", f"{gold['seconds']:.1f}s",
          "mask means", [float(m.float().mean()) for m in (out["mask_list"] or [])])


def record_sd2_shapes():
    """tests/golden/ref_unet_sd2_state_dict_shapes.json.gz: names and shapes of the reference UNet's state_dict at SD-2-base geometry
    (per-block heads, linear projections, 1024-wide text) with lora: 160."""
    rh._prepare_imports()
    from video_diffusion.models.unet_3d_condition import UNetPseudo3DConditionModel
    mc = dict(lora=160)
    unet = UNetPseudo3DConditionModel(**synth.SD2_UNET_CONFIG, **mc)
    rec = dict(unet_config={k: list(v) if isinstance(v, tuple) else v for k, v in synth.SD2_UNET_CONFIG.items()}, model_config=mc,
               shapes={k: list(v.shape) for k, v in unet.state_dict().items()})
    path = os.path.join(ROOT, "tests", "golden", "ref_unet_sd2_state_dict_shapes.json.gz")
    with gzip.open(path, "wt") as f:
        json.dump(rec, f)
    print("sd2 shapes ->", path, len(rec["shapes"]), "tensors")


if __name__ == "__main__":
    for n in (sys.argv[1:] or ["sd2_shapes", *sd2.SD2_CASES]):
        if n == "sd2_shapes":
            record_sd2_shapes()
        else:
            run_case(n)
