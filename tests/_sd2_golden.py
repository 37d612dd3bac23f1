"""Reading the compact SD-2 goldens (oracle/sd2.py's format) in the parity tests."""
import os

import torch

from _helpers import GOLDEN_DIR, synth_weights
from fatezero_b200 import synth
from oracle import sd2


def load(name: str) -> dict:
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    assert os.path.exists(path), f"missing golden fixture {path} (python -m oracle.make_sd2_golden {name})"
    g = torch.load(path)
    if "teacher_inv" in g:  # the samples of the steps kept in full are not stored twice
        g["inv_sample"] = torch.cat([g["inv_sample"], samples(g["teacher_inv"], g["lat_stride"])])
        g["edit_sample"] = torch.cat([samples(g["teacher_edit"], g["lat_stride"]), g["edit_sample"]])
    return g


def build_oracle(case: dict):
    return sd2.OracleUNetSD2(synth_weights(case["unet"], case["model_config"]), synth.UNET_CONFIGS[case["unet"]], case["model_config"])


def samples(traj: torch.Tensor, stride: int) -> torch.Tensor:
    """[steps, ...] trajectory -> [steps, k] strided samples, as the golden keeps them."""
    return torch.stack([sd2.sample(v, stride) for v in traj])


def sq_sums(traj: torch.Tensor) -> torch.Tensor:
    return torch.tensor([float((v.double() ** 2).sum()) for v in traj], dtype=torch.float64)


def teacher(case: dict, g: dict, x0: torch.Tensor) -> dict:
    """The reference latents a teacher-forced run_product_case starts its steps from (the last edit latent is never an input)."""
    return dict(inv_latents=[x0] + list(g["teacher_inv"]), edit_latents=list(g["teacher_edit"]))


def mask_mismatch(got, gold) -> float:
    assert len(got) == len(gold)
    return max((a.cpu().reshape(-1) != b.reshape(-1).to(a.dtype)).float().mean().item() for a, b in zip(got, gold))
