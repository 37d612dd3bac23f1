"""Text-to-video sampling and the Tune-A-Video DDIM pipeline for the parity tests: the cases, the oracle's sampler restatement, the
VAE stand-in that encodes and the golden format.  TEST INFRASTRUCTURE (plain torch, travels with the tests).

The sampler restates pipelines/stable_diffusion.py:519-549 (= ddim_spatial_temporal.py:255-284): classifier-free guidance when
guidance_scale > 1, then diffusers-0.11.1 DDIMScheduler.step with eta:
    x0 = (x - sqrt(1 - a_t) e) / sqrt(a_t),  std = eta sqrt(_get_variance(t, t_prev)),
    x  = sqrt(a_prev) x0 + sqrt(1 - a_prev - std^2) e  (+ std z at eta > 0),
_get_variance = (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev), a_prev = alphas_cumprod[0] past the last step (set_alpha_to_one=False).
oracle/make_sample_golden.py records the unmodified reference on these cases; tests/test_sample_cpu.py pins this restatement to them.

Golden files are kept small, in the compact format of oracle/sd2.py: the initial latents in full (`init`, fp32), every step's latents as a
fixed strided sample (every LAT_STRIDE-th element of the flattened tensor, `step_sample`) plus float64 sums and sums of squares (`sums`), the
variance noise the reference's scheduler drew at each step in full (`noise`, eta > 0 only) and, for the DDIM pipeline, the inversion's
latents as samples and sums (`inv_sample`, `inv_sums`).  The UNet's attention kernels need latents of at least 32 x 32 (the 2x2 mid level of
16 x 16 latents is not a multiple of 8 pixels), so every case runs at 256 x 256 pixels."""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn.functional as F

from oracle import fz_oracle as fo

MODEL_CONFIG = dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=128)
LAT_STRIDE = 8
SRC = "a silver jeep driving down a curvy road in the countryside"

SAMPLE_CASES = {
    # (a) two prompts x two clips each, CFG with a negative prompt, deterministic DDIM
    "t2v_cfg_batch": dict(pipeline="t2v", unet="mini", prompt=[SRC, "watercolor painting of a red car"], negative_prompt=["blurry", "dark"],
                          num_images_per_prompt=2, guidance_scale=7.5, eta=0.0, frames=4, size=32, steps=5, seed=11),
    # (b) one prompt, no guidance (one UNet row per frame), full stochastic DDIM
    "t2v_eta1_nocfg": dict(pipeline="t2v", unet="mini", prompt=SRC, negative_prompt=None, num_images_per_prompt=1, guidance_scale=1.0,
                           eta=1.0, frames=2, size=32, steps=5, seed=12),
    # (c) Tune-A-Video + DDIM inversion: invert with the source prompt, denoise with the target under CFG
    "ddim_invert_edit": dict(pipeline="ddim", unet="mini", source=SRC, prompt="a Porsche car driving down a curvy road in the countryside",
                             negative_prompt=None, num_images_per_prompt=1, guidance_scale=7.5, eta=0.0, frames=4, size=32, steps=5, seed=13),
    # (d) SD-2 mini geometry (heads 1 / 2 / 4 / 4, 1024-wide text), eta = 0.5
    "t2v_sd2mini_eta05": dict(pipeline="t2v", unet="sd2mini", prompt=SRC, negative_prompt=None, num_images_per_prompt=1, guidance_scale=7.5,
                              eta=0.5, frames=2, size=32, steps=4, seed=14),
}


class EncodingVaeStub(torch.nn.Module):
    """synth.VaeStub with an encoder: 8x8 average pooling of the three image channels plus their mean as the fourth latent channel,
    divided by 0.18215 (the pipelines scale encoded latents by it).  latent_dist.sample(generator) is deterministic and draws nothing."""

    class _Cfg:
        block_out_channels = (128, 256, 512, 512)

    def __init__(self):
        super().__init__()
        self.config = self._Cfg()
        self.dummy = torch.nn.Parameter(torch.zeros(1), requires_grad=False)

    def encode(self, image):
        p = F.avg_pool2d(image.float(), 8)
        z = torch.cat([p, p.mean(1, keepdim=True)], dim=1) / 0.18215

        class _Dist:
            def sample(self, generator=None):
                return z.to(image.dtype)

        class _O:
            latent_dist = _Dist()
        return _O()

    def decode(self, latents):
        class _O:
            pass
        o = _O()
        o.sample = F.interpolate(latents[:, :3].float(), scale_factor=8.0, mode="nearest")
        return o


def case_image(case: dict) -> torch.Tensor:
    """The frames [F, 3, 8 size, 8 size] the DDIM case inverts (seeded)."""
    g = torch.Generator().manual_seed(case["seed"])
    s = case["size"] * 8
    base = torch.randn(case["frames"], 3, s // 16, s // 16, generator=g)
    return (0.5 * F.interpolate(base, size=(s, s), mode="bilinear", align_corners=False)).clamp(-1, 1)


def strided(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().cpu().reshape(-1)[::LAT_STRIDE].clone()


def sums(ts) -> torch.Tensor:
    return torch.tensor([[v.double().sum(), (v.double() ** 2).sum()] for v in ts], dtype=torch.float64)


def sigma(ac: torch.Tensor, t: int, t_prev: int, eta: float) -> float:
    a_t = ac[t]
    a_p = ac[t_prev] if t_prev >= 0 else ac[0]
    return float(eta * (((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)) ** 0.5)


def sample(unet: fo.OracleUNet, x_T: torch.Tensor, text: torch.Tensor, num_steps: int, guidance_scale: float, eta: float = 0.0,
           noise: Optional[List[torch.Tensor]] = None, teacher: Optional[List[torch.Tensor]] = None) -> List[torch.Tensor]:
    """The sampler (see the module docstring) on clips x_T [B, 4, F, h, w]; text = [uncond_1..B ; cond_1..B] when guidance_scale > 1, else
    [B, 77, D].  noise[i]: the step's variance noise (eta > 0).  teacher: step i > 0 starts from teacher[i - 1].  Returns the N latents."""
    ac = fo.alphas_cumprod()
    ts = fo.ddim_timesteps(num_steps)
    x = x_T.clone().float()
    trace = []
    for i, t in enumerate(ts):
        if teacher is not None and i > 0:
            x = teacher[i - 1].clone().float()
        if guidance_scale > 1.0:
            e_u, e_c = unet.forward(torch.cat([x, x]), t, text).chunk(2)
            e = e_u + guidance_scale * (e_c - e_u)
        else:
            e = unet.forward(x, t, text)
        t_prev = t - 1000 // num_steps
        a_t = ac[t]
        a_p = ac[t_prev] if t_prev >= 0 else ac[0]
        std = sigma(ac, t, t_prev, eta)
        x0 = (x - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
        x = a_p ** 0.5 * x0 + (1 - a_p - std ** 2) ** 0.5 * e
        if eta > 0:
            x = x + std * noise[i].to(x.device, torch.float32)
        trace.append(x.clone())
    return trace


def encode_text(tokenizer, text_encoder, prompts: List[str], negative: Optional[List[str]], cfg: bool, per_prompt: int = 1) -> torch.Tensor:
    """stable_diffusion.py:180-295 for a list of prompts: [uncond ; cond] rows, each repeated per_prompt times."""
    def enc(ps):
        ids = tokenizer(ps, padding="max_length", max_length=tokenizer.model_max_length, truncation=True).input_ids
        with torch.no_grad():
            return text_encoder(ids)[0].float().repeat_interleave(per_prompt, dim=0)
    cond = enc(prompts)
    if not cfg:
        return cond
    return torch.cat([enc(negative if negative is not None else [""] * len(prompts)), cond])
