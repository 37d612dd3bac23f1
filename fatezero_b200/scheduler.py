"""DDIM scheduler with the diffusers-0.11.1 call surface the reference pipeline touches
(pipelines/p2p_ddim_spatial_temporal.py:154-156,367,407; pipelines/stable_diffusion.py:56-81,321-336).
Scalar tables live on the host; the tensor arithmetic of a step runs in fz_ddim_invert_step / fz_cfg_ddim_step."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import torch


class _Config(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


class DDIMScheduler:
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "scaled_linear", clip_sample: bool = False, set_alpha_to_one: bool = False,
                 steps_offset: int = 1, prediction_type: str = "epsilon", **unused):
        self._internal_dict = _Config(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                      beta_schedule=beta_schedule, clip_sample=clip_sample, set_alpha_to_one=set_alpha_to_one,
                                      steps_offset=steps_offset, prediction_type=prediction_type)
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        elif beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        else:
            raise NotImplementedError(beta_schedule)
        self.betas = betas
        self.alphas = 1.0 - betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    @property
    def config(self):
        return self._internal_dict

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.config.num_train_timesteps // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts) + self.config.steps_offset  # kept on the host: they only index tables

    def scale_model_input(self, sample, timestep=None):
        return sample

    def alpha_pair(self, timestep: int):
        """(alpha_bar_t, alpha_bar_prev) of a denoising step."""
        t = int(timestep)
        prev = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[t])
        a_p = float(self.alphas_cumprod[prev]) if prev >= 0 else float(self.final_alpha_cumprod)
        return a_t, a_p

    def sigma(self, timestep: int, eta: float) -> float:
        """eta * sqrt(_get_variance) of diffusers-0.11.1 DDIMScheduler: the standard deviation of the noise a step adds."""
        a_t, a_p = self.alpha_pair(timestep)
        return float(eta) * (((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)) ** 0.5

    def step(self, model_output, timestep, sample, eta: float = 0.0, use_clipped_model_output=False, generator=None,
             variance_noise=None, return_dict: bool = True):
        """Torch-tensor API for callers outside the fused loops, with diffusers-0.11.1 semantics: at eta > 0 the step adds
        sigma * variance_noise, drawn as torch.randn(model_output.shape, generator=generator) on model_output's device and dtype when not
        given (giving both is a ValueError), and the direction term becomes sqrt(1 - a_prev - sigma^2) * model_output."""
        a_t, a_p = self.alpha_pair(timestep)
        x0 = (sample - (1 - a_t) ** 0.5 * model_output) / a_t ** 0.5
        if self.config.clip_sample:
            x0 = x0.clamp(-1, 1)
        std = self.sigma(timestep, eta)
        prev = a_p ** 0.5 * x0 + (1 - a_p - std ** 2) ** 0.5 * model_output
        if eta > 0:
            if variance_noise is not None and generator is not None:
                raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or `variance_noise` "
                                 "stays `None`.")
            if variance_noise is None:
                variance_noise = torch.randn(model_output.shape, generator=generator, device=model_output.device, dtype=model_output.dtype)
            prev = prev + std * variance_noise
        return SimpleNamespace(prev_sample=prev, pred_original_sample=x0)
