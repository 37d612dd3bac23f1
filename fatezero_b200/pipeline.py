"""P2pDDIMSpatioTemporalPipeline — drop-in for video_diffusion/pipelines/p2p_ddim_spatial_temporal.py (+ the parts of
pipelines/stable_diffusion.py it inherits), same constructor, methods, kwargs and return types, so test_fatezero.py and
P2pSampleLogger (pipelines/p2p_validation_loop.py) drive it unchanged.

The two hot loops run on the GPU through libfatezero_b200.so:
  ddim_clean2noisy_loop  : N x { UNet (B=1, STORE fused in attention) ; fz_ddim_invert_step }
  sd_ddim_pipeline loop  : N x { UNet (B=2, INJECT/BLEND fused)       ; fz_cfg_ddim_step (+ latent blend) }
  _sample_loop           : N x { UNet (whole clips, un-hooked)       ; fz_ddim_sample_step (CFG or not, eta >= 0) }
The last one serves text-to-video sampling (SpatioTemporalStableDiffusionPipeline.__call__, pipelines/stable_diffusion.py:403-564) and the
Tune-A-Video + DDIM inversion baseline (DDIMSpatioTemporalStableDiffusionPipeline, pipelines/ddim_spatial_temporal.py).
Latents stay fp32 in HBM for the whole run; text encoder / VAE / tokenizer are whatever objects the caller passes (out of the
accelerated scope, SURVEY.md §8(f)).
"""
from __future__ import annotations

import inspect
import os
import sys
from typing import Callable, List, Optional, Union

import numpy as np
import torch

from . import controllers as attention_util
from . import ops
from .scheduler import DDIMScheduler


class StableDiffusionPipelineOutput(dict):
    def __init__(self, images, nsfw_content_detected=None):
        super().__init__(images=images, nsfw_content_detected=nsfw_content_detected)
        self.images = images
        self.nsfw_content_detected = nsfw_content_detected


class _NullBar:
    def __init__(self, total=None):
        self.total = total

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def update(self, n=1):
        pass


class SpatioTemporalStableDiffusionPipeline:
    """pipelines/stable_diffusion.py:33-336 (the members the FateZero flow uses)."""
    _optional_components: List[str] = []

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler):
        cfg = getattr(scheduler, "config", None)
        # scheduler-config fix-ups of stable_diffusion.py:56-81
        if cfg is not None and getattr(cfg, "steps_offset", 1) != 1:
            new = dict(cfg)
            new["steps_offset"] = 1
            scheduler._internal_dict = type(cfg)(new)
        if cfg is not None and getattr(cfg, "clip_sample", False) is True:
            new = dict(scheduler.config)
            new["clip_sample"] = False
            scheduler._internal_dict = type(scheduler.config)(new)
        self.vae, self.text_encoder, self.tokenizer, self.unet, self.scheduler = vae, text_encoder, tokenizer, unet, scheduler
        self._config = {k: (type(v).__module__, type(v).__name__) for k, v in
                        dict(vae=vae, text_encoder=text_encoder, tokenizer=tokenizer, unet=unet, scheduler=scheduler).items()}
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self._progress_bar_config = {}
        # CUDA-graph execution of the DDIM loops (graphs.py): "auto" = eager the first time a configuration is seen, captured and
        # replayed from its second occurrence on; "off" = always eager
        self.graph_mode = os.environ.get("FZ_GRAPHS", "auto")
        self._plans = {}
        self._seen = set()

    def release_graphs(self):
        """Drop every captured plan (and the HBM pools that hold their map caches)."""
        self._plans.clear()
        self._seen.clear()

    # ---- DiffusionPipeline surface ------------------------------------------------------------------------------
    @property
    def config(self):
        return self._config

    @property
    def device(self):
        for m in (self.unet, self.text_encoder, self.vae):
            if isinstance(m, torch.nn.Module):
                try:
                    return next(m.parameters()).device
                except StopIteration:
                    continue
        return torch.device("cpu")

    @property
    def _execution_device(self):
        return self.device

    def to(self, device):
        for m in (self.unet, self.text_encoder, self.vae):
            if isinstance(m, torch.nn.Module):
                m.to(device)
        return self

    def progress_bar(self, iterable=None, total=None):
        return _NullBar(total)

    def set_progress_bar_config(self, **kwargs):
        self._progress_bar_config = kwargs

    def enable_xformers_memory_efficient_attention(self, *a, **k):
        return None  # the fused sm_90a attention kernel is always on

    def disable_xformers_memory_efficient_attention(self, *a, **k):
        return None

    def enable_vae_slicing(self):
        if hasattr(self.vae, "enable_slicing"):
            self.vae.enable_slicing()

    def disable_vae_slicing(self):
        if hasattr(self.vae, "disable_slicing"):
            self.vae.disable_slicing()

    @staticmethod
    def numpy_to_pil(images):
        """stable_diffusion.py:566-576: [b, f, h, w, c] -> list (per clip) of lists of PIL frames."""
        from PIL import Image

        def frames(arr):
            if arr.ndim == 3:
                arr = arr[None, ...]
            arr = (arr * 255).round().astype("uint8")
            return [Image.fromarray(a) for a in arr]
        if images.ndim == 5:
            return [frames(seq) for seq in images]
        return [frames(images)]

    @staticmethod
    def _get_signature_keys(obj):
        params = inspect.signature(obj.__init__).parameters
        required = {k for k, v in params.items() if v.default is inspect._empty} - {"self"}
        optional = {k for k, v in params.items() if v.default is not inspect._empty}
        return required, optional

    def prepare_before_train_loop(self, params_to_optimize=None):
        for m in (self.vae, self.unet, self.text_encoder):
            if isinstance(m, torch.nn.Module):
                m.requires_grad_(False)
                m.eval()
        if params_to_optimize is not None:
            params_to_optimize.requires_grad = True

    def _text_forward(self, ids, mask):
        """The text encoder call of stable_diffusion.py:230,279.  A transformers CLIPTextModel living on the GPU is executed by
        clip.ClipTextEngine (sm_90a kernels, built once per module); any other module — or a padding mask — is simply called."""
        te = self.text_encoder
        if (mask is None and os.environ.get("FZ_CLIP", "1") != "0" and type(te).__name__ == "CLIPTextModel" and isinstance(te, torch.nn.Module)
                and next(te.parameters()).is_cuda):
            eng = getattr(self, "_clip_engine", None)
            if eng is None or eng[0] is not te:
                from .clip import ClipTextEngine
                try:
                    eng = (te, ClipTextEngine(te))
                except NotImplementedError:
                    eng = (te, None)
                self._clip_engine = eng
            if eng[1] is not None:
                return eng[1](ids)[0]
        return te(ids, attention_mask=mask)[0]

    def _encode_prompt(self, prompt, device, num_images_per_prompt, do_classifier_free_guidance, negative_prompt):
        """stable_diffusion.py:180-295: [uncond ; cond] text embeddings of shape [2*b, 77, D]."""
        batch_size = len(prompt) if isinstance(prompt, list) else 1
        tok = self.tokenizer
        text_inputs = tok(prompt, padding="max_length", max_length=tok.model_max_length, truncation=True, return_tensors="pt")
        ids = text_inputs.input_ids
        use_mask = bool(getattr(getattr(self.text_encoder, "config", None), "use_attention_mask", False))
        mask = text_inputs.attention_mask.to(device) if use_mask else None
        emb = self._text_forward(ids.to(device), mask)
        bs, seq, _ = emb.shape
        emb = emb.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq, -1)
        if do_classifier_free_guidance:
            if negative_prompt is None:
                uncond_tokens = [""] * batch_size
            elif type(prompt) is not type(negative_prompt):
                raise TypeError(f"`negative_prompt` should be the same type to `prompt`, but got {type(negative_prompt)} != {type(prompt)}.")
            elif isinstance(negative_prompt, str):
                uncond_tokens = [negative_prompt]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but `prompt`: {prompt} has "
                                 f"batch size {batch_size}. Please make sure that passed `negative_prompt` matches the batch size of `prompt`.")
            else:
                uncond_tokens = negative_prompt
            un = tok(uncond_tokens, padding="max_length", max_length=ids.shape[-1], truncation=True, return_tensors="pt")
            umask = un.attention_mask.to(device) if use_mask else None
            uemb = self._text_forward(un.input_ids.to(device), umask)
            uemb = uemb.repeat(1, num_images_per_prompt, 1).view(batch_size * num_images_per_prompt, uemb.shape[1], -1)
            emb = torch.cat([uemb, emb])
        return emb

    def _vae_engine(self):
        """The sm_90a VAE executor for `self.vae` (fatezero_b200.vae): our AutoencoderKL container or a foreign AutoencoderKL-shaped
        module on the GPU; None for anything else (stubs, CPU modules) — those are simply called."""
        if os.environ.get("FZ_VAE", "1") == "0":
            return None
        cached = getattr(self, "_vae_cache", None)
        if cached is None or cached[0] is not self.vae:
            from . import vae as vae_mod
            cached = (self.vae, vae_mod.engine_for(self.vae))
            self._vae_cache = cached
        return cached[1]

    def _vae_encode_sample(self, image, generator):
        """p2p_ddim_spatial_temporal.py:88-96: vae.encode(image).latent_dist.sample(generator)."""
        eng = self._vae_engine()
        if eng is None:
            return self.vae.encode(image).latent_dist.sample(generator)
        from .vae import DiagonalGaussianDistribution
        return DiagonalGaussianDistribution(eng.encode_moments(image).to(image.dtype)).sample(generator)

    def decode_latents(self, latents):
        """stable_diffusion.py:297-319 (VAE decode in chunks of 16 frames)."""
        is_video = latents.dim() == 5
        b = latents.shape[0]
        latents = 1 / 0.18215 * latents
        if is_video:
            latents = latents.permute(0, 2, 1, 3, 4).reshape(-1, *latents.shape[1:2], *latents.shape[3:])
        vdt = next(self.vae.parameters()).dtype if isinstance(self.vae, torch.nn.Module) else latents.dtype
        eng = self._vae_engine()
        if eng is not None:
            image = torch.cat([eng.decode(chunk) for chunk in torch.split(latents, 16, dim=0)], dim=0)
        else:
            image = torch.cat([self.vae.decode(chunk.to(vdt)).sample for chunk in torch.split(latents, 16, dim=0)], dim=0)
        image = (image / 2 + 0.5).clamp(0, 1).cpu().float().numpy()
        if is_video:
            image = image.reshape(b, -1, *image.shape[1:]).transpose(0, 1, 3, 4, 2)
        else:
            image = image.transpose(0, 2, 3, 1)
        return image

    @torch.no_grad()
    def decode_latents_u8(self, latents):
        """decode_latents + numpy_to_pil without leaving the device: uint8 frames [b, f, H, W, 3] for video latents [b, 4, f, h, w]
        ([N, H, W, 3] for image latents), bitwise the bytes of the PIL frames.  Needs the sm_90a VAE engine (fatezero_b200.vae)."""
        eng = self._vae_engine()
        if eng is None:
            raise RuntimeError("decode_latents_u8 runs on the sm_90a VAE engine: the pipeline's vae is not a fatezero_b200.vae.AutoencoderKL "
                               "nor an AutoencoderKL-shaped module on a CUDA device")
        is_video = latents.dim() == 5
        b = latents.shape[0]
        latents = 1 / 0.18215 * latents
        if is_video:
            latents = latents.permute(0, 2, 1, 3, 4).reshape(-1, *latents.shape[1:2], *latents.shape[3:])
        frames = torch.cat([ops.frames_to_u8(eng.decode(chunk)) for chunk in torch.split(latents, 16, dim=0)], dim=0)
        return frames.reshape(b, -1, *frames.shape[1:]) if is_video else frames

    def prepare_extra_step_kwargs(self, generator, eta):
        keys = set(inspect.signature(self.scheduler.step).parameters.keys())
        out = {}
        if "eta" in keys:
            out["eta"] = eta
        if "generator" in keys:
            out["generator"] = generator
        return out


    def check_inputs(self, prompt, height, width, callback_steps, strength=None):
        if not isinstance(prompt, str) and not isinstance(prompt, list):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if strength is not None and (strength <= 0 or strength > 1):
            raise ValueError(f"The value of strength should in (0.0, 1.0] but is {strength}")
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if (callback_steps is None) or (callback_steps is not None and (not isinstance(callback_steps, int) or callback_steps <= 0)):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type {type(callback_steps)}.")

    @staticmethod
    def check_frame_size(height: int, width: int, where: str):
        """A non-square clip must be a multiple of 64 pixels on both sides, so that the UNet's three stride-2 downsamples are exact and
        every level holds (h >> k) x (w >> k) latents; square clips keep the multiple-of-8 rule of check_inputs."""
        if height != width and (height % 64 or width % 64):
            raise ValueError(f"{where}: a non-square clip needs height and width that are multiples of 64, got {height} x {width}")

    def _engine_is_sharded(self) -> bool:
        engine = getattr(self.unet, "_engine", None)  # not built here: nothing may touch the GPU before the checks pass
        return getattr(engine, "shard", None) is not None

    # ---- scheduler tables (work with diffusers' DDIMScheduler or fatezero_b200.scheduler.DDIMScheduler) -------------
    def _alpha(self, t: int) -> float:
        return float(self.scheduler.alphas_cumprod[int(t)]) if int(t) >= 0 else float(self.scheduler.final_alpha_cumprod)

    # ---- DDIM inversion (p2p_ddim_spatial_temporal.py:68-161, ddim_spatial_temporal.py:45-119) -------------------------
    def _clean_latents_bcfhw(self, image, batch_size, generator):
        """VAE-encode the frames `image` [(b f), 3, H, W] and split them into `batch_size` clips [b, 4, f, h, w] (duplicating the clip when
        fewer images than clips are given)."""
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch size of "
                             f"{batch_size}. Make sure the batch size matches the length of the generators.")
        if isinstance(generator, list):
            init_latents = torch.cat([self._vae_encode_sample(image[i:i + 1], generator[i]) for i in range(batch_size)], dim=0)
        else:
            init_latents = self._vae_encode_sample(image, generator)
        init_latents = 0.18215 * init_latents
        if batch_size > init_latents.shape[0] and batch_size % init_latents.shape[0] != 0:
            raise ValueError(f"Cannot duplicate `image` of batch size {init_latents.shape[0]} to {batch_size} text prompts.")
        if batch_size > init_latents.shape[0]:
            init_latents = torch.cat([init_latents] * (batch_size // init_latents.shape[0]), dim=0)
        bf, c, h, w = init_latents.shape
        return init_latents.reshape(batch_size, bf // batch_size, c, h, w).permute(0, 2, 1, 3, 4)

    @torch.no_grad()
    def ddim_clean2noisy_loop(self, latent, text_embeddings, controller=None, teacher_latents=None):
        """p2p_ddim_spatial_temporal.py:131-148.  Returns N+1 latents (dtype of the input), [0] clean, [-1] x_T.
        teacher_latents (parity tests only): N+1 reference latents; step i then starts from teacher_latents[i] instead of this loop's
        own x_i (and the controller stores teacher_latents[i+1]), which isolates the per-forward kernel error from its amplification
        by the sampler."""
        weight_dtype = latent.dtype
        dev = self.unet.device
        ts = [int(t) for t in self.scheduler.timesteps]
        n = len(ts)
        step = self.scheduler.config.num_train_timesteps // self.scheduler.num_inference_steps
        with torch.cuda.device(dev):
            cond = text_embeddings.chunk(2)[1].to(dev).contiguous()

            def inv_step(i, x, cond_, ctrl, outputs):
                t = ts[n - 1 - i]
                eps = self.unet(x, t, encoder_hidden_states=cond_)["sample"]
                ops.ddim_invert_step(x, eps.contiguous(), self._alpha(min(t - step, 999)), self._alpha(t))
                if ctrl is not None:
                    ctrl.step_callback(x if teacher_latents is None else teacher_latents[i + 1].to(dev, torch.float32))
                outputs.append(x.to(dtype=weight_dtype).clone())

            # ---- CUDA-graph path (graphs.py): same launch sequence, captured once per configuration, no Python in the step ----
            sig = None
            if (self.graph_mode != "off" and teacher_latents is None
                    and isinstance(controller, (attention_util.AttentionStore, attention_util.AttentionStoreBatch))
                    and getattr(self.unet, "_controller", None) is controller and controller.is_pristine()):
                sig = controller.graph_signature()
            key = None if sig is None else ("inv", tuple(latent.shape), str(weight_dtype), tuple(ts), tuple(cond.shape), sig,
                                            id(self.unet.engine()), self.unet.engine().shard_signature())
            if key is not None and (key in self._plans or key in self._seen):
                plan = self._plans.get(key)
                if plan is None:
                    from .graphs import LoopPlan
                    plan = LoopPlan(dev)
                    plan.x = torch.empty(latent.shape, dtype=torch.float32, device=dev)
                    plan.text = torch.empty_like(cond)
                    plan.controller = controller
                    plan.x.copy_(latent)
                    plan.text.copy_(cond)
                    for i in range(n):
                        plan.steps.capture(lambda i=i: inv_step(i, plan.x, plan.text, controller, plan.outputs))
                    controller._graph_plan_id = plan.id
                    # the capture advanced the controller's Python state to the end of the loop; the replay below fills its tensors
                    self._plans[key] = plan
                plan.x.copy_(latent)
                plan.text.copy_(cond)
                for i in range(n):
                    plan.steps.replay(i)
                controller.adopt_from(plan.controller)
                return [latent] + [o.clone() for o in plan.outputs]
            if key is not None:
                self._seen.add(key)
            all_latent = [latent]
            x = latent.detach().to(dev, torch.float32).contiguous().clone()
            for i in range(n):
                if teacher_latents is not None:
                    x.copy_(teacher_latents[i].to(dev, torch.float32))
                inv_step(i, x, cond, controller, all_latent)
        return all_latent

    def next_clean2noise_step(self, model_output, timestep, sample):
        """p2p_ddim_spatial_temporal.py:150-161 on tensors (the loop above uses the fused kernel with the same coefficients)."""
        step = self.scheduler.config.num_train_timesteps // self.scheduler.num_inference_steps
        timestep, next_timestep = min(int(timestep) - step, 999), int(timestep)
        x = sample.detach().to(torch.float32).contiguous().clone()
        ops.ddim_invert_step(x, model_output.to(torch.float32).contiguous(), self._alpha(timestep), self._alpha(next_timestep))
        return x

    def get_timesteps(self, num_inference_steps, strength, device):
        init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
        t_start = max(num_inference_steps - init_timestep, 0)
        return self.scheduler.timesteps[t_start:], num_inference_steps - t_start

    # ---- text-to-video sampling (stable_diffusion.py:355-564) -----------------------------------------------------------
    MAX_SAMPLE_ROWS = 64  # attention rows (CFG halves x clips x frames) of one un-hooked UNet call: kMaxBF of fz_attention_f16

    def prepare_latents(self, batch_size, num_channels_latents, clip_length, height, width, dtype, device, generator, latents=None):
        """stable_diffusion.py:355-401: Gaussian latents [batch_size, C, clip_length, h, w] (one draw per generator of a list)."""
        shape = (batch_size, num_channels_latents, clip_length, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch size of "
                             f"{batch_size}. Make sure the batch size matches the length of the generators.")
        if latents is None:
            if isinstance(generator, list):
                latents = torch.cat([torch.randn((1,) + shape[1:], generator=g, device=device, dtype=dtype) for g in generator]).to(device)
            else:
                latents = torch.randn(shape, generator=generator, device=device, dtype=dtype).to(device)
        else:
            if latents.shape != shape:
                raise ValueError(f"Unexpected latents shape, got {latents.shape}, expected {shape}")
            latents = latents.to(device)
        return latents * self.scheduler.init_noise_sigma

    def _check_sampling(self, guidance_scale, eta, generator, clip_length):
        """The refusals of the sampler, before any GPU work."""
        if eta < 0:
            raise ValueError(f"eta must be >= 0, got {eta}")
        if eta > 0 and isinstance(generator, list):
            # DDIMScheduler.step draws its noise with torch.randn(generator=generator), which takes one generator
            raise ValueError("eta > 0 draws each step's noise from one generator: a list of generators is not supported")
        if self._engine_is_sharded():
            raise NotImplementedError("text-to-video sampling does not run frame-sharded")
        rows = (2 if guidance_scale > 1.0 else 1) * clip_length
        if rows > self.MAX_SAMPLE_ROWS:
            raise ValueError(f"a clip of {clip_length} frames needs {rows} attention rows per UNet call (CFG doubles them), more than "
                             f"{self.MAX_SAMPLE_ROWS}")

    def _ddim_sigma(self, t: int, eta: float) -> float:
        """eta * sqrt(DDIMScheduler._get_variance(t, t_prev)) of diffusers 0.11.1."""
        a_t, a_p = self._alpha(t), self._alpha(t - self.scheduler.config.num_train_timesteps // self.scheduler.num_inference_steps)
        return float(eta) * (((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)) ** 0.5

    def _sample_loop(self, latents, text_embeddings, guidance_scale, eta, generator, callback, callback_steps, variance_noise=None,
                     teacher_latents=None):
        """The denoising loop of stable_diffusion.py:519-549 (also ddim_spatial_temporal.py:255-284) on the un-hooked sm_90a UNet and
        fz_ddim_sample_step.  Clips run together in UNet calls of at most MAX_SAMPLE_ROWS attention rows; every clip gets, bit for bit, what
        a call of that clip alone gives it.  At eta > 0, step i adds sigma_i * z_i with z_i = torch.randn of the guided noise's shape from
        `generator` (the draw of DDIMScheduler.step), drawn in step order.  Returns the final latents in the latents' dtype.
        variance_noise / teacher_latents (parity tests only): the per-step noise to use instead of drawing it, and the reference latents
        after each step (step i > 0 then starts from teacher_latents[i - 1])."""
        latents_dtype = latents.dtype
        dev = self.unet.device
        engine = self.unet.engine()
        do_cfg = guidance_scale > 1.0
        timesteps = [int(t) for t in self.scheduler.timesteps]
        n = len(timesteps)
        step = self.scheduler.config.num_train_timesteps // self.scheduler.num_inference_steps
        coef = [(self._alpha(t), self._alpha(t - step), self._ddim_sigma(t, eta)) for t in timesteps]
        stochastic = eta > 0
        B, F = latents.shape[0], latents.shape[2]
        per_call = max(1, self.MAX_SAMPLE_ROWS // ((2 if do_cfg else 1) * F))
        spans = [(a, min(B, a + per_call)) for a in range(0, B, per_call)]
        text = text_embeddings.to(dev)
        if do_cfg:
            uncond, cond = text.chunk(2)
            texts = [torch.cat([uncond[a:b], cond[a:b]]).contiguous() for a, b in spans]
        else:
            texts = [text[a:b].contiguous() for a, b in spans]

        def draw(i):
            if variance_noise is not None:
                return variance_noise[i].to(dev, torch.float32)
            return torch.randn(latents.shape, generator=generator, device=dev, dtype=latents_dtype).to(torch.float32)

        def sample_step(i, x, texts_, z):
            t = timesteps[i]
            a_t, a_p, sigma = coef[i]
            for (a, b), tx in zip(spans, texts_):
                xc = x[a:b]
                eps = engine.forward(torch.cat([xc, xc]) if do_cfg else xc, float(t), tx, None, items=b - a)
                ops.ddim_sample_step(xc, eps, guidance_scale if do_cfg else None, a_t, a_p, sigma, None if z is None else z[a:b])

        with torch.cuda.device(dev):
            key = None
            if self.graph_mode != "off" and teacher_latents is None:
                key = ("sample", tuple(latents.shape), tuple(timesteps), tuple(text.shape), float(guidance_scale), float(eta), id(engine),
                       engine.shard_signature())
            if key is not None and (key in self._plans or key in self._seen):
                plan = self._plans.get(key)
                if plan is None:
                    from .graphs import LoopPlan
                    plan = LoopPlan(dev)
                    plan.x = torch.empty(latents.shape, dtype=torch.float32, device=dev)
                    plan.text = [torch.empty_like(tx) for tx in texts]
                    plan.noise = torch.zeros((n, *latents.shape), dtype=torch.float32, device=dev) if stochastic else None
                    plan.x.copy_(latents)
                    for buf, tx in zip(plan.text, texts):
                        buf.copy_(tx)
                    for i in range(n):
                        plan.steps.capture(lambda i=i: sample_step(i, plan.x, plan.text, None if plan.noise is None else plan.noise[i]))
                    self._plans[key] = plan
                # every step's noise is drawn before the replay, one draw per step in step order: the generator advances as in the eager loop
                if stochastic:
                    for i in range(n):
                        plan.noise[i].copy_(draw(i))
                plan.x.copy_(latents)
                for buf, tx in zip(plan.text, texts):
                    buf.copy_(tx)
                for i in range(n):
                    plan.steps.replay(i)
                    if callback is not None and i % callback_steps == 0:
                        callback(i, timesteps[i], plan.x.to(latents_dtype))
                x = plan.x.clone()
            else:
                if key is not None:
                    self._seen.add(key)
                x = latents.detach().to(dev, torch.float32).contiguous().clone()
                for i, t in enumerate(timesteps):
                    if teacher_latents is not None and i > 0:
                        x.copy_(teacher_latents[i - 1].to(dev, torch.float32))
                    sample_step(i, x, texts, draw(i) if stochastic else None)
                    if callback is not None and i % callback_steps == 0:
                        callback(i, t, x.to(latents_dtype))
        return x.to(latents_dtype)

    def _sample_output(self, latents, output_type, return_dict):
        if output_type == "latent":
            image = latents
        else:
            image = self.decode_latents(latents)
            if output_type == "pil":
                image = self.numpy_to_pil(image)
        if not return_dict:
            return (image, None)
        return StableDiffusionPipelineOutput(images=image, nsfw_content_detected=None)

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]], height: Optional[int] = None, width: Optional[int] = None, num_inference_steps: int = 50,
                 clip_length: int = 8, guidance_scale: float = 7.5, negative_prompt: Optional[Union[str, List[str]]] = None,
                 num_images_per_prompt: Optional[int] = 1, eta: float = 0.0,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None, latents: Optional[torch.FloatTensor] = None,
                 output_type: Optional[str] = "pil", return_dict: bool = True,
                 callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None, callback_steps: Optional[int] = 1,
                 variance_noise=None, teacher_latents=None):
        """Text-to-video generation, stable_diffusion.py:403-564: Gaussian latents (prepare_latents), then `num_inference_steps` DDIM steps
        with classifier-free guidance when guidance_scale > 1 and the stochastic DDIM noise of eta > 0 (diffusers' DDIMScheduler.step).
        The DDIM arithmetic runs in fp32 on the GPU.  output_type: "pil", "numpy" or "latent".
        variance_noise / teacher_latents are for parity tests only (see _sample_loop)."""
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps)
        self.check_frame_size(height, width, "__call__")
        self._check_sampling(guidance_scale, eta, generator, clip_length)
        batch_size = 1 if isinstance(prompt, str) else len(prompt)
        device = self._execution_device
        do_cfg = guidance_scale > 1.0
        text_embeddings = self._encode_prompt(prompt, device, num_images_per_prompt, do_cfg, negative_prompt)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        latents = self.prepare_latents(batch_size * num_images_per_prompt, self.unet.config.in_channels, clip_length, height, width,
                                       text_embeddings.dtype, device, generator, latents)
        latents = self._sample_loop(latents, text_embeddings, guidance_scale, eta, generator, callback, callback_steps, variance_noise,
                                    teacher_latents)
        return self._sample_output(latents, output_type, return_dict)


class P2pDDIMSpatioTemporalPipeline(SpatioTemporalStableDiffusionPipeline):
    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler, disk_store: bool = False):
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler)
        self.store_controller = attention_util.AttentionStore(disk_store=disk_store)
        self.empty_controller = attention_util.EmptyControl()

    # ---- inversion ----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def prepare_latents_ddim_inverted(self, image, batch_size, num_images_per_prompt, text_embeddings, store_attention=False,
                                      prompt=None, generator=None, LOW_RESOURCE=True, save_path=None):
        """p2p_ddim_spatial_temporal.py:68-129."""
        self.check_frame_size(image.shape[-2], image.shape[-1], "prepare_latents_ddim_inverted")
        self.prepare_before_train_loop()
        if store_attention:
            attention_util.register_attention_control(self, self.store_controller)
        resource_default_value = self.store_controller.LOW_RESOURCE
        self.store_controller.LOW_RESOURCE = LOW_RESOURCE
        init_bcfhw = self._clean_latents_bcfhw(image, batch_size * num_images_per_prompt, generator)
        out = self.ddim_clean2noisy_loop(init_bcfhw, text_embeddings, self.store_controller)
        if store_attention and (save_path is not None):
            os.makedirs(save_path + "/cross_attention")
            from .visualization import show_cross_attention
            show_cross_attention(self.tokenizer, prompt, self.store_controller, 16, ["up", "down"], save_path=save_path + "/cross_attention")
            attention_util.register_attention_control(self, self.empty_controller)
        self.store_controller.LOW_RESOURCE = resource_default_value
        return out

    # ---- edit -----------------------------------------------------------------------------------------------------------
    def _make_edit_controller(self, prompt: str, source_prompt: str, num_inference_steps: int, store=None, **kwargs):
        """The make_controller call of p2p_ddim_spatial_temporal.py:176-193: one target prompt against the inversion store (`store`, by
        default self.store_controller)."""
        len_source = len(source_prompt.split(" "))
        len_target = len(prompt.split(" "))
        equal_length = len_source == len_target
        return attention_util.make_controller(
            self.tokenizer, [source_prompt, prompt], NUM_DDIM_STEPS=num_inference_steps,
            is_replace_controller=kwargs.get("is_replace_controller", True) and equal_length,
            cross_replace_steps=kwargs["cross_replace_steps"], self_replace_steps=kwargs["self_replace_steps"],
            blend_words=kwargs.get("blend_words", None), equilizer_params=kwargs.get("eq_params", None),
            additional_attention_store=self.store_controller if store is None else store,
            use_inversion_attention=kwargs["use_inversion_attention"],
            blend_th=kwargs.get("blend_th", (0.3, 0.3)), blend_self_attention=kwargs.get("blend_self_attention", None),
            blend_latents=kwargs.get("blend_latents", None), save_path=kwargs.get("save_path", None),
            save_self_attention=kwargs.get("save_self_attention", True), disk_store=kwargs.get("disk_store", False))

    def p2preplace_edit(self, **kwargs):
        """p2p_ddim_spatial_temporal.py:172-222."""
        edit_controller = self._make_edit_controller(**kwargs)
        attention_util.register_attention_control(self, edit_controller)
        sdimage_output = self.sd_ddim_pipeline(controller=edit_controller, **kwargs)
        mask_list = edit_controller.latent_blend.mask_list if hasattr(edit_controller.latent_blend, "mask_list") else None
        attention_output = None
        if len(edit_controller.attention_store.keys()) > 0 and kwargs.get("output_type", "pil") != "latent":
            from .visualization import show_cross_attention
            attention_output = show_cross_attention(self.tokenizer, kwargs["prompt"], edit_controller, 16, ["up", "down"])
        self.last_edit_controller = edit_controller
        attention_util.register_attention_control(self, self.empty_controller)
        return {"sdimage_output": sdimage_output, "attention_output": attention_output, "mask_list": mask_list}

    MAX_BATCH_ROWS = 128  # CFG rows (2 x prompts x frames) of one grouped attention launch

    @torch.no_grad()
    def p2preplace_edit_batch(self, prompts: List[str], p2p_configs: List[dict], source_prompt: str, latents: torch.Tensor,
                              num_inference_steps: int, guidance_scale: float, save_path: Optional[str] = None, output_type: str = "pil",
                              negative_prompt=None, callback=None, callback_steps: int = 1):
        """Edit ONE inverted clip (`latents`: x_T [1, 4, F, h, w] of the inversion held by `self.store_controller`) with several target
        prompts in one batched pass: every UNet forward runs the K prompts' CFG rows together.  Prompt k gets, bit for bit, what
        `p2preplace_edit(prompt=prompts[k], **p2p_configs[k], ...)` gives it (latents, masks, running attention sums).  Returns one
        p2preplace_edit result dict per prompt; `self.last_edit_controllers` holds the K edit controllers.  callback(i, t, latents[K, ...])."""
        prompts = list(prompts)
        p2p_configs = [dict(c) for c in p2p_configs]
        K = len(prompts)
        if K == 0 or len(p2p_configs) != K:
            raise ValueError(f"p2preplace_edit_batch: {K} prompts and {len(p2p_configs)} p2p configs")
        if K > attention_util._lib.MAX_ATTN_GROUPS:
            raise ValueError(f"p2preplace_edit_batch: at most {attention_util._lib.MAX_ATTN_GROUPS} prompts per batch, got {K}")
        if latents is None or latents.dim() != 5 or latents.shape[0] != 1:
            raise ValueError("p2preplace_edit_batch: latents must be the inverted clip's x_T of shape [1, 4, F, h, w]")
        F = latents.shape[2]
        if 2 * K * F > self.MAX_BATCH_ROWS:
            raise ValueError(f"p2preplace_edit_batch: 2 x {K} prompts x {F} frames = {2 * K * F} CFG rows exceed {self.MAX_BATCH_ROWS}")
        for k, c in enumerate(p2p_configs):
            if int(c.get("num_inference_steps", num_inference_steps)) != int(num_inference_steps):
                raise ValueError(f"p2preplace_edit_batch: prompt {k} asks for num_inference_steps={c['num_inference_steps']}")
            if float(c.get("guidance_scale", guidance_scale)) != float(guidance_scale):
                raise ValueError(f"p2preplace_edit_batch: prompt {k} asks for guidance_scale={c['guidance_scale']}")
            if float(c.get("eta", 0.0)) != 0.0:
                raise NotImplementedError("FateZero's DDIM path is deterministic (eta = 0)")
        engine = getattr(self.unet, "_engine", None)  # not built here: nothing below may touch the GPU before the checks pass
        if getattr(engine, "shard", None) is not None:
            raise NotImplementedError("p2preplace_edit_batch: frame-sharded batched edits are not supported")
        store = self.store_controller
        if getattr(store, "disk_store", False) or getattr(store, "host_spill", False):
            raise NotImplementedError("p2preplace_edit_batch: disk_store / host_spill inversion stores are edited one prompt at a time")
        drop = ("prompt", "source_prompt", "num_inference_steps", "guidance_scale", "eta", "save_path", "latents", "output_type",
                "negative_prompt", "callback", "callback_steps")
        edits = [self._make_edit_controller(prompt=pr, source_prompt=source_prompt, num_inference_steps=num_inference_steps, save_path=save_path,
                                            **{k: v for k, v in c.items() if k not in drop})
                 for pr, c in zip(prompts, p2p_configs)]
        batch = attention_util.AttentionControlEditBatch(edits)
        attention_util.register_attention_control(self, batch)
        try:
            out = self.sd_ddim_pipeline(prompt=prompts, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                        negative_prompt=negative_prompt, latents=latents, output_type="latent", callback=callback,
                                        callback_steps=callback_steps, controller=batch)
        finally:
            attention_util.register_attention_control(self, self.empty_controller)
        self.last_edit_controllers = edits
        return self._batch_results(prompts, edits, out.images, output_type)

    def _batch_results(self, prompts, edits, lat, output_type):
        """One p2preplace_edit result dict per prompt of a batched edit."""
        results = []
        for k, (pr, e) in enumerate(zip(prompts, edits)):
            lk = lat[k:k + 1]
            if output_type == "latent":
                sd = StableDiffusionPipelineOutput(images=lk, nsfw_content_detected=None)
            else:
                image = self.decode_latents(lk)  # per prompt: the VAE's GroupNorm chunking depends on the batch
                sd = StableDiffusionPipelineOutput(images=self.numpy_to_pil(image) if output_type == "pil" else image, nsfw_content_detected=None)
            mask_list = e.latent_blend.mask_list if hasattr(e.latent_blend, "mask_list") else None
            attention_output = None
            if len(e.attention_store.keys()) > 0 and output_type != "latent":
                from .visualization import show_cross_attention
                attention_output = show_cross_attention(self.tokenizer, pr, e, 16, ["up", "down"])
            results.append({"sdimage_output": sd, "attention_output": attention_output, "mask_list": mask_list})
        return results

    # ---- several source clips in one pass (test_fatezero_dataset.py sweeps clip after clip) --------------------------------------
    def map_cache_admission(self, clips: int, frames: int, h: int, w: int, steps: int, save_self_attention: bool = True,
                            free_bytes: Optional[int] = None) -> int:
        """Bytes of the inversion map caches of `clips` clips of `frames` frames at latent size h x w over `steps` DDIM steps (the slab
        shapes of controllers.map_cache_bytes).  Raises ValueError when they exceed `free_bytes` (default: the free HBM of the UNet's
        device plus the blocks PyTorch holds unused)."""
        per_step, once = attention_util.map_cache_bytes(dict(self.unet.config), dict(self.unet.model_config), h, w, save_self_attention)
        need = clips * frames * (steps * per_step + once)
        if free_bytes is None:
            dev = self.unet.device
            if dev.type != "cuda":
                return need
            free_bytes = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        if need > free_bytes:
            raise ValueError(f"the inversion map caches of {clips} clips x {frames} frames x {steps} steps need {need / 2 ** 30:.1f} GiB, "
                             f"{free_bytes / 2 ** 30:.1f} GiB of HBM are free: invert the clips in smaller batches")
        return need

    @torch.no_grad()
    def prepare_latents_ddim_inverted_batch(self, source_prompts: List[str], images=None, latents=None, generator=None,
                                            store_attention: bool = True):
        """DDIM-invert K source clips in ONE batched pass (p2p_ddim_spatial_temporal.py:68-129 once per clip, as test_fatezero_dataset.py
        does): every UNet forward runs the K clips together, each with its own attention store.  `images`: K frame tensors [F, 3, H, W]
        (VAE-encoded clip by clip with `generator`, one generator or a list of K) or `latents`: K clean latents [1, 4, F, h, w].  The
        scheduler's current timesteps are used, as by prepare_latents_ddim_inverted.

        Clip k's N+1 latents, and the state of its store (`attention_store_all_step`, `attention_store`, `latents_store`, `cur_step`), are
        bit for bit those of prepare_latents_ddim_inverted(..., store_attention=store_attention) on that clip alone.  Returns the K lists
        of N+1 latents ([0] clean, [-1] x_T) and sets `self.store_controllers` to the K stores."""
        source_prompts = list(source_prompts)
        K = len(source_prompts)
        if (images is None) == (latents is None):
            raise ValueError("prepare_latents_ddim_inverted_batch: pass either images or latents")
        clips = list(images if images is not None else latents)
        if K == 0 or len(clips) != K:
            raise ValueError(f"prepare_latents_ddim_inverted_batch: {K} source prompts and {len(clips)} clips")
        if K > attention_util._lib.MAX_ATTN_GROUPS:
            raise ValueError(f"prepare_latents_ddim_inverted_batch: at most {attention_util._lib.MAX_ATTN_GROUPS} clips per batch, got {K}")
        if images is not None:
            if any(c.dim() != 4 for c in clips):
                raise ValueError("prepare_latents_ddim_inverted_batch: images must be frame tensors [F, 3, H, W]")
            geo = [(c.shape[0], c.shape[2] // self.vae_scale_factor, c.shape[3] // self.vae_scale_factor) for c in clips]
        else:
            if any(c.dim() != 5 or c.shape[0] != 1 for c in clips):
                raise ValueError("prepare_latents_ddim_inverted_batch: latents must be clean latents [1, 4, F, h, w]")
            geo = [(c.shape[2], c.shape[3], c.shape[4]) for c in clips]
        if len(set(geo)) != 1:
            raise ValueError(f"prepare_latents_ddim_inverted_batch: the clips differ in (frames, h, w): {geo}; batch clips of one geometry")
        F, h, w = geo[0]
        if images is not None:
            self.check_frame_size(clips[0].shape[2], clips[0].shape[3], "prepare_latents_ddim_inverted_batch")
        else:
            self.check_frame_size(h * self.vae_scale_factor, w * self.vae_scale_factor, "prepare_latents_ddim_inverted_batch")
        if K * F > self.MAX_BATCH_ROWS:
            raise ValueError(f"prepare_latents_ddim_inverted_batch: {K} clips x {F} frames = {K * F} rows exceed {self.MAX_BATCH_ROWS}")
        if self._engine_is_sharded():
            raise NotImplementedError("prepare_latents_ddim_inverted_batch: frame-sharded batched inversions are not supported")
        stores = [] if self.store_controller.disk_store else [attention_util.AttentionStore() for _ in range(K)]
        if not stores or any(s.host_spill for s in stores):
            raise NotImplementedError("prepare_latents_ddim_inverted_batch: disk_store / host_spill stores are inverted one clip at a time")
        gens = list(generator) if isinstance(generator, list) else [generator] * K
        if len(gens) != K:
            raise ValueError(f"prepare_latents_ddim_inverted_batch: {len(gens)} generators for {K} clips")
        N = len(self.scheduler.timesteps)
        batch = attention_util.AttentionStoreBatch(stores, store_maps=store_attention)
        for s in stores:
            s.LOW_RESOURCE = True  # before the plan signature is read: a captured inversion was keyed with it set
        # the previous batch's stores are let go before the admission counts the free HBM (a caller still holding them keeps their caches);
        # a batch that will replay a captured inversion refills that plan's caches and allocates none
        self.store_controllers = None
        replays = self.graph_mode != "off" and any(
            k[0] == "inv" and k[1] == (K, 4, F, h, w) and k[3] == tuple(int(t) for t in self.scheduler.timesteps) and k[5] == batch.graph_signature()
            for k in self._plans)
        if store_attention and not replays:
            self.map_cache_admission(K, F, h, w, N)
        self.prepare_before_train_loop()
        if images is not None:
            # clip by clip: the VAE's GroupNorm chunking depends on the batch
            clean = []
            for img, g in zip(clips, gens):
                z = 0.18215 * self._vae_encode_sample(img, g)
                clean.append(z.reshape(1, F, *z.shape[1:]).permute(0, 2, 1, 3, 4))
        else:
            clean = clips
        dev = self.unet.device
        per = [self._encode_prompt(p, dev, 1, True, None).to(dev) for p in source_prompts]
        text = torch.cat([e[:1] for e in per] + [e[1:] for e in per])
        attention_util.register_attention_control(self, batch)
        try:
            out = self.ddim_clean2noisy_loop(torch.cat(clean), text, batch)
        finally:
            attention_util.register_attention_control(self, self.empty_controller)
            for s in stores:
                s.LOW_RESOURCE = False
        self.store_controllers = stores
        return [[c] + [o[k:k + 1] for o in out[1:]] for k, c in enumerate(clean)]

    @torch.no_grad()
    def p2preplace_edit_clips(self, jobs: List[dict], num_inference_steps: int, guidance_scale: float, output_type: str = "pil",
                              save_path: Optional[str] = None, negative_prompt=None, callback=None, callback_steps: int = 1):
        """Edit several inverted clips in ONE batched pass (p2p_ddim_spatial_temporal.py:172-222 once per job).  Each job is
        dict(store=<the clip's AttentionStore>, latents=<its x_T [1, 4, F, h, w]>, prompt=..., source_prompt=..., **p2p_config); any
        number of jobs may edit the same clip.  Job j gets, bit for bit, what p2preplace_edit(prompt=..., **p2p_config) gives it against
        its own store (latents, masks, running attention sums).  Returns one p2preplace_edit result dict per job (VAE decode per job);
        `self.last_edit_controllers` holds the edit controllers.  callback(i, t, latents[J, ...])."""
        jobs = [dict(j) for j in jobs]
        J = len(jobs)
        if J == 0:
            raise ValueError("p2preplace_edit_clips: no jobs")
        if J > attention_util._lib.MAX_ATTN_GROUPS:
            raise ValueError(f"p2preplace_edit_clips: at most {attention_util._lib.MAX_ATTN_GROUPS} jobs per batch, got {J}")
        for k, j in enumerate(jobs):
            missing = [n for n in ("store", "latents", "prompt", "source_prompt") if j.get(n) is None]
            if missing:
                raise ValueError(f"p2preplace_edit_clips: job {k} lacks {missing}")
            if j["latents"].dim() != 5 or j["latents"].shape[0] != 1:
                raise ValueError(f"p2preplace_edit_clips: job {k}: latents must be the clip's x_T of shape [1, 4, F, h, w]")
        shapes = [tuple(j["latents"].shape) for j in jobs]
        if len(set(shapes)) != 1:
            raise ValueError(f"p2preplace_edit_clips: the clips differ in shape {shapes}; batch clips of one (frames, h, w)")
        F = shapes[0][2]
        self.check_frame_size(shapes[0][3] * self.vae_scale_factor, shapes[0][4] * self.vae_scale_factor, "p2preplace_edit_clips")
        if 2 * J * F > self.MAX_BATCH_ROWS:
            raise ValueError(f"p2preplace_edit_clips: 2 x {J} jobs x {F} frames = {2 * J * F} CFG rows exceed {self.MAX_BATCH_ROWS}")
        for k, j in enumerate(jobs):
            if int(j.get("num_inference_steps", num_inference_steps)) != int(num_inference_steps):
                raise ValueError(f"p2preplace_edit_clips: job {k} asks for num_inference_steps={j['num_inference_steps']}")
            if float(j.get("guidance_scale", guidance_scale)) != float(guidance_scale):
                raise ValueError(f"p2preplace_edit_clips: job {k} asks for guidance_scale={j['guidance_scale']}")
            if float(j.get("eta", 0.0)) != 0.0:
                raise NotImplementedError("FateZero's DDIM path is deterministic (eta = 0)")
            st = j["store"]
            if getattr(st, "disk_store", False) or getattr(st, "host_spill", False):
                raise NotImplementedError("p2preplace_edit_clips: disk_store / host_spill inversion stores are edited one clip at a time")
            if len(st.attention_store_all_step) != int(num_inference_steps):
                raise ValueError(f"p2preplace_edit_clips: job {k}'s store holds {len(st.attention_store_all_step)} inversion steps, the edit "
                                 f"runs {num_inference_steps}; batch clips inverted with one step count")
        stores = list({id(j["store"]): j["store"] for j in jobs}.values())
        plans = [s._graph_plan_id for s in stores if getattr(s, "_graph_plan_id", None) is not None]
        if len(set(plans)) != len(plans):
            raise ValueError("p2preplace_edit_clips: two stores hold the maps of the same captured inversion slot; only the clip inverted last "
                             "by that plan still has its maps")
        if self._engine_is_sharded():
            raise NotImplementedError("p2preplace_edit_clips: frame-sharded batched edits are not supported")
        drop = ("store", "latents", "prompt", "source_prompt", "num_inference_steps", "guidance_scale", "eta", "save_path", "output_type",
                "negative_prompt", "callback", "callback_steps")
        edits = [self._make_edit_controller(prompt=j["prompt"], source_prompt=j["source_prompt"], num_inference_steps=num_inference_steps,
                                            save_path=save_path, store=j["store"], **{k: v for k, v in j.items() if k not in drop})
                 for j in jobs]
        ctrl = attention_util.AttentionControlEditClips(edits)
        prompts = [j["prompt"] for j in jobs]
        attention_util.register_attention_control(self, ctrl)
        try:
            out = self.sd_ddim_pipeline(prompt=prompts, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                        negative_prompt=negative_prompt, latents=torch.cat([j["latents"] for j in jobs]), output_type="latent",
                                        callback=callback, callback_steps=callback_steps, controller=ctrl)
        finally:
            attention_util.register_attention_control(self, self.empty_controller)
        self.last_edit_controllers = edits
        return self._batch_results(prompts, edits, out.images, output_type)

    @torch.no_grad()
    def __call__(self, **kwargs):
        edit_type = kwargs["edit_type"]
        assert edit_type in ["save", "swap", None]
        if edit_type is None:
            return self.sd_ddim_pipeline(controller=None, **kwargs)
        if edit_type == "save":
            self.store_controller = attention_util.AttentionStore()
            attention_util.register_attention_control(self, self.store_controller)
            sdimage_output = self.sd_ddim_pipeline(controller=self.store_controller, **kwargs)
            from .visualization import show_cross_attention
            attention_output = show_cross_attention(self.tokenizer, kwargs["prompt"], self.store_controller, 16, ["up", "down"])
            attention_util.register_attention_control(self, self.empty_controller)
            return {"sdimage_output": sdimage_output, "attention_output": attention_output, "mask_list": None}
        return self.p2preplace_edit(**kwargs)

    @torch.no_grad()
    def sd_ddim_pipeline(self, prompt: Union[str, List[str]], image=None, height: Optional[int] = None, width: Optional[int] = None,
                         strength: float = None, num_inference_steps: int = 50, guidance_scale: float = 7.5,
                         negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                         eta: float = 0.0, generator=None, latents: Optional[torch.FloatTensor] = None, output_type: Optional[str] = "pil",
                         return_dict: bool = True, callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None,
                         callback_steps: Optional[int] = 1, controller=None, teacher_latents=None, **args):
        """p2p_ddim_spatial_temporal.py:260-435 (unknown kwargs are swallowed like the reference's **args).
        teacher_latents (parity tests only): reference latents AFTER each step; step i > 0 then starts from teacher_latents[i - 1]."""
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps, strength)
        self.check_frame_size(height, width, "sd_ddim_pipeline")
        if latents is not None:  # the clip's size is that of its latents
            self.check_frame_size(latents.shape[-2] * self.vae_scale_factor, latents.shape[-1] * self.vae_scale_factor, "sd_ddim_pipeline")
        if eta != 0.0:
            raise NotImplementedError("FateZero's DDIM path is deterministic (eta = 0)")
        batch_size = 1 if isinstance(prompt, str) else len(prompt)
        device = self._execution_device
        do_cfg = guidance_scale > 1.0
        if not do_cfg:
            raise NotImplementedError("guidance_scale <= 1 (no CFG batch) is not an editing configuration of the reference YAMLs")
        is_batch = isinstance(controller, attention_util.AttentionControlEditBatch)
        is_clips = isinstance(controller, attention_util.AttentionControlEditClips)
        if is_batch:
            # K prompts of one clip: [uncond_1..K ; cond_1..K], each prompt encoded on its own so that its embedding is bitwise the one of
            # its single-prompt pass
            if num_images_per_prompt != 1 or latents is None or len(prompt) != controller.prompt_groups:
                raise ValueError("a batched edit needs one prompt per edit controller, num_images_per_prompt=1 and the inverted latents")
            negs = negative_prompt if isinstance(negative_prompt, list) else [negative_prompt] * len(prompt)
            per = [self._encode_prompt(pr, device, 1, do_cfg, ng).to(self.unet.device) for pr, ng in zip(prompt, negs)]
            text_embeddings = torch.cat([e[:1] for e in per] + [e[1:] for e in per])
            if latents.shape[0] == 1 and not is_clips:
                latents = latents.expand(len(prompt), *latents.shape[1:])
        else:
            text_embeddings = self._encode_prompt(prompt, device, num_images_per_prompt, do_cfg, negative_prompt).to(self.unet.device)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = [int(t) for t in self.scheduler.timesteps]
        if latents is None:
            # the internal inversion runs batch 1 through the UNet: the edit controller registered by p2preplace_edit must not see it
            # (the reference's inversion hooks run the store logic of the edit controller on that pass; here it is detached)
            registered = getattr(self.unet, "_controller", None)
            attention_util.register_attention_control(self, self.empty_controller)
            try:
                latents = self.prepare_latents_ddim_inverted(image, batch_size, num_images_per_prompt, text_embeddings,
                                                             store_attention=False, generator=generator)[-1]
            finally:
                attention_util.register_attention_control(self, registered)
        latents_dtype = latents.dtype
        dev = self.unet.device
        text_embeddings = text_embeddings.contiguous()
        is_edit = is_batch or isinstance(controller, attention_util.AttentionControlEdit)
        step = self.scheduler.config.num_train_timesteps // self.scheduler.num_inference_steps
        n = len(timesteps)

        def edit_step(i, x, text, ctrl):
            t = timesteps[i]
            x2 = torch.cat([x, x], dim=0)
            eps2 = self.unet(x2, t, encoder_hidden_states=text).sample
            blend = ctrl.latent_blend_args(x.shape[-2], x.shape[-1]) if is_edit else None
            a_t, a_prev = self._alpha(t), self._alpha(t - step)
            if is_clips:
                ops.cfg_ddim_step_multi(x, eps2.contiguous(), guidance_scale, a_t, a_prev,
                                        blends=[None if b is None else dict(b, x_inv=b["x_inv"].contiguous()) for b in blend])
            elif is_batch:
                live = [b for b in blend if b is not None]
                x_inv = live[0]["x_inv"].contiguous() if live else None
                if any(b["x_inv"].data_ptr() != live[0]["x_inv"].data_ptr() for b in live[1:]):
                    raise RuntimeError("the edits of a batch disagree on the inverted latent of this step")
                ops.cfg_ddim_step_batched(x, eps2.contiguous(), guidance_scale, a_t, a_prev, x_inv=x_inv, blends=blend)
            elif blend is not None:
                ops.cfg_ddim_step(x, eps2.contiguous(), guidance_scale, a_t, a_prev, x_inv=blend["x_inv"].contiguous(),
                                  mask_a=blend["mask_a"], mask_b=blend["mask_b"], apply_blend=blend["apply_blend"])
            else:
                ops.cfg_ddim_step(x, eps2.contiguous(), guidance_scale, a_t, a_prev)
            if ctrl is not None:
                if is_edit:
                    ctrl.step_callback(x, blend_fused=True)
                else:
                    ctrl.step_callback(x)

        with torch.cuda.device(dev):
            sig = None
            if (self.graph_mode != "off" and teacher_latents is None and is_edit and getattr(self.unet, "_controller", None) is controller
                    and controller.cur_step == 0):
                sig = controller.graph_signature()
            key = None if sig is None else ("edit", tuple(latents.shape), tuple(timesteps), tuple(text_embeddings.shape), float(guidance_scale),
                                            sig[:-1], id(self.unet.engine()), self.unet.engine().shard_signature())
            store_plan = None if sig is None else sig[-1]
            if key is not None and store_plan is not None and ((key, store_plan) in self._plans or key in self._seen):
                plan = self._plans.get((key, store_plan))
                if plan is None:
                    from .graphs import LoopPlan
                    plan = LoopPlan(dev)
                    plan.x = torch.empty(latents.shape, dtype=torch.float32, device=dev)
                    plan.text = torch.empty_like(text_embeddings)
                    plan.controller = controller
                    controller.prepare_tables(dev)
                    plan.x.copy_(latents)
                    plan.text.copy_(text_embeddings)
                    for i in range(n):
                        plan.steps.capture(lambda i=i: edit_step(i, plan.x, plan.text, controller))
                    self._plans[(key, store_plan)] = plan
                plan.x.copy_(latents)
                plan.text.copy_(text_embeddings)
                plan.controller.load_tables_from(controller)
                for i in range(n):
                    plan.steps.replay(i)
                    if callback is not None and i % callback_steps == 0:
                        callback(i, timesteps[i], plan.x.to(latents_dtype))
                controller.adopt_from(plan.controller)
                x = plan.x.clone()
            else:
                if key is not None:
                    self._seen.add(key)
                x = latents.detach().to(dev, torch.float32).contiguous().clone()
                for i, t in enumerate(timesteps):
                    if teacher_latents is not None and i > 0:
                        x.copy_(teacher_latents[i - 1].to(x.device, torch.float32))
                    edit_step(i, x, text_embeddings, controller)
                    if callback is not None and i % callback_steps == 0:
                        callback(i, t, x.to(latents_dtype))
        latents = x.to(latents_dtype)
        if output_type == "latent":
            return StableDiffusionPipelineOutput(images=latents, nsfw_content_detected=None)
        image = self.decode_latents(latents)
        if output_type == "pil":
            image = self.numpy_to_pil(image)
        if not return_dict:
            return (image, None)
        return StableDiffusionPipelineOutput(images=image, nsfw_content_detected=None)

    def print_pipeline(self, logger):
        print("Overview function of pipeline: ")
        print(self.__class__)
        logger.info(str({k: getattr(self, k).__class__ for k in self.config.keys()}))
        print(f"python version {sys.version}")
        print(f"torch version {torch.__version__}")
        print("validate gpu status:")
        print(torch.tensor(1.0).cuda() * 2)
        from . import _lib
        print(f"libfatezero_b200 version {_lib.load().fz_version()} at {_lib.LIB_PATH}")


class DDIMSpatioTemporalStableDiffusionPipeline(SpatioTemporalStableDiffusionPipeline):
    """Drop-in for video_diffusion/pipelines/ddim_spatial_temporal.py (the "Tune-A-Video + DDIM inversion" baseline): DDIM-invert the
    clip with the source prompt, then denoise it with the target prompt under classifier-free guidance, with no attention control.  The
    inversion is the shared ddim_clean2noisy_loop, the denoising the text-to-video sampler's loop (_sample_loop)."""

    @torch.no_grad()
    def prepare_latents_ddim_inverted(self, image, batch_size, num_images_per_prompt, text_embeddings, generator=None):
        """ddim_spatial_temporal.py:45-90: VAE-encode `image` [(b f), 3, H, W] with b = batch_size * num_images_per_prompt, invert it with
        the cond half of `text_embeddings` ([uncond ; cond]) and return the N+1 latents ([0] clean, [-1] x_T)."""
        self.check_frame_size(image.shape[-2], image.shape[-1], "prepare_latents_ddim_inverted")
        init_bcfhw = self._clean_latents_bcfhw(image, batch_size * num_images_per_prompt, generator)
        return self.ddim_clean2noisy_loop(init_bcfhw, text_embeddings)

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]], image=None, height: Optional[int] = None, width: Optional[int] = None,
                 strength: float = None, num_inference_steps: int = 50, clip_length: int = 8, guidance_scale: float = 7.5,
                 negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1, eta: float = 0.0,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None, latents: Optional[torch.FloatTensor] = None,
                 output_type: Optional[str] = "pil", return_dict: bool = True,
                 callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None, callback_steps: Optional[int] = 1, **args):
        """ddim_spatial_temporal.py:130-299.  Without `latents` the clip `image` is inverted first (prepare_latents_ddim_inverted) with
        the prompt's own embeddings, which needs guidance_scale > 1 ([uncond ; cond]).  `strength` is validated and otherwise unused, and the
        keys SampleLogger passes (edit_type, source_prompt, uncond_embeddings_list, ...) are swallowed, as in the reference.  The parity-test
        hooks variance_noise / teacher_latents of _sample_loop are read from those keys."""
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps, strength)
        batch_size = 1 if isinstance(prompt, str) else len(prompt)
        do_cfg = guidance_scale > 1.0
        if latents is not None:
            self.check_frame_size(latents.shape[-2] * self.vae_scale_factor, latents.shape[-1] * self.vae_scale_factor, "__call__")
            frames = latents.shape[2]
        else:
            if image is None:
                raise ValueError("pass the clip to invert (`image`) or its inverted `latents`")
            if not do_cfg:
                # the inversion reads the cond half of [uncond ; cond] (ddim_spatial_temporal.py:95): there is none without guidance
                raise ValueError("inverting the clip needs guidance_scale > 1 (the [uncond ; cond] text embeddings)")
            self.check_frame_size(image.shape[-2], image.shape[-1], "__call__")
            frames = image.shape[0] // (batch_size * num_images_per_prompt)
        self._check_sampling(guidance_scale, eta, generator, frames)
        device = self._execution_device
        text_embeddings = self._encode_prompt(prompt, device, num_images_per_prompt, do_cfg, negative_prompt)
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        if latents is None:
            latents = self.prepare_latents_ddim_inverted(image, batch_size, num_images_per_prompt, text_embeddings, generator)[-1]
        latents = self._sample_loop(latents, text_embeddings, guidance_scale, eta, generator, callback, callback_steps,
                                    args.get("variance_noise"), args.get("teacher_latents"))
        return self._sample_output(latents, output_type, return_dict)
