"""Generate the sampling goldens (tests/golden/sample_*.pt, format of oracle/sample.py) by running the UNMODIFIED reference pipelines
SpatioTemporalStableDiffusionPipeline.__call__ (pipelines/stable_diffusion.py:403-564) and DDIMSpatioTemporalStableDiffusionPipeline
(pipelines/ddim_spatial_temporal.py:18-299) through the tests-only shim on CPU, with synthetic weights (synth recipe), ToyTextEncoder /
ToyTokenizer, oracle.sample.EncodingVaeStub and CPU generators.  Build container only (the reference does not travel).

Two things are set up around the reference, not changed in it:
  * its __call__ reads `self.unet.in_channels` (stable_diffusion.py:501), which UNetPseudo3DConditionModel never sets: the harness sets
    that attribute on its reference UNet instance;
  * the shim's DDIMScheduler implements eta = 0 only.  RecordingDDIMScheduler below restates the eta > 0 branch of diffusers-0.11.1
    scheduling_ddim.py (variance_noise or a torch.randn draw from `generator`, ValueError when both are given, prev_sample += std * noise)
    and records every drawn noise.  That branch is unpinned: the diffusers wheel is not installed here.
Usage: python -m oracle.make_sample_golden [case ...]"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fatezero_b200 import synth  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402
from oracle import sample as sm  # noqa: E402


def recording_scheduler():
    from diffusers.schedulers import DDIMScheduler

    class RecordingDDIMScheduler(DDIMScheduler):
        noise = []

        def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, generator=None, variance_noise=None,
                 return_dict=True):
            out = super().step(model_output, timestep, sample, 0.0, use_clipped_model_output, None, None, return_dict)
            if eta <= 0:
                return out
            prev_timestep = timestep - self.config.num_train_timesteps // self.num_inference_steps
            a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
            variance = self._get_variance(timestep, prev_timestep)
            std_dev_t = eta * variance ** 0.5
            x0 = out.pred_original_sample
            prev_sample = a_p ** 0.5 * x0 + (1 - a_p - std_dev_t ** 2) ** 0.5 * model_output
            if variance_noise is not None and generator is not None:
                raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either `generator` or"
                                 " `variance_noise` stays `None`.")
            if variance_noise is None:
                variance_noise = torch.randn(model_output.shape, generator=generator, device=model_output.device, dtype=model_output.dtype)
            self.noise.append(variance_noise.detach().clone())
            prev_sample = prev_sample + variance ** 0.5 * eta * variance_noise
            out.prev_sample = prev_sample
            return out

    return RecordingDDIMScheduler(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                                  clip_sample=False, set_alpha_to_one=False, steps_offset=1)


def run_case(name: str):
    c = sm.SAMPLE_CASES[name]
    rh._prepare_imports()
    from video_diffusion.models.unet_3d_condition import UNetPseudo3DConditionModel
    from video_diffusion.pipelines.ddim_spatial_temporal import DDIMSpatioTemporalStableDiffusionPipeline
    from video_diffusion.pipelines.stable_diffusion import SpatioTemporalStableDiffusionPipeline

    cfg = dict(synth.UNET_CONFIGS[c["unet"]])
    unet = UNetPseudo3DConditionModel(**cfg, **sm.MODEL_CONFIG)
    unet.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in unet.state_dict().items()}, 0))
    unet.eval().requires_grad_(False)
    unet.in_channels = cfg["in_channels"]  # read by stable_diffusion.py:501, never set by the reference model
    sched = recording_scheduler()
    sched.noise = []
    cls = SpatioTemporalStableDiffusionPipeline if c["pipeline"] == "t2v" else DDIMSpatioTemporalStableDiffusionPipeline
    pipe = cls(vae=sm.EncodingVaeStub(), text_encoder=synth.ToyTextEncoder(cfg["cross_attention_dim"]), tokenizer=synth.ToyTokenizer(),
               unet=unet, scheduler=sched)
    trace = []
    gen = torch.Generator().manual_seed(c["seed"])
    kw = dict(prompt=c["prompt"], height=8 * c["size"], width=8 * c["size"], num_inference_steps=c["steps"], clip_length=c["frames"],
              guidance_scale=c["guidance_scale"], negative_prompt=c["negative_prompt"], num_images_per_prompt=c["num_images_per_prompt"],
              eta=c["eta"], generator=gen, output_type="np", callback=lambda i, t, l: trace.append(l.detach().float().clone()))
    gold = dict(case=name, torch=str(torch.__version__))
    t0 = time.time()
    if c["pipeline"] == "t2v":
        # the initial latents are those prepare_latents draws from the seeded generator (stable_diffusion.py:503-513)
        orig = pipe.prepare_latents
        pipe.prepare_latents = lambda *a, **k: gold.setdefault("init", orig(*a, **k).detach().float().clone())
        with torch.no_grad():
            pipe(**kw)
    else:
        image = sm.case_image(c)
        with torch.no_grad():
            emb = pipe._encode_prompt(c["source"], torch.device("cpu"), 1, True, None)
            pipe.scheduler.set_timesteps(c["steps"])
            inv = pipe.prepare_latents_ddim_inverted(image, 1, 1, emb, generator=gen)
            gold["inv_sample"] = torch.stack([sm.strided(v) for v in inv])
            gold["inv_sums"] = sm.sums(inv)
            gold["init"] = inv[-1].float().clone()
            # the SampleLogger call of validation_loop.py:88-101 (keys the pipeline swallows included)
            pipe(image=image, latents=inv[-1], strength=None, source_prompt=c["source"], edit_type=None, uncond_embeddings_list=None,
                 **kw)
    gold["seconds"] = time.time() - t0
    steps = torch.stack(trace)
    gold["step_sample"] = torch.stack([sm.strided(v) for v in steps])
    gold["sums"] = sm.sums(steps)
    gold["abs_max"] = float(steps.abs().max())
    if c["eta"] > 0:
        gold["noise"] = torch.stack([z.float() for z in sched.noise])
        assert gold["noise"].shape[0] == c["steps"], "one noise draw per step"
    path = os.path.join(ROOT, "tests", "golden", f"sample_{name}.pt")
    torch.save(gold, path)
    print(name, "->", path, f"{os.path.getsize(path) / 1e3:.0f} kB", f"{gold['seconds']:.1f}s", "|x|max", float(steps.abs().max()))


if __name__ == "__main__":
    for n in (sys.argv[1:] or list(sm.SAMPLE_CASES)):
        run_case(n)
