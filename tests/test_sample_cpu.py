"""Text-to-video sampling and the Tune-A-Video DDIM pipeline without a GPU: the CPU oracle's sampler against the reference goldens of
oracle/sample.py, the eta > 0 DDIMScheduler.step against an fp64 restatement, the refusals the pipelines raise before any GPU work, the
alias module and the keyword set the reference's SampleLogger passes."""
import inspect
import os
from types import SimpleNamespace

import pytest
import torch

from _helpers import GOLDEN_DIR, synth_weights
from fatezero_b200 import synth
from fatezero_b200.pipeline import DDIMSpatioTemporalStableDiffusionPipeline, SpatioTemporalStableDiffusionPipeline
from fatezero_b200.scheduler import DDIMScheduler
from fatezero_b200.unet import UNetPseudo3DConditionModel
from oracle import fz_oracle as fo
from oracle import sample as sm

# max |oracle - reference| over every step's latents, relative to the golden's max |x| (CPU fp32 on both sides, different operation
# order; the random-weight sampler at CFG 7.5 amplifies the rounding step by step).  Measured: 4.6e-6 (a), 0 (b), 1.8e-5 (c), 3.3e-6 (d)
ORACLE_BOUND = 1e-4


def load(name):
    return torch.load(os.path.join(GOLDEN_DIR, f"sample_{name}.pt"))


def oracle_texts(c):
    cfg = synth.UNET_CONFIGS[c["unet"]]
    tok, te = synth.ToyTokenizer(), synth.ToyTextEncoder(cfg["cross_attention_dim"])
    prompts = c["prompt"] if isinstance(c["prompt"], list) else [c["prompt"]]
    neg = c["negative_prompt"]
    neg = neg if isinstance(neg, list) or neg is None else [neg]
    return tok, te, sm.encode_text(tok, te, prompts, neg, c["guidance_scale"] > 1, c["num_images_per_prompt"])


def oracle_unet(c):
    from oracle.sd2 import OracleUNetSD2
    cls = OracleUNetSD2 if c["unet"].startswith("sd2") else fo.OracleUNet
    return cls(synth_weights(c["unet"], sm.MODEL_CONFIG), synth.UNET_CONFIGS[c["unet"]], sm.MODEL_CONFIG)


@pytest.mark.parametrize("name", list(sm.SAMPLE_CASES))
def test_oracle_matches_reference_golden(name):
    c = sm.SAMPLE_CASES[name]
    g = load(name)
    ou = oracle_unet(c)
    tok, te, text = oracle_texts(c)
    if c["pipeline"] == "ddim":
        z = sm.EncodingVaeStub().encode(sm.case_image(c)).latent_dist.sample()
        x0 = (0.18215 * z).reshape(1, c["frames"], *z.shape[1:]).permute(0, 2, 1, 3, 4)
        src = fo.encode_prompts(tok, te, c["source"])
        inv = fo.invert(ou, x0, src[1:], c["steps"], None)
        inv_s = torch.stack([sm.strided(v) for v in inv])
        assert (inv_s - g["inv_sample"]).abs().max() <= ORACLE_BOUND * g["inv_sample"].abs().max()
        assert (inv[-1] - g["init"]).abs().max() <= ORACLE_BOUND * g["init"].abs().max()
    trace = sm.sample(ou, g["init"], text, c["steps"], c["guidance_scale"], c["eta"], noise=list(g["noise"]) if c["eta"] > 0 else None)
    got = torch.stack([sm.strided(v) for v in trace])
    assert got.shape == g["step_sample"].shape
    err = (got - g["step_sample"]).abs().max() / g["abs_max"]
    assert err <= ORACLE_BOUND, f"{name}: relative error {err:.3e}"
    sq = sm.sums(trace)[:, 1]
    assert ((sq - g["sums"][:, 1]).abs() / g["sums"][:, 1]).max() <= 10 * ORACLE_BOUND
    if c["eta"] > 0:
        assert g["noise"].shape == (c["steps"],) + tuple(g["init"].shape)


def test_golden_geometry_matches_cases():
    for name, c in sm.SAMPLE_CASES.items():
        g = load(name)
        batch = (len(c["prompt"]) if isinstance(c["prompt"], list) else 1) * c["num_images_per_prompt"]
        assert tuple(g["init"].shape) == (batch, 4, c["frames"], c["size"], c["size"]), name
        assert os.path.getsize(os.path.join(GOLDEN_DIR, f"sample_{name}.pt")) < 1 << 20


# ---- DDIMScheduler.step at eta > 0 ----------------------------------------------------------------------------------------------------
def _step64(s, e, x, t, eta, z):
    a = s.alphas_cumprod.double()
    tp = t - 1000 // s.num_inference_steps
    a_t, a_p = a[t], (a[tp] if tp >= 0 else s.final_alpha_cumprod.double())
    std = eta * (((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)) ** 0.5
    x0 = (x.double() - (1 - a_t) ** 0.5 * e.double()) / a_t ** 0.5
    return a_p ** 0.5 * x0 + (1 - a_p - std ** 2) ** 0.5 * e.double() + std * z.double()


@pytest.mark.parametrize("eta", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("t_index", [0, 2, 4])
def test_scheduler_step_eta_matches_fp64(eta, t_index):
    s = DDIMScheduler()
    s.set_timesteps(5)
    t = int(s.timesteps[t_index])  # t_index 4: the last step, a_prev = final_alpha_cumprod
    g = torch.Generator().manual_seed(3)
    x, e, z = (torch.randn(1, 4, 2, 8, 8, generator=g) for _ in range(3))
    out = s.step(e, t, x, eta=eta, variance_noise=z).prev_sample
    ref = _step64(s, e, x, t, eta, z if eta > 0 else torch.zeros_like(z))
    assert (out.double() - ref).abs().max() < 2e-5 * ref.abs().max()


def test_scheduler_step_noise_semantics():
    s = DDIMScheduler()
    s.set_timesteps(5)
    t = int(s.timesteps[1])
    x, e = torch.randn(1, 4, 2, 8, 8), torch.randn(1, 4, 2, 8, 8)
    # the draw is torch.randn(model_output.shape, generator=generator, device, dtype)
    drawn = s.step(e, t, x, eta=0.7, generator=torch.Generator().manual_seed(5)).prev_sample
    z = torch.randn(e.shape, generator=torch.Generator().manual_seed(5), dtype=e.dtype)
    assert torch.equal(drawn, s.step(e, t, x, eta=0.7, variance_noise=z).prev_sample)
    with pytest.raises(ValueError):
        s.step(e, t, x, eta=0.7, generator=torch.Generator(), variance_noise=z)
    # eta = 0 draws nothing and keeps the deterministic step
    g = torch.Generator().manual_seed(9)
    s.step(e, t, x, eta=0.0, generator=g)
    assert torch.equal(g.get_state(), torch.Generator().manual_seed(9).get_state())


# ---- the pipelines' refusals (nothing here reaches the GPU) -------------------------------------------------------------------------
def cpu_pipe(cls=SpatioTemporalStableDiffusionPipeline):
    unet = UNetPseudo3DConditionModel(**synth.MINI_UNET_CONFIG, **sm.MODEL_CONFIG)
    return cls(sm.EncodingVaeStub(), synth.ToyTextEncoder(128), synth.ToyTokenizer(), unet, DDIMScheduler())


def test_sampler_input_errors():
    pipe = cpu_pipe()
    with pytest.raises(ValueError):
        pipe(prompt=3, height=128, width=128, clip_length=2)
    with pytest.raises(ValueError):
        pipe(prompt="a", height=120, width=128, clip_length=2)  # non-square sides must be multiples of 64
    with pytest.raises(ValueError):
        pipe(prompt="a", height=128, width=128, clip_length=2, latents=torch.zeros(1, 4, 3, 16, 16))
    with pytest.raises(ValueError):
        pipe(prompt=["a", "b"], height=128, width=128, clip_length=2, generator=[torch.Generator()])
    with pytest.raises(ValueError):
        pipe(prompt="a", height=128, width=128, clip_length=33)  # 66 CFG rows > 64
    with pytest.raises(ValueError):
        pipe(prompt="a", height=128, width=128, clip_length=65, guidance_scale=1.0)
    with pytest.raises(ValueError):
        pipe(prompt=["a", "b"], height=128, width=128, clip_length=2, eta=0.5, generator=[torch.Generator(), torch.Generator()])
    with pytest.raises(ValueError):
        pipe(prompt="a", height=128, width=128, clip_length=2, eta=-0.1)
    pipe.unet._engine = SimpleNamespace(shard=(0, 2, None))
    with pytest.raises(NotImplementedError):
        pipe(prompt="a", height=128, width=128, clip_length=2)


def test_ddim_pipeline_input_errors():
    pipe = cpu_pipe(DDIMSpatioTemporalStableDiffusionPipeline)
    image = torch.zeros(2, 3, 128, 128)
    with pytest.raises(ValueError):
        pipe(prompt="a", image=image, guidance_scale=1.0)  # the inversion needs [uncond ; cond]
    with pytest.raises(ValueError):
        pipe(prompt="a", image=image, strength=1.5)
    with pytest.raises(ValueError):
        pipe(prompt="a", image=torch.zeros(34, 3, 128, 128))  # a 34-frame clip: 68 CFG rows
    with pytest.raises(ValueError):
        pipe.prepare_latents_ddim_inverted(torch.zeros(2, 3, 128, 128), 2, 1, torch.zeros(4, 77, 128), generator=[torch.Generator()])
    pipe.unet._engine = SimpleNamespace(shard=(1, 2, None))
    with pytest.raises(NotImplementedError):
        pipe(prompt="a", image=image)


def test_prepare_latents_follows_the_reference():
    pipe = cpu_pipe()
    shape = (2, 4, 3, 16, 16)
    a = pipe.prepare_latents(2, 4, 3, 128, 128, torch.float32, torch.device("cpu"), torch.Generator().manual_seed(1))
    assert torch.equal(a, torch.randn(shape, generator=torch.Generator().manual_seed(1)))
    gens = [torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)]
    b = pipe.prepare_latents(2, 4, 3, 128, 128, torch.float32, torch.device("cpu"), gens)
    assert torch.equal(b[1:], torch.randn((1,) + shape[1:], generator=torch.Generator().manual_seed(2)))
    with pytest.raises(ValueError):
        pipe.prepare_latents(2, 4, 3, 128, 128, torch.float32, torch.device("cpu"), gens[:1])


def test_ddim_alias_module_resolves_to_this_repo():
    from video_diffusion.pipelines.ddim_spatial_temporal import DDIMSpatioTemporalStableDiffusionPipeline as D
    from video_diffusion.pipelines.stable_diffusion import SpatioTemporalStableDiffusionPipeline as S
    assert D is DDIMSpatioTemporalStableDiffusionPipeline and S is SpatioTemporalStableDiffusionPipeline
    assert callable(S.__call__) and issubclass(D, S)


def test_sample_logger_keywords_bind_to_the_ddim_pipeline():
    """The pipeline call of SampleLogger.log_sample_images (validation_loop.py:88-101), keyword for keyword."""
    kw = dict(prompt="a jeep", edit_type=None, image=torch.zeros(8, 3, 512, 512), strength=None, generator=torch.Generator(),
              num_inference_steps=50, clip_length=8, guidance_scale=7.5, num_images_per_prompt=1, latents=None, uncond_embeddings_list=None)
    bound = inspect.signature(DDIMSpatioTemporalStableDiffusionPipeline.__call__).bind(None, **kw)
    assert set(bound.arguments["args"]) == {"edit_type", "uncond_embeddings_list"}
    # text-to-video has the reference's signature, without **kwargs
    params = inspect.signature(SpatioTemporalStableDiffusionPipeline.__call__).parameters
    ref = ["self", "prompt", "height", "width", "num_inference_steps", "clip_length", "guidance_scale", "negative_prompt",
           "num_images_per_prompt", "eta", "generator", "latents", "output_type", "return_dict", "callback", "callback_steps"]
    assert list(params)[:len(ref)] == ref
    assert not any(p.kind == p.VAR_KEYWORD for p in params.values())
