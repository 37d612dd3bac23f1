"""Text-to-video sampling (SpatioTemporalStableDiffusionPipeline.__call__) and the Tune-A-Video DDIM pipeline on the sm_90a kernels.

  * fz_ddim_sample_step against an fp64 restatement (K clips, CFG on / off, eta, the last step, a scalar-path element count), and bitwise
    equal to fz_cfg_ddim_step at cfg = 1, sigma = 0;
  * the reference goldens of oracle/sample.py, free-running and teacher-forced, fed the golden's variance noise;
  * bitwise: every clip of a batched or chunked call == its own call; graph replay == eager at eta = 0 and eta > 0; the DDIM pipeline's
    inversion == P2pDDIMSpatioTemporalPipeline.prepare_latents_ddim_inverted(store_attention=False), and its denoising with the source
    prompt == P2pDDIMSpatioTemporalPipeline(edit_type=None);
  * the draw count of eta > 0 on a seeded CUDA generator; a 512x768 clip and the SD-2-base geometry against the CPU oracle (run on the GPU
    in fp32); a config/tune/jeep.yaml-shaped call sequence end to end."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import os  # noqa: E402

from _helpers import GOLDEN_DIR, synth_weights  # noqa: E402
from fatezero_b200 import ops, synth  # noqa: E402
from fatezero_b200.pipeline import (DDIMSpatioTemporalStableDiffusionPipeline, P2pDDIMSpatioTemporalPipeline,  # noqa: E402
                                    SpatioTemporalStableDiffusionPipeline)
from fatezero_b200.scheduler import DDIMScheduler  # noqa: E402
from fatezero_b200.unet import UNetPseudo3DConditionModel  # noqa: E402
from oracle import fz_oracle as fo  # noqa: E402
from oracle import sample as sm  # noqa: E402

dev = "cuda"

# fz_ddim_sample_step vs fp64: max |got - ref| / max |ref|.  fp32 arithmetic of the same expression (a handful of roundings); measured
# on an H100 SXM 80 GB (700 W): at most 4.5e-7 over every parameter set.
STEP_BOUND = 2e-6
# product (fp16 tensor-core UNet, fp32 DDIM) vs the reference: max |d| / max |x| over all steps.  Teacher-forced: every step starts from
# the oracle's latent (the oracle itself is within 2.1e-5 of the golden), so each carries one step of kernel error; measured (a) 1.4e-3,
# (b) 2.1e-4, (c) 5.0e-3, (d) 2.4e-3.  Free-running against the golden's samples, where the random-weight sampler at CFG 7.5 amplifies
# the error step by step: measured (a) 3.7e-3, (b) 6.3e-4, (c) 1.9e-2, (d) 3.3e-3; the DDIM case's inversion 2.5e-3.  512x768 (mini,
# eta 0.5) and SD-2-base geometry against the oracle after 2 steps: 5.3e-3 and 4.9e-3.  All on an H100 SXM 80 GB (700 W power limit).
TEACHER_BOUND = 1.25e-2
FREE_BOUND = 5e-2
GEOMETRY_BOUND = 1.5e-2


class RowwiseText(synth.ToyTextEncoder):
    """ToyTextEncoder that encodes prompt by prompt, so that a prompt's embedding does not depend on the batch it is encoded in (the
    per-clip invariance tests compare batched calls with single calls)."""

    def forward(self, input_ids, attention_mask=None):
        return (torch.cat([super(RowwiseText, self).forward(input_ids[i:i + 1])[0] for i in range(input_ids.shape[0])]),)


def make_unet(name="mini"):
    cfg = synth.UNET_CONFIGS[name]
    unet = UNetPseudo3DConditionModel(**cfg, **sm.MODEL_CONFIG)
    unet.load_state_dict(synth_weights(name, sm.MODEL_CONFIG))
    return unet.to(dev)


def make_pipe(cls=SpatioTemporalStableDiffusionPipeline, unet=None, name="mini", rowwise=False):
    unet = unet if unet is not None else make_unet(name)
    dim = synth.UNET_CONFIGS[name]["cross_attention_dim"]
    te = (RowwiseText if rowwise else synth.ToyTextEncoder)(dim).to(dev)
    return cls(sm.EncodingVaeStub().to(dev), te, synth.ToyTokenizer(), unet, DDIMScheduler())


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


# ---- the kernel ------------------------------------------------------------------------------------------------------------------------
def ref_step64(x, eps, K, cfg, g, a_t, a_p, eta, z):
    x, eps, z = x.double().cpu(), eps.double().cpu(), z.double().cpu()
    e = eps[:K] + g * (eps[K:] - eps[:K]) if cfg else eps
    sigma = eta * (((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)) ** 0.5
    x0 = (x - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
    return a_p ** 0.5 * x0 + (1 - a_p - sigma ** 2) ** 0.5 * e + sigma * z, sigma


@pytest.mark.parametrize("K", [1, 2, 5])
@pytest.mark.parametrize("cfg", [0, 1])
@pytest.mark.parametrize("eta", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("shape", [(4, 3, 8, 8), (5, 7)], ids=["latents", "odd"])  # (5, 7): 35 per item, not a multiple of 4
@pytest.mark.parametrize("last", [False, True])
def test_sample_step_kernel_vs_fp64(K, cfg, eta, shape, last, report):
    s = DDIMScheduler()
    s.set_timesteps(10)
    t = int(s.timesteps[-1 if last else 3])
    a_t, a_p = s.alpha_pair(t)  # last step: a_p = final_alpha_cumprod
    g = torch.Generator(device=dev).manual_seed(K * 100 + cfg * 10 + int(10 * eta))
    x = torch.randn((K, *shape), generator=g, device=dev)
    eps = torch.randn(((2 if cfg else 1) * K, *shape), generator=g, device=dev)
    z = torch.randn((K, *shape), generator=g, device=dev)
    ref, sigma = ref_step64(x, eps, K, cfg, 7.5, a_t, a_p, eta, z if eta > 0 else torch.zeros_like(z))
    ops.ddim_sample_step(x, eps, 7.5 if cfg else None, a_t, a_p, sigma, z if sigma > 0 else None)
    err = rel(x, ref)
    report.update(err=err)
    assert err <= STEP_BOUND


@pytest.mark.parametrize("K", [1, 3])
def test_sample_step_equals_cfg_ddim_step_bitwise(K):
    s = DDIMScheduler()
    s.set_timesteps(50)
    g = torch.Generator(device=dev).manual_seed(K)
    for t in (int(s.timesteps[0]), int(s.timesteps[25]), int(s.timesteps[-1])):
        a_t, a_p = s.alpha_pair(t)
        x = torch.randn(K, 4, 8, 64, 64, generator=g, device=dev)
        eps = torch.randn(2 * K, 4, 8, 64, 64, generator=g, device=dev)
        y = x.clone()
        if K == 1:
            ops.cfg_ddim_step(x, eps, 7.5, a_t, a_p)
        else:
            ops.cfg_ddim_step_batched(x, eps, 7.5, a_t, a_p)
        ops.ddim_sample_step(y, eps, 7.5, a_t, a_p, 0.0, None)
        assert torch.equal(x, y)


# ---- the reference goldens ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_tf32():
    """The oracle runs on the GPU in fp32: no TF32 in its convolutions and matmuls."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def oracle_trace(c, g):
    """The CPU oracle's sampler (pinned to the golden by tests/test_sample_cpu.py), on the GPU in fp32, from the golden's x_T and noise."""
    from oracle.sd2 import OracleUNetSD2
    cfg = synth.UNET_CONFIGS[c["unet"]]
    cls = OracleUNetSD2 if c["unet"].startswith("sd2") else fo.OracleUNet
    ou = cls(synth_weights(c["unet"], sm.MODEL_CONFIG), cfg, sm.MODEL_CONFIG).to(dev)
    prompts = c["prompt"] if isinstance(c["prompt"], list) else [c["prompt"]]
    neg = c["negative_prompt"] if isinstance(c["negative_prompt"], list) or c["negative_prompt"] is None else [c["negative_prompt"]]
    text = sm.encode_text(synth.ToyTokenizer(), synth.ToyTextEncoder(cfg["cross_attention_dim"]), prompts, neg, c["guidance_scale"] > 1,
                          c["num_images_per_prompt"]).to(dev)
    with torch.no_grad():
        return [v.cpu() for v in sm.sample(ou, g["init"].to(dev), text, c["steps"], c["guidance_scale"], c["eta"],
                                           noise=list(g["noise"]) if c["eta"] > 0 else None)]


def run_golden(name, teacher=None):
    """The case through the reference-facing API; teacher: latents after each step that step i > 0 starts from."""
    c = sm.SAMPLE_CASES[name]
    g = torch.load(os.path.join(GOLDEN_DIR, f"sample_{name}.pt"))
    trace = []
    kw = dict(height=8 * c["size"], width=8 * c["size"], num_inference_steps=c["steps"], clip_length=c["frames"],
              guidance_scale=c["guidance_scale"], negative_prompt=c["negative_prompt"], num_images_per_prompt=c["num_images_per_prompt"],
              eta=c["eta"], output_type="latent", callback=lambda i, t, l: trace.append(l.float().cpu()),
              variance_noise=list(g["noise"]) if c["eta"] > 0 else None, teacher_latents=teacher)
    inv_err = None
    if c["pipeline"] == "t2v":
        out = make_pipe(name=c["unet"])(prompt=c["prompt"], latents=g["init"].to(dev), **kw)
    else:
        pipe = make_pipe(DDIMSpatioTemporalStableDiffusionPipeline, name=c["unet"])
        image = sm.case_image(c).to(dev)
        emb = pipe._encode_prompt(c["source"], dev, 1, True, None)
        pipe.scheduler.set_timesteps(c["steps"])
        inv = pipe.prepare_latents_ddim_inverted(image, 1, 1, emb)
        inv_err = rel(torch.stack([sm.strided(v) for v in inv]), g["inv_sample"])
        out = pipe(prompt=c["prompt"], image=image, latents=(g["init"].to(dev) if teacher is not None else inv[-1]), strength=None,
                   source_prompt=c["source"], edit_type=None, uncond_embeddings_list=None, **kw)
    assert torch.equal(out.images.float().cpu(), trace[-1])
    return trace, g, inv_err


@pytest.mark.parametrize("name", list(sm.SAMPLE_CASES))
def test_pipeline_free_running_matches_reference_golden(name, report):
    trace, g, inv_err = run_golden(name)
    err = (torch.stack([sm.strided(v) for v in trace]) - g["step_sample"]).abs().max().item() / g["abs_max"]
    report.update(err=err, inv_err=inv_err, xmax=g["abs_max"])
    assert err <= FREE_BOUND
    if inv_err is not None:
        assert inv_err <= TEACHER_BOUND


@pytest.mark.parametrize("name", list(sm.SAMPLE_CASES))
def test_pipeline_teacher_forced_matches_reference(name, no_tf32, report):
    """Teacher: the oracle's trajectory from the golden's x_T and noise (held to the golden here too, as on the CPU)."""
    c = sm.SAMPLE_CASES[name]
    g = torch.load(os.path.join(GOLDEN_DIR, f"sample_{name}.pt"))
    ref = oracle_trace(c, g)
    oracle_err = (torch.stack([sm.strided(v) for v in ref]) - g["step_sample"]).abs().max().item() / g["abs_max"]
    trace, _, _ = run_golden(name, teacher=ref)
    err = rel(torch.stack(trace), torch.stack(ref))
    report.update(err=err, oracle_err=oracle_err)
    assert oracle_err <= 1e-4
    assert err <= TEACHER_BOUND


# ---- bitwise properties ------------------------------------------------------------------------------------------------------------
def test_batched_clips_equal_single_clip_calls():
    """Case (a): 2 prompts x 2 clips, CFG, in one UNet call per step == each clip alone."""
    c = sm.SAMPLE_CASES["t2v_cfg_batch"]
    g = torch.load(os.path.join(GOLDEN_DIR, "sample_t2v_cfg_batch.pt"))
    pipe = make_pipe(rowwise=True)
    pipe.graph_mode = "off"
    kw = dict(height=8 * c["size"], width=8 * c["size"], num_inference_steps=c["steps"], clip_length=c["frames"], guidance_scale=7.5,
              output_type="latent")
    batch = pipe(prompt=c["prompt"], negative_prompt=c["negative_prompt"], num_images_per_prompt=2, latents=g["init"].to(dev), **kw).images
    for k in range(4):
        p = k // 2
        one = pipe(prompt=[c["prompt"][p]], negative_prompt=[c["negative_prompt"][p]], latents=g["init"][k:k + 1].to(dev), **kw).images
        assert torch.equal(batch[k:k + 1], one), k


def test_chunked_batch_equals_single_clip_calls():
    """5 clips of 8 frames under CFG (80 attention rows) run as UNet calls of 4 + 1 clips; eta > 0 with the noise given."""
    pipe = make_pipe(rowwise=True)
    pipe.graph_mode = "off"
    prompts = [f"clip number {k} of a jeep" for k in range(5)]
    gen = torch.Generator(device=dev).manual_seed(3)
    init = torch.randn(5, 4, 8, 32, 32, generator=gen, device=dev)
    noise = [torch.randn(5, 4, 8, 32, 32, generator=gen, device=dev) for _ in range(2)]
    kw = dict(height=256, width=256, num_inference_steps=2, clip_length=8, guidance_scale=7.5, eta=0.5, output_type="latent")
    batch = pipe(prompt=prompts, latents=init, variance_noise=noise, **kw).images
    for k in range(5):
        one = pipe(prompt=[prompts[k]], latents=init[k:k + 1], variance_noise=[z[k:k + 1] for z in noise], **kw).images
        assert torch.equal(batch[k:k + 1], one), k


@pytest.mark.parametrize("eta", [0.0, 0.7])
def test_graph_replay_equals_eager(eta):
    pipe = make_pipe()
    kw = dict(prompt=["a jeep", "a car"], height=256, width=256, num_inference_steps=4, clip_length=4, guidance_scale=7.5, eta=eta,
              output_type="latent")
    outs = []
    for _ in range(3):  # eager (configuration seen), captured + replayed, replayed
        outs.append(pipe(generator=torch.Generator(device=dev).manual_seed(21), **kw).images)
    assert len(pipe._plans) == 1
    pipe.graph_mode = "off"
    eager = pipe(generator=torch.Generator(device=dev).manual_seed(21), **kw).images
    for o in outs:
        assert torch.equal(o, eager)


def test_generator_draw_count_and_order():
    pipe = make_pipe()
    gen = torch.Generator(device=dev).manual_seed(77)
    for graph_mode in ("off", "auto", "auto"):
        pipe.graph_mode = graph_mode
        gen.manual_seed(77)
        pipe(prompt="a jeep", height=256, width=256, num_inference_steps=3, clip_length=2, eta=1.0, generator=gen, output_type="latent")
        got = torch.randn(16, generator=gen, device=dev)
        # the reference's draws: the initial latents (stable_diffusion.py:503-513), then one DDIMScheduler.step draw per step
        ref = torch.Generator(device=dev).manual_seed(77)
        torch.randn((1, 4, 2, 32, 32), generator=ref, device=dev)
        for _ in range(3):
            torch.randn((1, 4, 2, 32, 32), generator=ref, device=dev)
        assert torch.equal(got, torch.randn(16, generator=ref, device=dev)), graph_mode


def test_ddim_pipeline_equals_p2p_paths():
    c = sm.SAMPLE_CASES["ddim_invert_edit"]
    unet = make_unet()
    ddim = make_pipe(DDIMSpatioTemporalStableDiffusionPipeline, unet=unet)
    p2p = make_pipe(P2pDDIMSpatioTemporalPipeline, unet=unet)
    image = sm.case_image(c).to(dev)
    emb = ddim._encode_prompt(c["source"], dev, 1, True, None)
    for p in (ddim, p2p):
        p.scheduler.set_timesteps(c["steps"])
    a = ddim.prepare_latents_ddim_inverted(image, 1, 1, emb)
    b = p2p.prepare_latents_ddim_inverted(image, 1, 1, emb, store_attention=False)
    assert len(a) == len(b) == c["steps"] + 1
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    kw = dict(prompt=c["source"], num_inference_steps=c["steps"], clip_length=c["frames"], guidance_scale=7.5, latents=a[-1],
              output_type="latent", height=8 * c["size"], width=8 * c["size"])
    x = ddim(image=image, **kw).images
    y = p2p(edit_type=None, source_prompt=c["source"], image=image, **kw).images
    assert torch.equal(x, y)


# ---- larger geometries against the oracle ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unet_name,h,w,eta", [("mini", 512, 768, 0.5), ("sd2", 256, 256, 0.0)])
def test_geometry_matches_oracle(unet_name, h, w, eta, no_tf32, report):
    from oracle.sd2 import OracleUNetSD2
    cfg = synth.UNET_CONFIGS[unet_name]
    pipe = make_pipe(name=unet_name)
    gen = torch.Generator(device=dev).manual_seed(5)
    init = torch.randn(1, 4, 2, h // 8, w // 8, generator=gen, device=dev)
    noise = [torch.randn(1, 4, 2, h // 8, w // 8, generator=gen, device=dev) for _ in range(2)]
    out = pipe(prompt="a jeep", height=h, width=w, num_inference_steps=2, clip_length=2, guidance_scale=7.5, eta=eta, latents=init,
               variance_noise=noise if eta > 0 else None, output_type="latent").images
    cls = OracleUNetSD2 if unet_name.startswith("sd2") else fo.OracleUNet
    ou = cls(synth_weights(unet_name, sm.MODEL_CONFIG), cfg, sm.MODEL_CONFIG).to(dev)
    text = sm.encode_text(synth.ToyTokenizer(), synth.ToyTextEncoder(cfg["cross_attention_dim"]), ["a jeep"], None, True).to(dev)
    with torch.no_grad():
        ref = sm.sample(ou, init, text, 2, 7.5, eta, noise=noise)[-1]
    err = rel(out, ref)
    report.update(err=err)
    assert err <= GEOMETRY_BOUND


def test_tune_config_call_sequence():
    """config/tune/jeep.yaml through train_tune_a_video.py:361-385 and validation_loop.py:86-101: _encode_prompt, one inversion, then one
    __call__ per editing prompt with the logger's keywords, PIL output."""
    pipe = make_pipe(DDIMSpatioTemporalStableDiffusionPipeline)
    pipe.scheduler.set_timesteps(3)
    images = sm.case_image(dict(seed=1, frames=8, size=32)).to(dev)
    emb = pipe._encode_prompt(sm.SRC, dev, 1, True, None)
    lat = pipe.prepare_latents_ddim_inverted(images, batch_size=1, num_images_per_prompt=1, text_embeddings=emb)
    for prompt in (sm.SRC, "a jeep in the snow"):
        out = pipe(prompt=prompt, edit_type=None, image=images, strength=None, generator=torch.Generator(device=dev).manual_seed(0),
                   num_inference_steps=3, clip_length=8, guidance_scale=7.5, num_images_per_prompt=1, latents=lat[-1],
                   uncond_embeddings_list=None)
        frames = out.images[0]
        assert len(frames) == 8 and frames[0].size == (256, 256)
