"""VAE encode / decode on the sm_90a kernels (fatezero_b200/vae.py) against the fp32 torch restatement oracle/vae_oracle.py on the same
name-keyed synthetic weights.  NOTE (DESIGN.md §5): that restatement is NOT pinned to the real diffusers package (absent offline), so this
is parity of two independent restatements of the published AutoencoderKL; bounds are fp16-storage bounds, 2x the measured values."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from fatezero_b200 import synth  # noqa: E402
from fatezero_b200 import vae as fzvae  # noqa: E402
from oracle import vae_oracle as vo  # noqa: E402

SMALL = dict(in_channels=3, out_channels=3, block_out_channels=(32, 64, 128, 128), layers_per_block=2, latent_channels=4, norm_num_groups=32)


def _weights(cfg):
    spec = fzvae.vae_param_spec(cfg)
    assert {k: tuple(v) for k, v in spec.items()} == {k: tuple(v) for k, v in vo.vae_param_spec(cfg).items()}  # product and oracle agree on the layout
    return synth.synth_state_dict(dict(spec), seed=3)


@pytest.mark.parametrize("cfg_name,n,size", [("small", 2, 128), ("sd14", 1, 256), ("sd14", 1, 512)])
def test_vae_encode_decode_vs_restatement(cfg_name, n, size, report):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = SMALL if cfg_name == "small" else dict(vo.SD14_VAE_CONFIG)
    sd = _weights(cfg)
    eng = fzvae.VaeEngine(sd, cfg, torch.device("cuda"))
    orc = vo.VaeOracle(sd, cfg).to("cuda")
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(n, 3, size, size, generator=g) * 2 - 1).cuda()
    m_ref = orc.encode_moments(img)
    m_got = eng.encode_moments(img)
    z = (torch.randn(n, cfg["latent_channels"], size // 8, size // 8, generator=g) * 0.8).cuda()
    d_ref = orc.decode(z)
    d_got = eng.decode(z)
    e_enc = (m_got - m_ref).abs().max().item() / max(1.0, m_ref.abs().max().item())
    e_dec = (d_got - d_ref).abs().max().item() / max(1.0, d_ref.abs().max().item())
    report[f"vae_{cfg_name}_{size}"] = dict(encode_rel=e_enc, decode_rel=e_dec, moments_abs_max=m_ref.abs().max().item(), image_abs_max=d_ref.abs().max().item())
    print(f"\nVAE {cfg_name} {size}x{size}: encode rel {e_enc:.3e} (max|m| {m_ref.abs().max().item():.2f}), decode rel {e_dec:.3e} (max|x| {d_ref.abs().max().item():.2f})")
    assert e_enc < 4e-3 and e_dec < 4.5e-3  # measured 1.5e-3 .. 2.0e-3 (fp16 activations through ~30 convs)


def test_pipeline_brackets_with_the_engine(report):
    """prepare_latents_ddim_inverted / decode_latents route an AutoencoderKL-shaped `vae` through the engine (p2p_ddim_spatial_temporal.py:88-96,
    stable_diffusion.py:297-319): images -> latents -> images keeps shapes, scaling and the generator-driven sampling."""
    import sys
    sys.path.insert(0, __file__.rsplit("/", 1)[0])
    from _helpers import build_product
    pipe = build_product("mini", dict(lora=160))
    v = fzvae.AutoencoderKL(**SMALL)
    v.load_state_dict(_weights(SMALL))
    pipe.vae = v.cuda()
    assert pipe._vae_engine() is not None
    img = (torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)) * 2 - 1).cuda()
    gen = torch.Generator(device="cuda").manual_seed(7)
    lat = pipe._vae_encode_sample(img, gen)
    assert lat.shape == (2, 4, 16, 16)
    dist = v.encode(img).latent_dist
    gen2 = torch.Generator(device="cuda").manual_seed(7)
    assert torch.equal(lat, dist.sample(gen2))
    out = pipe.decode_latents(0.18215 * lat.reshape(1, 2, 4, 16, 16).permute(0, 2, 1, 3, 4))
    assert out.shape == (1, 2, 128, 128, 3) and out.min() >= 0 and out.max() <= 1
