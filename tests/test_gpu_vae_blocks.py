"""The VAE engine (fatezero_b200/vae.py) checked call by call and block by block in fp64, at the image sizes users decode at.

a. Every kernel call of `VaeEngine.encode_moments` / `decode` at the engine's own shapes (SD-1.4 channels, 512x512 and 768x768, and a
   2-image decode so that GroupNorm and the per-image attention loop run with NB > 1): `fatezero_b200.vae.ops` is replaced by CheckedOps,
   which runs each call on the real kernel and checks it right away against tests/_ref64.py (check_tap for 3x3 convs and GEMMs,
   gn_check for GroupNorm, check_probs for the row softmax, exact equality for upsample and the RGB / latent im2col), then drops the
   copies.  Outputs of more than SAMPLE_ABOVE elements are checked on a row sample: the first and last pixel of every row segment, the
   top and bottom image rows, the last tile and random rows.  The number of calls of each kind is asserted, so a path the engine stops
   taking fails loudly.
b. Block semantics: each engine block against VaeBlocks64 (an fp64 restatement of diffusers 0.11.1, independent of oracle/vae_oracle.py)
   on the same fp16 input, on the fp16 floor: the engine may deviate from fp64 at most 1.5 times as much as the same restatement run in
   torch fp16, plus two fp16 ulps.  The weights (vae_block_state_dict) make the mid attention peaked (asserted: median row maximum above
   0.5) and one resnet input has a near-constant group, so that GroupNorm's eps of 1e-6 matters.
c. Image sizes end to end against oracle/vae_oracle.py with the bounds of test_gpu_vae.py: 576, 640 and 768 square, 512x768, the SD-1.4
   channels at 768, and the pipeline's encode / decode of a 2-frame 768 clip.

576, 640 and 768 pixels reach 3x3 convs whose output width is 144, 160, 192, 288, 320 or 576: not a multiple of 128.
"""
import collections
import zlib

import pytest
import torch
import torch.nn.functional as F

from _ref64 import (C_DC, VaeBlocks64, check_block, check_probs, check_tap, conv3x3_rows_ref, f32, gemm_ref, gn_check, softmax64,
                    vae_block_state_dict)

pytestmark = pytest.mark.gpu

from fatezero_b200 import ops, synth  # noqa: E402
from fatezero_b200 import vae as fzvae  # noqa: E402
from oracle import vae_oracle as vo  # noqa: E402

dev = "cuda"
SD14 = dict(vo.SD14_VAE_CONFIG)
SMALL = dict(in_channels=3, out_channels=3, block_out_channels=(32, 64, 128, 128), layers_per_block=2, latent_channels=4, norm_num_groups=32)

SAMPLE_ABOVE = 1 << 24  # output elements above which a call is checked on a row sample
N_RANDOM = 2048         # random rows in a sample


def segment_width(Wo: int) -> int:
    """The 3x3 conv's row-segment width: the largest divisor of Wo up to 128."""
    bw = min(Wo, 128)
    while Wo % bw:
        bw -= 1
    return bw


def image_rows(NB, Ho, Wo, seed):
    """Sampled flat rows of an output [NB, Ho, Wo]: first and last pixel of every row segment, the top and bottom image rows, the last
    tile (128 rows) and N_RANDOM random rows."""
    bw = segment_width(Wo)
    xs = torch.cat([torch.arange(0, Wo, bw), torch.arange(bw - 1, Wo, bw)])
    ny = torch.arange(NB * Ho)[:, None]
    edges = (ny * Wo + xs[None]).flatten()
    tb = torch.cat([(n * Ho + y) * Wo + torch.arange(Wo) for n in range(NB) for y in (0, Ho - 1)])
    M = NB * Ho * Wo
    rand = torch.randint(0, M, (N_RANDOM,), generator=torch.Generator().manual_seed(seed))
    return torch.unique(torch.cat([edges, tb, torch.arange(max(0, M - 128), M), rand]))


def flat_rows(M, seed):
    """Sampled rows of a GEMM output: the first and the last tile and 4 N_RANDOM random rows."""
    rand = torch.randint(0, M, (4 * N_RANDOM,), generator=torch.Generator().manual_seed(seed))
    return torch.unique(torch.cat([torch.arange(min(M, 128)), torch.arange(max(0, M - 128), M), rand]))


def im2col_want(lat):
    """fz_im2col_latents_f16 in torch: latents [B, Cl, F, H, W] fp32 -> [B F H W, 64] fp16, column tap * Cl + c, zero halo and zero pad."""
    B, Cl, Fr, H, W = lat.shape
    xp = F.pad(lat.permute(0, 2, 3, 4, 1).reshape(B * Fr, H, W, Cl), (0, 0, 1, 1, 1, 1))
    taps = torch.stack([xp[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], 3)
    want = torch.zeros(B * Fr * H * W, 64, device=lat.device)
    want[:, :9 * Cl] = taps.reshape(-1, 9 * Cl)
    return want.half()


class CheckedOps:
    """Stands in for fatezero_b200.ops inside fatezero_b200.vae: each call runs on the real kernel, is checked against its fp64 / exact
    reference at once and counted by kind."""

    def __init__(self, report, tag):
        self.report, self.tag = report, tag
        self.counts = collections.Counter()

    def _key(self, kind, shape):
        self.counts[kind] += 1
        return f"{self.tag}/{kind}#{self.counts[kind]}_{'x'.join(map(str, shape))}"

    def conv3x3(self, x, w9, bias=None, stride=1, residual=None, asym_pad=False):
        out = ops.conv3x3(x, w9, bias=bias, stride=stride, residual=residual, asym_pad=asym_pad)
        NB, Ho, Wo, Cout = out.shape
        M = NB * Ho * Wo
        key = self._key("conv3x3_down_asym" if asym_pad else f"conv3x3_s{stride}", (*x.shape, Cout))
        rows = image_rows(NB, Ho, Wo, self.counts.total()) if M * Cout > SAMPLE_ABOVE else torch.arange(M)
        rows = rows.to(out.device)
        res = () if residual is None else (residual.reshape(M, Cout)[rows],)
        ref, terms = conv3x3_rows_ref(x, w9, rows, stride, asym_pad, bias=bias, residuals=res)
        check_tap(out.reshape(M, Cout)[rows], ref, terms, 9 * x.shape[-1] + (bias is not None) + len(res), self.report, key)
        return out

    def gemm(self, a, w, bias=None, residual=None, out=None):
        res_out = ops.gemm(a, w, bias=bias, residual=residual, out=out)
        M, K = a.shape
        N = w.shape[0]
        key = self._key("gemm", (M, N, K))
        rows = (flat_rows(M, self.counts.total()) if M * N > SAMPLE_ABOVE else torch.arange(M)).to(a.device)
        res = () if residual is None else (residual[rows],)
        ref, terms = gemm_ref(a[rows], w, bias=bias, residuals=res)
        check_tap(res_out[:, :N][rows], ref, terms, K + (bias is not None) + len(res), self.report, key)
        return res_out

    def softmax_rows_(self, x, scale):
        rows, n = x.shape
        key = self._key("softmax", (rows, n))
        sel = (flat_rows(rows, self.counts.total()) if rows * n > SAMPLE_ABOVE else torch.arange(rows)).to(x.device)
        x_in = x[sel].clone()
        ops.softmax_rows_(x, scale)
        p = softmax64(x_in.double() * f32(scale))
        del x_in
        check_probs(x[sel], p, self.report, key)
        self.report[key]["median_row_max"] = p.amax(-1).median().item()
        return x

    def groupnorm(self, x, gamma, beta, eps, groups, frames_per_stat, silu):
        out = ops.groupnorm(x, gamma, beta, eps, groups, frames_per_stat, silu)
        gn_check(out, x, gamma, beta, eps, groups, frames_per_stat, silu, self.report, self._key("groupnorm", x.shape), c_dc=C_DC)
        return out

    def upsample2x(self, x):
        out = ops.upsample2x(x)
        self._key("upsample", x.shape)
        assert torch.equal(out, x.repeat_interleave(2, 1).repeat_interleave(2, 2)), "upsample2x differs from nearest 2x"
        return out

    def im2col_latents(self, x):
        out = ops.im2col_latents(x)
        self._key("im2col", x.shape)
        assert torch.equal(out, im2col_want(x)), "im2col_latents differs from the tap-major im2col"
        return out


def expected_calls(cfg, NB, encode):
    """Kernel calls of one encode_moments / decode by kind, from the AutoencoderKL topology."""
    ch, lpb = list(cfg["block_out_channels"]), cfg["layers_per_block"]
    c = collections.Counter(im2col=1, gemm=1)  # the input conv: im2col + GEMM

    def resnet(ci, co):
        c["groupnorm"] += 2
        c["conv3x3_s1"] += 2
        c["gemm"] += int(ci != co)  # 1x1 conv_shortcut

    def mid(cm):
        resnet(cm, cm)
        c["groupnorm"] += 1
        c["gemm"] += 2 + 3 * NB     # fused q|k and proj_attn, per image Q K^T, V^T, P V
        c["softmax"] += NB          # one row softmax per image
        resnet(cm, cm)

    levels = ch if encode else ch[::-1]
    co = levels[0]
    if not encode:
        mid(co)
    for i, cc in enumerate(levels):
        for j in range(lpb if encode else lpb + 1):
            resnet(co if j == 0 else cc, cc)
        co = cc
        if i != len(levels) - 1:
            if encode:
                c["conv3x3_down_asym"] += 1  # one right/bottom-padded downsample per level except the last
            else:
                c["upsample"] += 1
                c["conv3x3_s1"] += 1
    if encode:
        mid(co)
    c["groupnorm"] += 1  # conv_norm_out
    c["conv3x3_s1"] += 1  # conv_out (quant_conv folded in for the encoder)
    return c


@pytest.fixture(scope="module")
def sd14_engine():
    sd = synth.synth_state_dict(dict(fzvae.vae_param_spec(SD14)), seed=3)
    return fzvae.VaeEngine(sd, SD14, torch.device(dev))


@pytest.mark.parametrize("what,size,n", [("encode", 512, 1), ("encode", 768, 1), ("decode", 512, 1), ("decode", 768, 1), ("decode", 512, 2)])
def test_engine_calls_fp64(sd14_engine, what, size, n, report, monkeypatch):
    eng = sd14_engine
    g = torch.Generator().manual_seed(11)
    if what == "encode":
        x = (torch.rand(n, 3, size, size, generator=g) * 2 - 1).to(dev)
        run = eng.encode_moments
    else:
        x = (torch.randn(n, 4, size // 8, size // 8, generator=g) * 0.8).to(dev)
        run = eng.decode
    plain = run(x)
    chk = CheckedOps(report, f"{what}_{size}_n{n}")
    monkeypatch.setattr(fzvae, "ops", chk)
    got = run(x)
    monkeypatch.undo()
    assert torch.equal(got, plain), "the checked run must launch exactly what the plain run launches"
    want = expected_calls(SD14, n, what == "encode")
    assert dict(chk.counts) == dict(want), (dict(chk.counts), dict(want))
    report[f"{what}_{size}_n{n}/calls"] = dict(chk.counts)
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------------- b. blocks
# id, state-dict prefix, VaeBlocks64 / engine method, NCHW input shape
BLOCKS = [
    ("resnet_shortcut_constgroup", "encoder.down_blocks.1.resnets.0", "resnet", (1, 128, 32, 32)),
    ("resnet_128", "decoder.up_blocks.3.resnets.1", "resnet", (1, 128, 48, 64)),
    ("resnet_512_2img", "encoder.mid_block.resnets.0", "resnet", (2, 512, 16, 16)),
    ("attn_encoder_64x64", "encoder.mid_block.attentions.0", "attn", (1, 512, 64, 64)),
    ("attn_decoder_2img_32x48", "decoder.mid_block.attentions.0", "attn", (2, 512, 32, 48)),
    ("down_64x64", "encoder.down_blocks.0.downsamplers.0", "down", (1, 128, 64, 64)),
    ("down_to_192", "encoder.down_blocks.1.downsamplers.0", "down", (1, 256, 8, 384)),
    ("up_16x16", "decoder.up_blocks.0.upsamplers.0", "up", (1, 512, 16, 16)),
    ("up_to_192", "decoder.up_blocks.2.upsamplers.0", "up", (1, 256, 8, 96)),
    ("encoder_in", None, "encoder_in", (1, 3, 64, 64)),
    ("encoder_out", None, "encoder_out", (1, 512, 16, 16)),
    ("decoder_in", None, "decoder_in", (1, 4, 16, 16)),
    ("decoder_out", None, "decoder_out", (1, 128, 64, 64)),
]


@pytest.fixture(scope="module")
def block_weights():
    sd = vae_block_state_dict(fzvae.vae_param_spec(SD14), seed=5)
    return sd, fzvae.VaeEngine(sd, SD14, torch.device(dev))


def block_input(bid, shape):
    g = torch.Generator().manual_seed(zlib.crc32(bid.encode()))
    if bid == "encoder_in":
        return (torch.rand(shape, generator=g) * 2 - 1).half().to(dev)
    x = torch.randn(shape, generator=g) * (0.8 if bid == "decoder_in" else 1.0)
    if "constgroup" in bid:  # GroupNorm group 0 (4 of 128 channels) near-constant: var ~ 1e-6, the size of eps
        x[:, :4] = 1e-3 * torch.randn(shape[0], 4, *shape[2:], generator=g)
    return x.half().to(dev)


def run_engine_block(eng, name, method, x):
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    if method in ("resnet", "attn", "down", "up"):
        y = getattr(eng, "_" + method)(name, nhwc)
    elif method == "encoder_in":
        y = eng._conv_in("encoder.conv_in", x.float())
    elif method == "decoder_in":
        y = eng._decoder_in(x.float())
    else:
        return getattr(eng, "_" + method)(nhwc)  # the heads return NCHW fp32
    return y.permute(0, 3, 1, 2)


@pytest.mark.parametrize("bid,name,method,shape", BLOCKS, ids=[b[0] for b in BLOCKS])
def test_block_vs_fp64_restatement(block_weights, bid, name, method, shape, report):
    sd, eng = block_weights
    x = block_input(bid, shape)
    args = (lambda t: (t,)) if name is None else (lambda t: (name, t))
    probs = [] if method == "attn" else None
    with torch.no_grad():
        ref = getattr(VaeBlocks64(sd, torch.float64, dev), method)(*args(x.double()), **({} if probs is None else dict(probs_out=probs)))
        o16 = getattr(VaeBlocks64(sd, torch.float16, dev), method)(*args(x))
        got = run_engine_block(eng, name, method, x)
    extra = {}
    if probs:
        med = probs[0].amax(-1).median().item()
        extra["median_row_max_prob"] = med
        del probs
        assert med > 0.5, f"attention not peaked (median row maximum {med:.3f}): the block would not tell the probabilities apart"
    check_block(got, ref, o16, report, f"block_{bid}")
    report[f"block_{bid}"].update(extra)


# ------------------------------------------------------------------------------------------------------------- c. image sizes end to end
@pytest.mark.parametrize("cfg_name,n,h,w", [("small", 2, 576, 576), ("small", 1, 640, 640), ("small", 1, 768, 768), ("small", 1, 512, 768),
                                            ("sd14", 1, 768, 768)])
def test_vae_sizes_vs_restatement(cfg_name, n, h, w, report):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = SMALL if cfg_name == "small" else SD14
    sd = synth.synth_state_dict(dict(fzvae.vae_param_spec(cfg)), seed=3)
    eng = fzvae.VaeEngine(sd, cfg, torch.device(dev))
    orc = vo.VaeOracle(sd, cfg).to(dev)
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(n, 3, h, w, generator=g) * 2 - 1).to(dev)
    m_ref, m_got = orc.encode_moments(img), eng.encode_moments(img)
    z = (torch.randn(n, cfg["latent_channels"], h // 8, w // 8, generator=g) * 0.8).to(dev)
    d_ref, d_got = orc.decode(z), eng.decode(z)
    e_enc = (m_got - m_ref).abs().max().item() / max(1.0, m_ref.abs().max().item())
    e_dec = (d_got - d_ref).abs().max().item() / max(1.0, d_ref.abs().max().item())
    report[f"vae_{cfg_name}_{h}x{w}"] = dict(encode_rel=e_enc, decode_rel=e_dec)
    assert e_enc < 4e-3 and e_dec < 4.5e-3  # the bounds of test_gpu_vae.py
    del orc, eng
    torch.cuda.empty_cache()


def test_pipeline_vae_768_clip(report):
    """The pipeline's encode (p2p_ddim_spatial_temporal.py:88-96) and decode_latents (stable_diffusion.py:297-319) of a 2-frame 768x768
    clip run on the engine and give what the engine gives."""
    from _helpers import build_product
    pipe = build_product("mini", dict(lora=160))
    v = fzvae.AutoencoderKL(**SMALL)
    v.load_state_dict(synth.synth_state_dict(dict(fzvae.vae_param_spec(SMALL)), seed=3))
    pipe.vae = v.cuda()
    eng = pipe._vae_engine()
    assert eng is not None
    img = (torch.rand(2, 3, 768, 768, generator=torch.Generator().manual_seed(1)) * 2 - 1).to(dev)
    lat = pipe._vae_encode_sample(img, torch.Generator(device=dev).manual_seed(7))
    assert lat.shape == (2, 4, 96, 96)
    assert torch.equal(lat, fzvae.DiagonalGaussianDistribution(eng.encode_moments(img)).sample(torch.Generator(device=dev).manual_seed(7)))
    video = 0.18215 * lat.reshape(1, 2, 4, 96, 96).permute(0, 2, 1, 3, 4)
    out = pipe.decode_latents(video)
    assert out.shape == (1, 2, 768, 768, 3)
    frames = (1 / 0.18215 * video).permute(0, 2, 1, 3, 4).reshape(2, 4, 96, 96)  # the frames decode_latents hands the engine
    want = (eng.decode(frames) / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).cpu().numpy()
    assert (out[0] == want).all()
