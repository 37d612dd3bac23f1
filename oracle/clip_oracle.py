"""fp32 restatement of OpenAI CLIP's ViT model (the network FateZero's evaluation calls, CLIP/clip/model.py) and of its preprocess
(CLIP/clip/clip.py:79-86) for the CLIP-evaluation tests, plus the deterministic weights and frames those tests share with
tests/golden/clip_vitb32.pt.  Parameter names and shapes are the OpenAI state-dict layout, so `ClipOracle.state_dict()` loads into
fatezero_b200.clip_eval.ClipEvaluator and the module can be traced into a TorchScript archive like OpenAI's ViT-B-32.pt."""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

# CLIP(embed_dim, image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size, transformer_width,
#      transformer_heads, transformer_layers) of ViT-B/32
VITB32 = (512, 224, 12, 768, 32, 77, 49408, 512, 8, 12)
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


class _Block(nn.Module):
    def __init__(self, width: int, heads: int, causal: bool, ctx: int):
        super().__init__()
        self.heads, self.causal = heads, causal
        self.ln_1 = nn.LayerNorm(width)
        self.attn = nn.Module()
        self.attn.in_proj_weight = nn.Parameter(torch.empty(3 * width, width))
        self.attn.in_proj_bias = nn.Parameter(torch.empty(3 * width))
        self.attn.out_proj = nn.Linear(width, width)
        self.ln_2 = nn.LayerNorm(width)
        self.mlp = nn.Module()
        self.mlp.c_fc = nn.Linear(width, 4 * width)
        self.mlp.c_proj = nn.Linear(4 * width, width)

    def forward(self, x):  # [B, L, C]
        B, L, C = x.shape
        h = self.ln_1(x)
        q, k, v = F.linear(h, self.attn.in_proj_weight, self.attn.in_proj_bias).split(C, dim=-1)
        d = C // self.heads
        q, k, v = (t.reshape(B, L, self.heads, d).transpose(1, 2) for t in (q, k, v))
        s = (q @ k.transpose(-1, -2)) * d ** -0.5
        if self.causal:
            s = s + torch.full((L, L), float("-inf"), dtype=s.dtype, device=s.device).triu(1)
        o = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, L, C)
        x = x + self.attn.out_proj(o)
        m = self.mlp.c_fc(self.ln_2(x))
        return x + self.mlp.c_proj(m * torch.sigmoid(1.702 * m))


class _Tower(nn.Module):
    def __init__(self, width, layers, heads, causal, ctx):
        super().__init__()
        self.resblocks = nn.Sequential(*[_Block(width, heads, causal, ctx) for _ in range(layers)])


class ClipOracle(nn.Module):
    def __init__(self, embed_dim=512, image_resolution=224, vision_layers=12, vision_width=768, patch=32, context_length=77,
                 vocab_size=49408, transformer_width=512, transformer_heads=8, transformer_layers=12):
        super().__init__()
        g = image_resolution // patch
        self.visual = nn.Module()
        self.visual.conv1 = nn.Conv2d(3, vision_width, patch, patch, bias=False)
        self.visual.class_embedding = nn.Parameter(torch.empty(vision_width))
        self.visual.positional_embedding = nn.Parameter(torch.empty(g * g + 1, vision_width))
        self.visual.ln_pre = nn.LayerNorm(vision_width)
        self.visual.transformer = _Tower(vision_width, vision_layers, vision_width // 64, False, g * g + 1)
        self.visual.ln_post = nn.LayerNorm(vision_width)
        self.visual.proj = nn.Parameter(torch.empty(vision_width, embed_dim))
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, transformer_width))
        self.transformer = _Tower(transformer_width, transformer_layers, transformer_heads, True, context_length)
        self.ln_final = nn.LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]))

    def encode_image(self, image):
        v = self.visual
        x = v.conv1(image.to(v.conv1.weight.dtype)).flatten(2).transpose(1, 2)
        x = torch.cat([v.class_embedding.expand(x.shape[0], 1, -1), x], 1) + v.positional_embedding
        x = v.transformer.resblocks(v.ln_pre(x))
        return v.ln_post(x[:, 0]) @ v.proj

    def encode_text(self, ids):
        x = self.token_embedding(ids) + self.positional_embedding
        x = self.ln_final(self.transformer.resblocks(x))
        return x[torch.arange(x.shape[0]), ids.argmax(-1)] @ self.text_projection

    def forward(self, image, ids):
        a, b = self.encode_image(image), self.encode_text(ids)
        a = a / a.norm(dim=1, keepdim=True)
        b = b / b.norm(dim=1, keepdim=True)
        li = self.logit_scale.exp() * a @ b.t()
        return li, li.t()


def synth_clip_state_dict(seed: int = 0, shapes=None):
    """fatezero_b200.synth weights under the OpenAI names and shapes of ViT-B/32, logit_scale = ln 100."""
    from fatezero_b200 import synth
    if shapes is None:
        with torch.device("meta"):
            shapes = {k: tuple(v.shape) for k, v in ClipOracle(*VITB32).state_dict().items()}
    sd = {k: synth.synth_tensor(k, s, seed) for k, s in sorted(shapes.items())}
    sd["logit_scale"] = torch.tensor(math.log(100.0))
    return sd


def oracle_model(seed: int = 0) -> ClipOracle:
    m = ClipOracle(*VITB32)
    m.load_state_dict(synth_clip_state_dict(seed))
    return m.eval().requires_grad_(False)


def crop_read(img):
    """frame_acc_tem_con.py:11-16 on a PIL image: a frame with h > w keeps its bottom w x w square."""
    w, h = img.size
    return img.crop((0, h - w, w, h)) if h > w else img


def preprocess(img, n_px: int = 224) -> torch.Tensor:
    """Resize(n_px, BICUBIC) + CenterCrop + ToTensor + Normalize of a PIL RGB image -> [3, n_px, n_px] fp32."""
    import torchvision.transforms as T
    t = T.Compose([T.Resize(n_px, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(n_px), T.ToTensor(), T.Normalize(MEAN, STD)])
    return t(img.convert("RGB"))


def _frame(h: int, w: int, t: float, rng: np.random.Generator) -> np.ndarray:
    """Smooth gradients, flat patches and hard-edged saturated shapes (ringing of the cubic filter clips at 0 and 255)."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3))
    img[..., 0] = 127 + 120 * np.sin(2 * np.pi * (xx / w * 1.5 + t))
    img[..., 1] = 255 * (yy / max(h - 1, 1))
    img[..., 2] = 127 + 100 * np.cos(2 * np.pi * (xx + yy) / (w + h) * 3 - t)
    img[: h // 4, : w // 4] = (30, 200, 90)                                     # flat
    cx, cy = w * (0.5 + 0.2 * np.sin(2 * np.pi * t)), h * 0.55
    disk = (xx - cx) ** 2 + (yy - cy) ** 2 < (0.18 * min(h, w)) ** 2
    img[disk] = (255, 255, 255)                                                 # hard edge, saturated
    bars = ((xx // max(w // 40, 1)) % 2 == 0) & (yy > 0.8 * h)
    img[bars] = (0, 0, 0)
    img += rng.normal(0, 6, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def synth_clip_frames() -> dict:
    """name -> uint8 [F, H, W, 3]: an 8-frame 512x512 clip and single frames at 640x360, 360x640 (bottom-square crop), 150x100 (upscale)
    and 224x224 (width x height)."""
    rng = np.random.default_rng(20260)
    out = {"clip512": np.stack([_frame(512, 512, i / 8, rng) for i in range(8)])}
    for name, (w, h) in (("w640h360", (640, 360)), ("w360h640", (360, 640)), ("w150h100", (150, 100)), ("w224h224", (224, 224))):
        out[name] = _frame(h, w, 0.3, rng)[None]
    return out


def array_sha256(a: np.ndarray) -> str:
    """Digest of an array's shape, dtype and bytes."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.shape}{a.dtype}".encode() + a.tobytes()).hexdigest()


def frames_sha256(frames: dict) -> str:
    h = hashlib.sha256()
    for k in sorted(frames):
        h.update(k.encode())
        h.update(np.ascontiguousarray(frames[k]).tobytes())
    return h.hexdigest()
