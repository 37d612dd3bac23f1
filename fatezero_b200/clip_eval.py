"""CLIP scoring of edited clips on the sm_90a kernels: the reference's evaluation (CLIP/frame_acc_tem_con.py) without leaving the device.

For every frame the reference asks a CLIP ViT-B/32 whether the frame matches the target prompt better than the source prompt ("frame
accuracy", the two-way softmax of `logit_scale.exp() * cos` at CLIP/clip/model.py:358-372) and averages the cosine similarity of the image
features of consecutive frames ("temporal consistency", frame_acc_tem_con.py:35-54).  `ClipEvaluator` computes both from uint8 frames on the
GPU:
  * frame read (frame_acc_tem_con.py:11-16: a frame with h > w is cropped to its bottom w x w square) and Resize(224, BICUBIC) as Pillow's
    fixed-point two-pass resample: `fz_resize_bicubic_u8` with the coefficient tables of `resize_tables` (computed here, on the host);
  * CenterCrop + ToTensor + Normalize (CLIP/clip/clip.py:79-86) rounded to fp16 and written as conv1's im2col rows: `fz_clip_patchify_f16`;
  * the image tower (model.py:206-238): conv1 on `fz_gemm_f16`, class token + positional embedding + ln_pre in `fz_clip_embed_f16`, the
    residual blocks of `clip.transformer_blocks` (non-causal, 50 tokens), ln_post on the class tokens, `@ proj` on `fz_gemm_f16`;
  * the text tower (model.py:343-356): the same blocks with the causal mask, ln_final on the first end-of-text position, `@ text_projection`;
  * the scoring head `fz_clip_scores`: norms, logits, probabilities, success flags, margins, consecutive-frame cosines, per-clip means.
fp16 storage with fp32 accumulation in the towers (the reference runs the whole model in fp16), fp32 features and statistics.
"""
from __future__ import annotations

import glob
import math
import os
import sys
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from .clip import transformer_blocks

f16, f32 = torch.float16, torch.float32

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
# fz_attention_f16 copies its per-row K/V source table into the kernel's parameter block, which holds at most 64 rows (BF <= 64): the towers
# run in chunks of at most 64 images (or prompts).
MAX_ATTN_ROWS = 64
MAX_CLIPS_PER_LAUNCH = 256  # FZ_CLIP_MAX_CLIPS
PRECISION_BITS = 22  # Pillow's 8-bit resample: 32 - 8 - 2


# ---------------------------------------------------------------------------------------------------------------------------------------
# Pillow's bicubic resample (libImaging/Resample.c), host side
# ---------------------------------------------------------------------------------------------------------------------------------------
def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def resize_coeffs(in_size: int, out_size: int):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the a = -0.5 cubic: int32 weights [out_size, ksize] with 22 fractional bits
    and int32 (first input pixel, tap count) [out_size, 2]."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resize {in_size} -> {out_size}")
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    k = np.zeros((out_size, ksize), dtype=np.int32)
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = sum(w)
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            k[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return k, bounds


def resample_numpy(img: np.ndarray, size) -> np.ndarray:
    """uint8 [H, W, C] -> [h, w, C] with Pillow's two-pass 8-bit bicubic (horizontal pass first, uint8 in between); size = (w, h)."""
    w, h = size
    H, W = img.shape[:2]

    def one_pass(x, kk, bb, axis):
        x = np.moveaxis(x.astype(np.int64), axis, 0)
        acc = np.full((kk.shape[0],) + x.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
        for o in range(kk.shape[0]):
            s, n = bb[o]
            acc[o] += np.tensordot(kk[o, :n].astype(np.int64), x[s:s + n], axes=(0, 0))
        return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)

    out = img
    if w != W:
        out = one_pass(out, *resize_coeffs(W, w), axis=1)
    if h != H:
        out = one_pass(out, *resize_coeffs(H, h), axis=0)
    return out


def resized_size(w: int, h: int, n_px: int = 224):
    """torchvision Resize(n_px) on a PIL image: the short side becomes n_px, the long side int(n_px * long / short); returns (w, h)."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = n_px, int(n_px * long / short)
    return (new_short, new_long) if w <= h else (new_long, new_short)


def frame_read_size(w: int, h: int):
    """frame_acc_tem_con.py:11-16: (w, h) after the bottom-square crop of a frame with h > w."""
    return (w, w) if h > w else (w, h)


def resize_tables(w: int, h: int, n_px: int, device) -> dict:
    """Device tables of fz_resize_bicubic_u8 for a (cropped) w x h frame."""
    wo, ho = resized_size(w, h, n_px)
    kx, bx = resize_coeffs(w, wo)
    ky, by = resize_coeffs(h, ho)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
    return dict(kx=t(kx), bx=t(bx), ky=t(ky), by=t(by))


# ---------------------------------------------------------------------------------------------------------------------------------------
# OpenAI CLIP state dicts
# ---------------------------------------------------------------------------------------------------------------------------------------
def parse_state_dict(sd: Dict[str, torch.Tensor]) -> dict:
    """Geometry of an OpenAI-layout CLIP state dict (CLIP/clip/model.py:400-430 build_model).  Only the ViT image tower is supported."""
    if "visual.proj" not in sd:
        found = sorted({k.split(".")[1] for k in sd if k.startswith("visual.")})[:6]
        raise NotImplementedError(f"only ViT CLIP image towers are supported; this state dict has a ResNet-style image tower "
                                  f"(visual.* entries {found}, no visual.proj)")
    need = ["visual.conv1.weight", "visual.class_embedding", "visual.positional_embedding", "visual.ln_pre.weight", "visual.ln_pre.bias",
            "visual.ln_post.weight", "visual.ln_post.bias", "token_embedding.weight", "positional_embedding", "ln_final.weight",
            "ln_final.bias", "text_projection", "logit_scale"]
    missing = [k for k in need if k not in sd]
    if missing:
        raise KeyError(f"CLIP state dict lacks {missing}")
    conv = sd["visual.conv1.weight"]
    if conv.dim() != 4 or conv.shape[1] != 3 or conv.shape[2] != conv.shape[3]:
        raise NotImplementedError(f"visual.conv1.weight of shape {tuple(conv.shape)}: only square RGB patches are supported")
    width, patch = int(conv.shape[0]), int(conv.shape[-1])
    tokens = int(sd["visual.positional_embedding"].shape[0])
    grid = int(round((tokens - 1) ** 0.5))
    if grid * grid + 1 != tokens:
        raise NotImplementedError(f"visual.positional_embedding has {tokens} rows: not a square patch grid plus a class token")

    def count(prefix):
        return len({k.split(".")[len(prefix.split(".")) - 1] for k in sd if k.startswith(prefix)})

    g = dict(width=width, patch=patch, grid=grid, resolution=grid * patch, vision_layers=count("visual.transformer.resblocks."),
             vision_heads=width // 64, embed_dim=int(sd["text_projection"].shape[1]), context_length=int(sd["positional_embedding"].shape[0]),
             vocab_size=int(sd["token_embedding.weight"].shape[0]), text_width=int(sd["ln_final.weight"].shape[0]),
             text_layers=count("transformer.resblocks."))
    g["text_heads"] = g["text_width"] // 64
    if int(sd["visual.proj"].shape[1]) != g["embed_dim"]:
        raise ValueError(f"visual.proj {tuple(sd['visual.proj'].shape)} does not project to the text embedding width {g['embed_dim']}")
    for tower, pre in (("vision", "visual.transformer.resblocks."), ("text", "transformer.resblocks.")):
        for i in range(g[tower + "_layers"]):
            for s in ("ln_1.weight", "ln_1.bias", "attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight", "attn.out_proj.bias",
                      "ln_2.weight", "ln_2.bias", "mlp.c_fc.weight", "mlp.c_fc.bias", "mlp.c_proj.weight", "mlp.c_proj.bias"):
                if f"{pre}{i}.{s}" not in sd:
                    raise KeyError(f"CLIP state dict lacks {pre}{i}.{s}")
    return g


def load_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """A plain state-dict file (torch.save) or a TorchScript archive such as OpenAI's ViT-B-32.pt, read on the CPU."""
    try:
        return {k: v for k, v in torch.jit.load(path, map_location="cpu").state_dict().items()}
    except RuntimeError:
        obj = torch.load(path, map_location="cpu", weights_only=True)
        return dict(obj.get("state_dict", obj)) if isinstance(obj, dict) else obj


def _default_tokenize() -> Callable:
    """OpenAI `clip.tokenize`, from an installed `clip` package or the reference checkout ($FATEZERO_REFERENCE_ROOT/CLIP)."""
    root = os.environ.get("FATEZERO_REFERENCE_ROOT")
    if root and os.path.isdir(os.path.join(root, "CLIP", "clip")) and os.path.join(root, "CLIP") not in sys.path:
        sys.path.append(os.path.join(root, "CLIP"))
    try:
        import clip  # noqa: F401
        return clip.tokenize
    except ImportError as e:
        raise RuntimeError("string prompts need a tokenizer: fatezero_b200 ships no BPE vocabulary; install OpenAI CLIP, set "
                           "FATEZERO_REFERENCE_ROOT to a FateZero checkout, or pass tokenize= (a callable list[str] -> int64 [P, 77])") from e


Frames = Union[torch.Tensor, Sequence, str]


class ClipEvaluator:
    """CLIP ViT on the sm_90a kernels plus the reference's two edit metrics.  Build with `from_state_dict` or `load`."""

    def __init__(self, sd: Dict[str, torch.Tensor], device="cuda", tokenize: Optional[Callable] = None):
        self.geom = g = parse_state_dict(sd)
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("ClipEvaluator runs on the sm_90a kernels and needs a CUDA device (there is no CPU path)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.dev = dev
        self.tokenize = tokenize
        self.eps = 1e-5  # CLIP/clip/model.py LayerNorm: nn.LayerNorm's default

        def h(t):
            return t.detach().to(dev, f16).contiguous()

        def f(t):
            return t.detach().to(dev, f32).contiguous()

        def blocks(prefix, n):
            out = []
            for i in range(n):
                q = f"{prefix}{i}."
                out.append(dict(ln1=(f(sd[q + "ln_1.weight"]), f(sd[q + "ln_1.bias"])), ln2=(f(sd[q + "ln_2.weight"]), f(sd[q + "ln_2.bias"])),
                                qkv_w=h(sd[q + "attn.in_proj_weight"]), qkv_b=f(sd[q + "attn.in_proj_bias"]),
                                out_w=h(sd[q + "attn.out_proj.weight"]), out_b=f(sd[q + "attn.out_proj.bias"]),
                                fc1_w=h(sd[q + "mlp.c_fc.weight"]), fc1_b=f(sd[q + "mlp.c_fc.bias"]),
                                fc2_w=h(sd[q + "mlp.c_proj.weight"]), fc2_b=f(sd[q + "mlp.c_proj.bias"])))
            return out

        self.conv_w = h(sd["visual.conv1.weight"].reshape(g["width"], -1))
        self.cls = f(sd["visual.class_embedding"])
        self.v_pos = f(sd["visual.positional_embedding"])
        self.ln_pre = (f(sd["visual.ln_pre.weight"]), f(sd["visual.ln_pre.bias"]))
        self.v_layers = blocks("visual.transformer.resblocks.", g["vision_layers"])
        self.ln_post = (f(sd["visual.ln_post.weight"]), f(sd["visual.ln_post.bias"]))
        self.v_proj = h(sd["visual.proj"].t())
        self.tok = f(sd["token_embedding.weight"])
        self.t_pos = f(sd["positional_embedding"])
        self.t_layers = blocks("transformer.resblocks.", g["text_layers"])
        self.ln_final = (f(sd["ln_final.weight"]), f(sd["ln_final.bias"]))
        self.t_proj = h(sd["text_projection"].t())
        # model.py:366 `self.logit_scale.exp()` on the fp32 parameter (convert_weights leaves it in fp32)
        self.logit_scale = float(sd["logit_scale"].detach().float().cpu().exp())
        self._tables = {}

    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], device="cuda", tokenize: Optional[Callable] = None) -> "ClipEvaluator":
        return cls(sd, device, tokenize)

    @classmethod
    def load(cls, path: str, device="cuda", tokenize: Optional[Callable] = None) -> "ClipEvaluator":
        return cls(load_state_dict(path), device, tokenize)

    # ---- the reference's own surface (model.py) -----------------------------------------------------------------------------------------
    @torch.no_grad()
    def preprocess_u8(self, frames: torch.Tensor, crop_bottom_square: bool = False) -> torch.Tensor:
        """Device uint8 frames [N, H, W, 3] -> Resize + CenterCrop + ToTensor + Normalize (clip.py:79-86) as fp16 conv1 im2col rows
        [N * grid^2, 3 * patch^2]; crop_bottom_square applies the frame read of frame_acc_tem_con.py:11-16 first."""
        if frames.dim() != 4 or frames.shape[-1] != 3 or frames.dtype != torch.uint8:
            raise ValueError(f"preprocess_u8 expects uint8 [N, H, W, 3] frames, got {frames.dtype} {tuple(frames.shape)}")
        g = self.geom
        frames = frames.to(self.dev).contiguous()
        _, H, W, _ = frames.shape
        w, h = frame_read_size(W, H) if crop_bottom_square else (W, H)
        key = (w, h)
        if key not in self._tables:
            self._tables[key] = resize_tables(w, h, g["resolution"], self.dev)
        with torch.cuda.device(self.dev):
            r = ops.resize_bicubic_u8(frames, self._tables[key], crop_bottom_square=crop_bottom_square)
            return ops.clip_patchify(r, g["resolution"], g["patch"], CLIP_MEAN, CLIP_STD)

    def _patches(self, pixels: torch.Tensor) -> torch.Tensor:
        g = self.geom
        if pixels.dim() == 2:
            return pixels.to(self.dev, f16).contiguous()
        N, P, G = pixels.shape[0], g["patch"], g["grid"]
        if tuple(pixels.shape[1:]) != (3, g["resolution"], g["resolution"]):
            raise ValueError(f"pixels {tuple(pixels.shape)}: expected [N, 3, {g['resolution']}, {g['resolution']}] or preprocess_u8 rows")
        x = pixels.to(self.dev, f16).reshape(N, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5)
        return x.reshape(N * G * G, 3 * P * P).contiguous()

    @torch.no_grad()
    def encode_image(self, pixels: torch.Tensor) -> torch.Tensor:
        """model.py:338-340: normalised pixels [N, 3, R, R] (or preprocess_u8's rows) -> image features [N, embed_dim] fp32."""
        g = self.geom
        x = self._patches(pixels)
        T, g2, C = g["grid"] ** 2 + 1, g["grid"] ** 2, g["width"]
        N = x.shape[0] // g2
        outs = []
        with torch.cuda.device(self.dev):
            for s in range(0, N, MAX_ATTN_ROWS):
                n = min(MAX_ATTN_ROWS, N - s)
                e = ops.gemm(x[s * g2:(s + n) * g2], self.conv_w)
                e = ops.clip_embed(e, self.cls, self.v_pos, *self.ln_pre, self.eps, n)
                e = transformer_blocks(e, self.v_layers, n, T, C, g["vision_heads"], self.eps, causal=False)
                e = ops.layernorm(e.view(n, T, C)[:, 0].contiguous(), *self.ln_post, eps=self.eps)
                outs.append(ops.gemm(e, self.v_proj).float())
        return torch.cat(outs)

    def _ids(self, text) -> torch.Tensor:
        if isinstance(text, str):
            text = [text]
        if not torch.is_tensor(text):
            tok = self.tokenize or _default_tokenize()
            text = tok(list(text))
        ids = torch.as_tensor(text).to(self.dev, torch.int64)
        if ids.dim() == 1:
            ids = ids[None]
        if ids.dim() != 2 or ids.shape[1] != self.geom["context_length"]:
            raise ValueError(f"token ids {tuple(ids.shape)}: expected [P, {self.geom['context_length']}]")
        return ids.contiguous()

    @torch.no_grad()
    def encode_text(self, text) -> torch.Tensor:
        """model.py:343-356: token ids [P, 77] (or prompt strings) -> text features [P, embed_dim] fp32, pooled at the first end-of-text
        position (`text.argmax(-1)`)."""
        g = self.geom
        ids = self._ids(text)
        L, C = ids.shape[1], g["text_width"]
        outs = []
        with torch.cuda.device(self.dev):
            for s in range(0, ids.shape[0], MAX_ATTN_ROWS):
                b = ids[s:s + MAX_ATTN_ROWS]
                n = b.shape[0]
                x = ops.embed_tokens(self.tok, self.t_pos, b)
                x = transformer_blocks(x, self.t_layers, n, L, C, g["text_heads"], self.eps, causal=True)
                x = x.view(n, L, C)[torch.arange(n, device=self.dev), b.argmax(-1)].contiguous()
                x = ops.layernorm(x, *self.ln_final, eps=self.eps)
                outs.append(ops.gemm(x, self.t_proj).float())
        return torch.cat(outs)

    def _logits(self, img: torch.Tensor, txt: torch.Tensor) -> torch.Tensor:
        """scale * cos of every (image, prompt) pair through fz_clip_scores, two prompts per launch."""
        N, P = img.shape[0], txt.shape[0]
        out = torch.empty((N, P), dtype=f32, device=self.dev)
        for s in range(0, N, MAX_CLIPS_PER_LAUNCH):
            n = min(MAX_CLIPS_PER_LAUNCH, N - s)
            for j in range(0, P, 2):
                jj = min(j + 1, P - 1)
                r = ops.clip_scores(img[s:s + n].contiguous(), txt, [1] * n, [(j, jj)] * n, self.logit_scale)
                out[s:s + n, j] = r["logits"][:, 0]
                out[s:s + n, jj] = r["logits"][:, 1]
        return out

    @torch.no_grad()
    def __call__(self, image: torch.Tensor, text):
        """model.py:358-372: (logits_per_image [N, P], logits_per_text [P, N])."""
        with torch.cuda.device(self.dev):
            li = self._logits(self.encode_image(image), self.encode_text(text))
        return li, li.t()

    # ---- scoring --------------------------------------------------------------------------------------------------------------------------
    def _frames(self, clip: Frames) -> List[torch.Tensor]:
        """A clip as device uint8 [n, H, W, 3] runs of equally sized frames, in frame order."""
        if isinstance(clip, str):
            clip = _read_folder(clip)
        if torch.is_tensor(clip):
            if clip.dtype != torch.uint8 or clip.dim() != 4 or clip.shape[-1] != 3 or clip.shape[0] < 1:
                raise ValueError(f"frames must be uint8 [F, H, W, 3], got {clip.dtype} {tuple(clip.shape)}")
            return [clip.to(self.dev).contiguous()]
        arrs = []
        for im in clip:
            a = np.asarray(im.convert("RGB") if hasattr(im, "convert") else im)
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[-1] != 3:
                raise ValueError(f"frames must be RGB uint8 images, got {a.dtype} {a.shape}")
            arrs.append(a)
        if not arrs:
            raise ValueError("a clip has no frames")
        runs, cur = [], [arrs[0]]
        for a in arrs[1:]:
            if a.shape == cur[-1].shape:
                cur.append(a)
            else:
                runs.append(cur)
                cur = [a]
        runs.append(cur)
        return [torch.from_numpy(np.stack(r)).to(self.dev) for r in runs]

    @torch.no_grad()
    def score_batch(self, clips: Sequence[Frames], source, targets) -> List[dict]:
        """Score K clips, clip k against (source, targets[k]), with one image-tower pass over all frames and one text-tower pass over
        {source} + targets.  Each result equals `score(clips[k], source, targets[k])` bit for bit."""
        clips = list(clips)
        if isinstance(targets, str):
            targets = [targets]
        if torch.is_tensor(targets):
            targets = list(targets.reshape(-1, targets.shape[-1]))
        targets = list(targets)
        if not clips:
            raise ValueError("score_batch needs at least one clip")
        if len(targets) != len(clips):
            raise ValueError(f"{len(clips)} clips but {len(targets)} target prompts")
        # prompt rows: the source first, then each distinct target
        prompts, keys, rows = [source], [_prompt_key(source)], []
        for t in targets:
            k = _prompt_key(t)
            if k not in keys:
                keys.append(k)
                prompts.append(t)
            rows.append(keys.index(k))
        with torch.cuda.device(self.dev):
            ids = torch.cat([self._ids(p) for p in prompts])
            frames = [self._frames(c) for c in clips]
            counts = [sum(r.shape[0] for r in runs) for runs in frames]
            pix = torch.cat([self.preprocess_u8(r, crop_bottom_square=True) for runs in frames for r in runs])
            img = self.encode_image(pix)
            txt = self.encode_text(ids)
            out, first = [], 0
            for s in range(0, len(clips), MAX_CLIPS_PER_LAUNCH):
                ks = range(s, min(s + MAX_CLIPS_PER_LAUNCH, len(clips)))
                n = sum(counts[k] for k in ks)
                r = ops.clip_scores(img[first:first + n].contiguous(), txt, [counts[k] for k in ks], [(0, rows[k]) for k in ks],
                                    self.logit_scale)
                r = {k: v.cpu() for k, v in r.items()}
                f0 = 0
                for i, k in enumerate(ks):
                    F = counts[k]
                    sl = slice(f0, f0 + F)
                    succ = r["success"][sl].bool()
                    out.append(dict(accuracy=float(succ.sum().item()) / F, consistency=float(r["clip_mean"][i]), success=succ,
                                    probs=r["probs"][sl], logits=r["logits"][sl], margins=r["margin"][sl], cosines=r["cosine"][sl][:F - 1],
                                    image_features=img[first + f0:first + f0 + F], text_features=txt[[0, rows[k]]]))
                    f0 += F
                first += n
        return out

    def score(self, frames: Frames, source, target) -> dict:
        """One clip: device uint8 frames [F, H, W, 3], a list of PIL images or a folder of PNGs, against (source, target).  Returns
        accuracy (share of frames with probs[target] >= probs[source]), consistency (mean cosine of consecutive frames' image features;
        NaN for one frame), per-frame success, probs [F, 2] and logits [F, 2] (source, target), margins (logit_t - logit_s), cosines [F-1]."""
        return self.score_batch([frames], source, [target])[0]

    def folder_success(self, folder: str, source, target):
        """frame_acc_tem_con.py:35-54: (success rate, temporal consistency) of the PNG frames of `folder`, in sorted file order."""
        r = self.score(folder, source, target)
        return r["accuracy"], r["consistency"]

    def score_latents(self, pipe, latents_list: Sequence[torch.Tensor], source, targets) -> List[dict]:
        """Score the `output_type="latent"` results of `p2preplace_edit_batch` (latents [1, 4, F, h, w] per target) without a host round
        trip: decode_latents_u8 on the device, then score_batch."""
        clips = [pipe.decode_latents_u8(lat).flatten(0, -4) for lat in latents_list]
        return self.score_batch(clips, source, targets)


def _prompt_key(p):
    return p if isinstance(p, str) else tuple(torch.as_tensor(p).reshape(-1).tolist())


def _read_folder(folder: str):
    from PIL import Image
    files = sorted(glob.glob(folder + "/*png"))
    if not files:
        raise FileNotFoundError(f"no PNG frames in {folder}")
    out = []
    for p in files:
        with Image.open(p) as im:
            out.append(im.convert("RGB"))
    return out
