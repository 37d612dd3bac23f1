"""Synthetic, portable inputs for tests / bench: UNet geometries, a seeded weight recipe, toy tokenizer / text encoder.

There is no network and no SD checkpoint on the build or GPU boxes (SURVEY.md §8(c)/(d)), so every test and bench
run uses random weights of the right geometry.  The recipe below is *name-keyed* (one RNG stream per state-dict key),
so the reference UNet (built through the oracle shim), the CPU oracle and the CUDA engine all get bit-identical
weights without depending on module construction order.
"""
from __future__ import annotations

import zlib
from typing import Dict, List

import torch

# SD-1.4 `unet/config.json` values (SURVEY.md §8(d) "Synthetic inputs")
SD14_UNET_CONFIG = dict(
    sample_size=64, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True, freq_shift=0,
    down_block_types=("CrossAttnDownBlockPseudo3D", "CrossAttnDownBlockPseudo3D", "CrossAttnDownBlockPseudo3D",
                      "DownBlockPseudo3D"),
    up_block_types=("UpBlockPseudo3D", "CrossAttnUpBlockPseudo3D", "CrossAttnUpBlockPseudo3D",
                    "CrossAttnUpBlockPseudo3D"),
    block_out_channels=(320, 640, 1280, 1280), layers_per_block=2, downsample_padding=1, mid_block_scale_factor=1,
    act_fn="silu", norm_num_groups=32, norm_eps=1e-5, cross_attention_dim=768, attention_head_dim=8,
)

# Small geometry with the same topology (16 transformers, 22 resnets): seconds per step on CPU.
MINI_UNET_CONFIG = dict(SD14_UNET_CONFIG, block_out_channels=(64, 128, 256, 256), cross_attention_dim=128)

# Medium geometry whose head dims (40, 80, 160, 160) equal SD-1.4's at a quarter of the channel count.
MID_UNET_CONFIG = dict(SD14_UNET_CONFIG, block_out_channels=(160, 320, 640, 640), attention_head_dim=4,
                       cross_attention_dim=256)

# SD-2.0 / 2.1-base `unet/config.json` values: heads per block 5 / 10 / 20 / 20 (head dim 64 at every level), linear proj_in / proj_out,
# 1024-wide OpenCLIP text (the text stand-in is ToyTextEncoder(1024)).
SD2_UNET_CONFIG = dict(SD14_UNET_CONFIG, attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024, use_linear_projection=True,
                       upcast_attention=False)

# Small SD-2 geometry: same topology and head dim 64 at every level (heads 1 / 2 / 4 / 4), 1024-wide text.
SD2_MINI_UNET_CONFIG = dict(SD2_UNET_CONFIG, block_out_channels=(64, 128, 256, 256), attention_head_dim=(1, 2, 4, 4))

UNET_CONFIGS = {"sd14": SD14_UNET_CONFIG, "mini": MINI_UNET_CONFIG, "mid": MID_UNET_CONFIG, "sd2": SD2_UNET_CONFIG,
                "sd2mini": SD2_MINI_UNET_CONFIG}

DEFAULT_MODEL_CONFIG = dict(lora=160, SparseCausalAttention_index=["mid"], least_sc_channel=640)


def _gen(name: str, seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(name.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


def synth_tensor(name: str, shape, seed: int = 0) -> torch.Tensor:
    """Deterministic fp32 tensor for state-dict key `name` (scale chosen so activations stay O(1))."""
    shape = tuple(shape)
    g = _gen(name, seed)
    if name.endswith("bias"):
        return 0.02 * torch.randn(shape, generator=g)
    if len(shape) == 1:  # norm weights
        return 1.0 + 0.05 * torch.randn(shape, generator=g)
    fan_in = 1
    for s in shape[1:]:
        fan_in *= s
    std = fan_in ** -0.5
    if "conv_temporal.up" in name:
        std *= 0.5  # non-degenerate temporal LoRA (reference zero-inits it: lora.py:42)
    if "attn_temporal.to_out.0.weight" in name:
        std *= 0.5  # reference zero-inits this one (models/attention.py:224)
    if "to_out" in name or "proj_out" in name or "conv2" in name or "ff.net.2" in name:
        std *= 0.5  # keep residual branches tame
    return std * torch.randn(shape, generator=g)


def synth_state_dict(shapes: Dict[str, tuple], seed: int = 0, degenerate_temporal: bool = False) -> Dict[str, torch.Tensor]:
    """`shapes`: {state-dict key: shape}. With degenerate_temporal the reference's zero inits are kept."""
    sd = {}
    for name in sorted(shapes):
        t = synth_tensor(name, shapes[name], seed)
        if degenerate_temporal and ("conv_temporal.up" in name or "attn_temporal.to_out.0.weight" in name):
            t = torch.zeros_like(t)
        sd[name] = t
    return sd


def synth_latents(frames: int, h: int, w: int, seed: int = 1, channels: int = 4) -> torch.Tensor:
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn((1, channels, frames, h, w), generator=g)


class ToyTokenizer:
    """Word-level tokenizer with the CLIP call surface the reference uses (encode / decode / __call__).

    Words longer than `split_at` characters become two tokens so the multi-token branches of
    `ptp_utils.get_word_inds` / `seq_aligner` are exercised. ids: BOS 49406, EOS = pad = 49407 as in SD.
    """
    bos_token_id = 49406
    eos_token_id = 49407
    model_max_length = 77

    def __init__(self, split_at: int = 9):
        self.split_at = split_at
        self._id2piece: Dict[int, str] = {}

    def _piece_id(self, piece: str) -> int:
        i = 1000 + (zlib.crc32(piece.encode()) % 40000)
        self._id2piece[i] = piece
        return i

    def _pieces(self, text: str) -> List[str]:
        out = []
        for word in text.split(" "):
            if word == "":
                continue
            if len(word) > self.split_at:
                out += [word[: len(word) // 2], word[len(word) // 2:]]
            else:
                out.append(word)
        return out

    def encode(self, text: str) -> List[int]:
        return [self.bos_token_id] + [self._piece_id(p) for p in self._pieces(text)] + [self.eos_token_id]

    def decode(self, ids) -> str:
        out = []
        if isinstance(ids, int) or (torch.is_tensor(ids) and ids.dim() == 0):
            ids = [int(ids)]
        for i in ids:
            i = int(i)
            if i == self.bos_token_id:
                out.append("<|startoftext|>")
            elif i == self.eos_token_id:
                out.append("<|endoftext|>")
            else:
                out.append(self._id2piece.get(i, "?"))
        return " ".join(out)

    def batch_decode(self, batch):
        return [self.decode(x) for x in batch]

    def __call__(self, prompt, padding="max_length", max_length=None, truncation=True, return_tensors="pt"):
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        rows = [self.encode(p) for p in prompts]
        if padding == "max_length":
            L = max_length or self.model_max_length
        else:
            L = max(len(r) for r in rows)
        ids = torch.full((len(rows), L), self.eos_token_id, dtype=torch.long)
        for i, r in enumerate(rows):
            r = r[:L]
            if len(r) == L:
                r[-1] = self.eos_token_id
            ids[i, : len(r)] = torch.tensor(r)

        class _Out:
            pass
        o = _Out()
        o.input_ids = ids
        o.attention_mask = torch.ones_like(ids)
        return o


class ToyTextEncoder(torch.nn.Module):
    """Deterministic stand-in for CLIPTextModel: hidden[b, p] = E[id % V] + P[p] (then one mixing layer)."""

    class _Cfg:
        use_attention_mask = False

    def __init__(self, dim: int = 768, seed: int = 0, vocab: int = 4096):
        super().__init__()
        self.config = self._Cfg()
        self.vocab = vocab
        self.emb = torch.nn.Parameter(synth_tensor("toy_text.emb.weight", (vocab, 64), seed) * 8.0, requires_grad=False)
        self.pos = torch.nn.Parameter(synth_tensor("toy_text.pos.weight", (77, 64), seed) * 8.0, requires_grad=False)
        self.proj = torch.nn.Parameter(synth_tensor("toy_text.proj.weight", (dim, 64), seed), requires_grad=False)

    def forward(self, input_ids, attention_mask=None):
        h = self.emb[input_ids % self.vocab] + self.pos[None, : input_ids.shape[1]]
        h = torch.tanh(h) @ self.proj.t()
        return (h,)


class VaeStub(torch.nn.Module):
    """Latent-level tests bypass the VAE (SURVEY.md §8(c)); only `.config.block_out_channels` is read."""

    class _Cfg:
        block_out_channels = (128, 256, 512, 512)

    def __init__(self):
        super().__init__()
        self.config = self._Cfg()
        self.dummy = torch.nn.Parameter(torch.zeros(1), requires_grad=False)

    def decode(self, latents):
        class _O:
            pass
        o = _O()
        x = latents[:, :3]
        o.sample = torch.nn.functional.interpolate(x.float(), scale_factor=8.0, mode="nearest")
        return o
