"""CLIP text encoder on the sm_90a kernels (SURVEY.md §8(f) rank 4).  The reference encodes prompts with transformers' CLIPTextModel
(`pipelines/stable_diffusion.py:230,279`: `self.text_encoder(ids, attention_mask=...)[0]`); `ClipTextEngine` executes the same pre-LN
transformer (token + position embedding, N x {LN, causal self-attention, LN, quick_gelu / gelu MLP}, final LN) with fz_layernorm / fz_gemm /
fz_attention (causal = 1) / fz_quick_gelu (SD-1.x) or fz_gelu (the exact-erf GELU of the SD-2.x OpenCLIP text towers): fp16 storage,
fp32 accumulation, fp32 output.  Weights are read from a CLIPTextModel-shaped
state dict (`text_model.*` names); anything else (attention masks, projection heads, other activations) is refused, and the pipeline then
keeps calling the caller's module."""
from __future__ import annotations

from typing import Dict

import torch

from . import ops

f16, f32 = torch.float16, torch.float32


# transformers' CLIPMLP activation (config.hidden_act) -> the in-place kernel that computes it
ACTIVATIONS = {"quick_gelu": ops.quick_gelu_, "gelu": ops.gelu_}


class ClipTextEngine:
    def __init__(self, text_encoder: torch.nn.Module):
        cfg = text_encoder.config
        act = getattr(cfg, "hidden_act", "quick_gelu")
        if act not in ACTIVATIONS:
            raise NotImplementedError(f"CLIP hidden_act {act!r} (SD-1.x text encoders use quick_gelu, SD-2.x gelu)")
        self.act = ACTIVATIONS[act]
        sd: Dict[str, torch.Tensor] = {k: v.detach() for k, v in text_encoder.state_dict().items()}
        dev = next(text_encoder.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("ClipTextEngine needs the text encoder on a CUDA device")
        self.dev = dev
        self.C = int(cfg.hidden_size)
        self.heads = int(cfg.num_attention_heads)
        self.d = self.C // self.heads
        self.L = int(cfg.max_position_embeddings)
        self.eps = float(getattr(cfg, "layer_norm_eps", 1e-5))
        if self.d % 8 or self.d > 192:
            raise NotImplementedError(f"CLIP head dim {self.d}")
        p = "text_model."

        def h(t):
            return t.to(dev, f16).contiguous()

        def f(t):
            return t.to(dev, f32).contiguous()

        self.tok = f(sd[p + "embeddings.token_embedding.weight"])
        self.pos = f(sd[p + "embeddings.position_embedding.weight"])
        self.layers = []
        for i in range(int(cfg.num_hidden_layers)):
            q = f"{p}encoder.layers.{i}."
            self.layers.append(dict(
                ln1=(f(sd[q + "layer_norm1.weight"]), f(sd[q + "layer_norm1.bias"])),
                ln2=(f(sd[q + "layer_norm2.weight"]), f(sd[q + "layer_norm2.bias"])),
                qkv_w=h(torch.cat([sd[q + "self_attn.q_proj.weight"], sd[q + "self_attn.k_proj.weight"], sd[q + "self_attn.v_proj.weight"]], 0)),
                qkv_b=f(torch.cat([sd[q + "self_attn.q_proj.bias"], sd[q + "self_attn.k_proj.bias"], sd[q + "self_attn.v_proj.bias"]], 0)),
                out_w=h(sd[q + "self_attn.out_proj.weight"]), out_b=f(sd[q + "self_attn.out_proj.bias"]),
                fc1_w=h(sd[q + "mlp.fc1.weight"]), fc1_b=f(sd[q + "mlp.fc1.bias"]),
                fc2_w=h(sd[q + "mlp.fc2.weight"]), fc2_b=f(sd[q + "mlp.fc2.bias"])))
        self.ln_f = (f(sd[p + "final_layer_norm.weight"]), f(sd[p + "final_layer_norm.bias"]))

    @torch.no_grad()
    def __call__(self, input_ids: torch.Tensor, attention_mask=None):
        if attention_mask is not None:
            raise NotImplementedError("padding masks are not used by SD-1.x text encoders (config.use_attention_mask is False)")
        B, L = input_ids.shape
        if L > self.L:
            raise ValueError(f"{L} tokens > max_position_embeddings {self.L}")
        with torch.cuda.device(self.dev):
            x = ops.embed_tokens(self.tok, self.pos, input_ids.to(self.dev))
            x = transformer_blocks(x, self.layers, B, L, self.C, self.heads, self.eps, causal=True, act=self.act)
            out = ops.layernorm(x, *self.ln_f, eps=self.eps)
        return (out.float().view(B, L, self.C),)


def transformer_blocks(x: torch.Tensor, layers, B: int, L: int, C: int, heads: int, eps: float, causal: bool,
                       act=ops.quick_gelu_) -> torch.Tensor:
    """The pre-LN CLIP residual blocks on the current device: x [B*L, C] fp16 (B <= 64 sequences of L tokens, fz_attention_f16's row
    limit) through {LN, self-attention, LN, MLP with the in-place activation `act`} per layer dict (ln1, ln2, qkv_w / qkv_b with q | k | v rows, out_w / out_b,
    fc1_w / fc1_b, fc2_w / fc2_b)."""
    d = C // heads
    ld = (L + 7) // 8 * 8
    vt = torch.zeros((B, heads, d, ld), dtype=f16, device=x.device)
    for ly in layers:
        hn = ops.layernorm(x, *ly["ln1"], eps=eps)
        qk = ops.gemm(hn, ly["qkv_w"], bias=ly["qkv_b"], vt=dict(out=vt, col_start=2 * C, S=L, d=d, heads=heads, ld=ld))
        o = torch.empty((B * L, C), dtype=f16, device=x.device)
        ops.attention(qk[:, :C], qk[:, C:], vt, o, S_q=L, keys_per_slot=L, n_src=B, d=d, heads=heads, F=1, BF=B, scale=d ** -0.5,
                      src_index=[list(range(B))], causal=causal)
        x = ops.gemm(o, ly["out_w"], bias=ly["out_b"], residual=x)
        hn = ops.layernorm(x, *ly["ln2"], eps=eps)
        m = act(ops.gemm(hn, ly["fc1_w"], bias=ly["fc1_b"]))
        x = ops.gemm(m, ly["fc2_w"], bias=ly["fc2_b"], residual=x)
    return x
