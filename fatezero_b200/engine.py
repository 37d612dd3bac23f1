"""UNetEngine — executes one UNetPseudo3DConditionModel forward with the sm_90a kernels of libfatezero_b200.so.

Data layout in HBM: every activation is fp16 channels-last, `[B*F, H, W, C]` == token-major `[B*F*H*W, C]` (frame-minor batch
order like the reference's "(b f)" rearranges), so conv / linear / attention kernels read and write the same buffers without
transposes; weights are packed once per model into fp16 K-major matrices (`[9][Cout][Cin]` for 3x3 convs, `[3][Cout][Cin]` for the
temporal LoRA, `[N][K]` for linears, tile-interleaved for GEGLU, Q|K|V fused).  Text K / V^T of all 16 cross-attention layers are
computed once per prompt (they are constant over frames and steps: models/attention.py:104).

Reference forward restated: models/unet_3d_condition.py:307-446 (+ unet_3d_blocks.py, resnet.py:335-394, attention.py:95-144,271-337).
The attention controller is not called back per layer; it is asked for kernel arguments (`self_attn_args` / `cross_attn_args`)
and the STORE / INJECT / BLEND work happens inside fz_attention_f16.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

import ctypes as C

from . import _lib, ops
from .unet import transformer_heads

f16 = torch.float16
f32 = torch.float32


def sc_frame_indices(index_list, clip_length: int) -> List[List[int]]:
    """Source frame of every query frame, per K/V slot (attention_register.py:168-188)."""
    out = []
    for index in index_list:
        if isinstance(index, str):
            if index == "first":
                fi = [0] * clip_length
            elif index == "last":
                fi = [clip_length - 1] * clip_length
            elif index in ("mid", "middle"):
                fi = [int((clip_length - 1) // 2)] * clip_length
            else:
                raise ValueError(f"unknown SparseCausalAttention_index entry {index!r}")
        else:
            if not isinstance(index, int):
                raise AssertionError("relative index must be int")
            fi = [min(max(f + index, 0), clip_length - 1) for f in range(clip_length)]
        out.append(fi)
    return out


class UNetEngine:
    def __init__(self, unet, exact_skips: bool = True):
        dev = unet.device
        if dev.type != "cuda":
            raise RuntimeError("UNetEngine needs the UNet parameters on a CUDA device (sm_90a); no CPU fallback exists")
        lib = _lib.load()
        _lib.check(lib.fz_device_check(), "fz_device_check")
        with torch.cuda.device(dev):
            _lib.check(lib.fz_init(ops._stream()), "fz_init")
            ops._workspace(dev, 1 << 20)  # GroupNorm partial-sum workspace: allocated up front (never inside a graph capture)
        self.cfg = dict(unet.config)
        self.mc = dict(unet.model_config)
        self.dev = dev
        self.heads = transformer_heads(self.cfg)  # transformer prefix -> head count of its level (SD-2.x: 5 / 10 / 20 / 20)
        self.groups = self.cfg["norm_num_groups"]
        self.eps = float(self.cfg["norm_eps"])
        self.ch = list(self.cfg["block_out_channels"])
        self.exact_skips = exact_skips
        self.w: Dict[str, torch.Tensor] = {}
        self._text_key = None
        self._text_kv: Dict[str, tuple] = {}
        self._foreign = None  # reference-protocol controller of the current forward (slow path), see _foreign_attention
        self.shard = None  # frame sharding over GPUs: (rank, world, process group), see set_frame_shard
        # batched edit of K prompts (controller.prompt_groups = K > 1): the GroupNorm chunking is planned per prompt (NB / K images) so
        # that every prompt's statistics are bitwise those of its own single-prompt pass; None = planned for the whole batch
        self._images_per_item = None
        self._prepare({k: v.detach() for k, v in unet.state_dict().items()})

    # ---------------------------------------------------------------------------------------------------------------
    # frame sharding (SURVEY.md §8(e)): the frames of ONE clip are split contiguously over the GPUs of one NVSwitch box; every rank
    # calls forward() with its own frames [B, 4, F/world, H, W].  Exchanges: (1) all-gather of K and V^T over the frame axis for the
    # sparse-causal self-attention, (2) all-reduce of the GroupNorm (sum, sumsq) of the joint-frame norms.  The temporal LoRA convs and
    # the temporal attention need frame halos / an all-to-all: supported when they are exact identities (un-tuned SD weights, which is
    # what the reference's zero-shot configs run), otherwise rejected.
    # ---------------------------------------------------------------------------------------------------------------
    def set_frame_shard(self, rank: int, world: int, group=None):
        """The frames of ONE clip are split contiguously over `world` GPUs; this rank then calls forward() with ITS frames.  Sets up the
        symmetric peer-memory arena (p2p.Arena; torch.distributed must be initialised — it carries the one-time IPC handle exchange)."""
        if world <= 1:
            self.shard = None
            self.arena = None
            return
        from . import p2p
        self.shard = (int(rank), int(world), group)
        if getattr(self, "arena", None) is None or self.arena.world != world or self.arena.rank != rank:
            self.arena = p2p.Arena(int(rank), int(world), self.dev, group)

    def shard_signature(self):
        """Part of the CUDA-graph plan keys (graphs.py): a frame-sharded forward launches a different kernel sequence."""
        return None if self.shard is None else (self.shard[0], self.shard[1])

    # ---- exchange helpers (all of them: fz_p2p_push into the peers' site buffers, then a wait kernel on the local flags) -------------
    def _gn_joint(self, name: str, x3: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, F: int, silu: bool) -> torch.Tensor:
        """nn.GroupNorm over (C/G, F_total, H, W) (resnet.py:338,369; unet_3d_condition.py:439) with the frames of other ranks included:
        every rank pushes its per-image (sum, sumsq) [NB, G] into each peer's inbox (512 B .. 2 KiB over NVLink), fz_gn_combine waits for the
        peers and folds everything, in fp64, into the layout the apply kernel reads."""
        if self.shard is None:
            return ops.groupnorm(x3, gamma, beta, eps, self.groups, F, silu, images_per_item=self._images_per_item)
        rank, world, _ = self.shard
        ar = self.arena
        NB, G = x3.shape[0], self.groups
        nb = NB * G * 16                                                   # two 8-byte {value, epoch} words per (image, group)
        sums = ops.groupnorm_stats(x3, G)                                  # [NB, G, 2] fp32 view into the workspace
        site = ar.site(("gn", name, NB), world * nb)
        totals = torch.empty((NB, G, 2), dtype=torch.float64, device=x3.device)
        pi = (C.c_void_p * world)(*[ar.peer_ptr(r, site, rank * nb) if r != rank else None for r in range(world)])
        _lib.call("fz_gn_combine", C.c_void_p(ar.base + site.flag_offset + 4 * 31), pi, C.c_void_p(ar.base + site.offset),
                  C.c_void_p(sums.data_ptr()), C.c_void_p(totals.data_ptr()), NB, F, G, world, rank, ops._stream())
        return ops.groupnorm_apply(x3, gamma, beta, eps, G, F, F * world, silu, totals)

    def _halo_ext(self, key: tuple, y4: torch.Tensor) -> torch.Tensor:
        """y4 [B, F, HW, C] (this rank's frames) -> [B, F+2, HW, C] in the arena: interior = y4, frame 0 / F+1 = the last / first frame of the
        left / right neighbour rank (zeros at the clip ends: the zero padding of the un-sharded Conv1d, resnet.py:72-78)."""
        rank, world, _ = self.shard
        ar = self.arena
        B, F, HW, Cc = y4.shape
        fb = HW * Cc * 2
        site = ar.site(key + (B, F, HW, Cc), B * (F + 2) * fb)
        src = y4.data_ptr()
        segs = [(src, F * fb, rank, ar.peer_ptr(rank, site, fb), (F + 2) * fb, B, F * fb)]
        srcs = []
        if rank > 0:
            segs.append((src, F * fb, rank - 1, ar.peer_ptr(rank - 1, site, (F + 1) * fb), (F + 2) * fb, B, fb))
            srcs.append(rank - 1)
        if rank < world - 1:
            segs.append((src + (F - 1) * fb, F * fb, rank + 1, ar.peer_ptr(rank + 1, site, 0), (F + 2) * fb, B, fb))
            srcs.append(rank + 1)
        ar.exchange(site, segs, srcs, ops._stream())
        return ar.tensor(site, 0, (B, F + 2, HW, Cc))

    def _temporal_attn_sharded(self, name: str, qkvt: torch.Tensor, B: int, F: int, S: int, heads: int, d: int, scale: float) -> torch.Tensor:
        """Temporal attention over ALL frames of the clip (models/attention.py:327-337) as a frames<->pixels exchange: rank q receives the
        q-th pixel slice of every frame's q|k|v, attends over the whole frame axis for those pixels and returns the outputs to the frames'
        owners (3.5 C values per token over NVLink at 8 GPUs instead of the 14 C of a K/V all-gather)."""
        rank, world, _ = self.shard
        ar = self.arena
        Cc = heads * d
        if S % world:
            raise NotImplementedError(f"frame sharding: {S} pixels do not split over {world} ranks")
        Ss, Ft = S // world, F * world
        st = ops._stream()
        row_in = Ss * 3 * Cc * 2
        site_in = ar.site(("ta_in", name, B, F, S, Cc), B * Ft * row_in)
        q0 = qkvt.data_ptr()
        segs = [(q0 + (b * F * S + r * Ss) * 3 * Cc * 2, S * 3 * Cc * 2, r, ar.peer_ptr(r, site_in, (b * Ft + rank * F) * row_in), row_in, F, row_in)
                for r in range(world) for b in range(B)]
        ar.exchange(site_in, segs, range(world), st)
        buf = ar.tensor(site_in, 0, (B * Ft * Ss, 3 * Cc))
        os_ = ops.temporal_attn(buf, B, Ft, Ss, heads, d, scale)             # [B * Ft * Ss, C]
        row_out = Ss * Cc * 2
        site_out = ar.site(("ta_out", name, B, F, S, Cc), B * F * S * Cc * 2)
        o0 = os_.data_ptr()
        segs = [(o0 + (b * Ft + r * F) * row_out, row_out, r, ar.peer_ptr(r, site_out, (b * F * S + rank * Ss) * Cc * 2), S * Cc * 2, F, row_out)
                for r in range(world) for b in range(B)]
        ar.exchange(site_out, segs, range(world), st)
        return ar.tensor(site_out, 0, (B * F * S, Cc))

    def _kv_exchange(self, name: str, qk: torch.Tensor, vt: torch.Tensor, index_list, B: int, F: int, S: int, Cc: int, heads: int, d: int):
        """K and V^T of the frames the sparse-causal attention reads (attention_register.py:162-193).  Constant source frames ('first',
        'mid', 'last': the reference's zero-shot configs) are pushed by their owner to every rank (1/F_total of an all-gather); relative
        indices take the all-gather over the frame axis.  Returns (k_src, vt_src, n_src, src_index)."""
        from . import dist as fzdist
        rank, world, _ = self.shard
        ar = self.arena
        st = ops._stream()
        fis = sc_frame_indices(index_list, F * world)  # indices over the GLOBAL frames; rank r holds [r*F, (r+1)*F)
        kb, vb = S * Cc * 2, heads * d * S * 2         # bytes of one frame's K rows / V^T block
        q0, v0 = qk.data_ptr(), vt.data_ptr()
        ld = qk.stride(0) * 2
        if all(isinstance(ix, str) for ix in index_list):
            n = len(fis)
            site = ar.site(("kv_const", name, B, F, S, Cc, n), n * B * (kb + vb))
            voff = n * B * kb
            # all slots this rank owns travel in ONE push, so that every owner raises its flag exactly once per exchange
            segs = []
            for sl, fi in enumerate(fis):
                owner, gl = fi[0] // F, fi[0] % F
                if owner == rank:
                    for r in range(world):
                        for b in range(B):
                            segs.append((q0 + (b * F + gl) * S * ld + Cc * 2, ld, r, ar.peer_ptr(r, site, (sl * B + b) * kb), Cc * 2, S, Cc * 2))
                            segs.append((v0 + (b * F + gl) * vb, vb, r, ar.peer_ptr(r, site, voff + (sl * B + b) * vb), vb, 1, vb))
            ar.exchange(site, segs, sorted({fi[0] // F for fi in fis}), st)
            k_src = ar.tensor(site, 0, (n * B * S, Cc))
            vt_src = ar.tensor(site, voff, (n * B, heads, d, S))
            src_index = [[sl * B + b for b in range(B) for _ in range(F)] for sl in range(n)]
            return k_src, vt_src, n * B, src_index
        NB = B * F
        site = ar.site(("kv_all", name, B, F, S, Cc), world * NB * (kb + vb))
        voff = world * NB * kb
        segs = []
        for r in range(world):
            segs.append((q0 + Cc * 2, ld, r, ar.peer_ptr(r, site, rank * NB * kb), Cc * 2, NB * S, Cc * 2))
            segs.append((v0, NB * vb, r, ar.peer_ptr(r, site, voff + rank * NB * vb), NB * vb, 1, NB * vb))
        ar.exchange(site, segs, range(world), st)
        k_src = ar.tensor(site, 0, (world * NB * S, Cc))
        vt_src = ar.tensor(site, voff, (world * NB, heads, d, S))
        src_index = [fzdist.gathered_source_rows(fi, rank, world, F, B) for fi in fis]
        return k_src, vt_src, world * NB, src_index

    # ---------------------------------------------------------------------------------------------------------------
    # weight packing
    # ---------------------------------------------------------------------------------------------------------------
    def _prepare(self, sd: Dict[str, torch.Tensor]):
        w = self.w
        dev = self.dev

        def h(t):
            return t.to(dev, f16).contiguous()

        def f(t):
            return t.to(dev, f32).contiguous()

        self.has = set(sd.keys())
        self.lora_skip = {}
        for name, t in sd.items():
            if name.endswith(".weight") and t.dim() == 4 and t.shape[-1] == 3 and name not in ("conv_in.weight",):
                co, ci = t.shape[:2]
                if name == "conv_out.weight":
                    w9 = torch.zeros(9, 16, ci)
                    w9[:, :co] = t.permute(2, 3, 0, 1).reshape(9, co, ci)
                    w[name] = h(w9)  # padded to one 16-wide MMA tile
                else:
                    w[name] = h(t.permute(2, 3, 0, 1).reshape(9, co, ci))
            elif name == "conv_in.weight":
                co, ci = t.shape[:2]
                wp = torch.zeros(co, 64)
                wp[:, : 9 * ci] = t.permute(0, 2, 3, 1).reshape(co, 9 * ci)  # col = tap*Cin + c
                w[name] = h(wp)
            elif name.endswith(".weight") and t.dim() == 4 and t.shape[-1] == 1:
                w[name] = h(t.reshape(t.shape[0], t.shape[1]))
            elif "conv_temporal" in name and name.endswith(".weight") and t.dim() == 3:
                if name.startswith("conv_out."):
                    w[name + "#f32"] = f(t)  # tiny (C=4): handled by fz_out_temporal_f32
                w[name] = h(t.permute(2, 0, 1))  # [3][Cout][Cin]
            elif name == "conv_out.bias":
                w[name] = f(torch.nn.functional.pad(t.float(), (0, 16 - t.shape[0])))
            elif name.endswith(".time_emb_proj.weight") or any(name.endswith(sfx) for sfx in (
                    "attn1.to_q.weight", "attn1.to_k.weight", "attn1.to_v.weight", "attn2.to_k.weight", "attn2.to_v.weight",
                    "attn_temporal.to_q.weight", "attn_temporal.to_k.weight", "attn_temporal.to_v.weight")):
                continue  # only used through the fused matrices built below
            elif name.endswith("ff.net.0.proj.weight"):
                pw, pb, bn = ops.pack_geglu(t.float(), sd[name[:-6] + "bias"].float())
                w[name] = h(pw)
                w[name[:-6] + "bias"] = f(pb)
                w[name + "#bn"] = bn
            elif name.endswith("ff.net.0.proj.bias"):
                continue
            elif name.endswith(".weight") and t.dim() == 2:
                w[name] = h(t)
            else:
                w[name] = f(t)
        # fused projections
        for name in list(sd.keys()):
            if name.endswith("attn1.to_q.weight"):
                p = name[: -len("to_q.weight")]
                w[p + "qkv"] = h(torch.cat([sd[p + "to_q.weight"], sd[p + "to_k.weight"], sd[p + "to_v.weight"]], 0))
            if name.endswith("attn_temporal.to_q.weight"):
                p = name[: -len("to_q.weight")]
                w[p + "qkv"] = h(torch.cat([sd[p + "to_q.weight"], sd[p + "to_k.weight"], sd[p + "to_v.weight"]], 0))
            if name.endswith("attn2.to_k.weight"):
                p = name[: -len("to_k.weight")]
                w[p + "kv"] = h(torch.cat([sd[p + "to_k.weight"], sd[p + "to_v.weight"]], 0))
        # exact algebraic skips (identity temporal layers of un-tuned SD weights: lora.py:42, models/attention.py:224)
        for name, t in sd.items():
            if name.endswith("conv_temporal.up.weight"):
                self.lora_skip[name[: -len(".conv_temporal.up.weight")]] = self.exact_skips and bool((t == 0).all())
            if name.endswith("attn_temporal.to_out.0.weight") and self.exact_skips and bool((t == 0).all()):
                tp = name[: -len(".transformer_blocks.0.attn_temporal.to_out.0.weight")]
                bt = sd[name[:-6] + "bias"].float()
                wpo = sd[tp + ".proj_out.weight"].float().reshape(bt.shape[0], -1)
                # proj_out(h + b_t) = proj_out(h) + W_po b_t : fold the constant into the proj_out bias
                w[tp + ".proj_out.bias#folded"] = f(sd[tp + ".proj_out.bias"].float() + wpo @ bt)
        # the 22 time_emb_proj layers as one row-vector GEMM
        names = [n[: -len(".time_emb_proj.weight")] for n in sd if n.endswith(".time_emb_proj.weight")]
        self.temb_slices = {}
        off = 0
        ws, bs = [], []
        for n in names:
            co = sd[n + ".time_emb_proj.weight"].shape[0]
            self.temb_slices[n] = (off, off + co)
            off += co
            ws.append(sd[n + ".time_emb_proj.weight"])
            bs.append(sd[n + ".time_emb_proj.bias"])
        w["#temb_proj.weight"] = h(torch.cat(ws, 0))
        w["#temb_proj.bias"] = f(torch.cat(bs, 0))

    # ---------------------------------------------------------------------------------------------------------------
    # text K / V^T cache (attention_register.py:99-100 recomputes these per frame, layer and step)
    # ---------------------------------------------------------------------------------------------------------------
    def _ensure_text(self, text: torch.Tensor):
        key = (text.data_ptr(), tuple(text.shape), text._version)
        if key == self._text_key:
            return
        B, L, D = text.shape
        if L != 77:
            raise NotImplementedError("cross-attention expects 77 text tokens (CLIP max length)")
        t16 = text.to(self.dev, f16).reshape(B * L, D).contiguous()
        self._text_kv = {}
        for name in self.w:
            if name.endswith("attn2.kv"):
                wkv = self.w[name]
                if wkv.shape[1] != D:
                    raise ValueError(f"encoder_hidden_states width {D} != cross_attention_dim {wkv.shape[1]}")
                heads = self.heads[name[: -len(".transformer_blocks.0.attn2.kv")]]
                c = wkv.shape[0] // 2
                d = c // heads
                vt = torch.zeros((B, heads, d, 80), dtype=f16, device=self.dev)
                k = ops.gemm(t16, wkv, vt=dict(out=vt, col_start=c, S=L, d=d, heads=heads, ld=80))
                self._text_kv[name[: -len(".kv")]] = (k, vt)
        self._text_key = key
        self._text_ref = text  # keep alive so data_ptr stays unique

    # ---------------------------------------------------------------------------------------------------------------
    # building blocks
    # ---------------------------------------------------------------------------------------------------------------
    def _temporal(self, name: str, y: torch.Tensor, B: int, F: int, group_bias=None, residual2=None) -> torch.Tensor:
        """y [B*F, H, W, C] conv output -> temporal conv (resnet.py:72-78) fused with +temb / +shortcut."""
        w = self.w
        NB, H, W, C = y.shape
        M = NB * H * W
        y4 = y.view(B, F, H * W, C)
        sh = self.shard is not None
        if name + ".conv_temporal.down.weight" in w:
            # frame-sharded: the Conv1d pair needs one boundary frame of the neighbour ranks for each conv (y, then the rank-160 intermediate)
            mid = ops.tconv3(self._halo_ext(("halo_y", name), y4) if sh else y4, w[name + ".conv_temporal.down.weight"], halo=sh)
            out = ops.tconv3(self._halo_ext(("halo_mid", name), mid) if sh else mid, w[name + ".conv_temporal.up.weight"], residual=y4,
                             residual2=residual2, group_bias=group_bias, rows_per_group=M, halo=sh)
        else:
            out = ops.tconv3(self._halo_ext(("halo_y", name), y4) if sh else y4, w[name + ".conv_temporal.weight"],
                             bias=w[name + ".conv_temporal.bias"], residual2=residual2, group_bias=group_bias, rows_per_group=M, halo=sh)
        return out.view(NB, H, W, C)

    def _has_temporal(self, name: str) -> bool:
        if name + ".conv_temporal.down.weight" in self.w:
            return not self.lora_skip.get(name, False)
        return name + ".conv_temporal.weight" in self.w

    def conv(self, name: str, x: torch.Tensor, B: int, F: int, stride: int = 1, group_bias=None, residual=None) -> torch.Tensor:
        """PseudoConv3d.forward for k=3 (resnet.py:57-80), with the epilogue additions of the caller fused in."""
        w = self.w
        M_out = x.shape[0] * (x.shape[1] // stride) * (x.shape[2] // stride)
        if self._has_temporal(name):
            y = ops.conv3x3(x, w[name + ".weight"], bias=w[name + ".bias"], stride=stride)
            return self._temporal(name, y, B, F, group_bias=group_bias, residual2=residual)
        return ops.conv3x3(x, w[name + ".weight"], bias=w[name + ".bias"], stride=stride, residual=residual, group_bias=group_bias,
                           rows_per_group=M_out)

    def resnet(self, p: str, x: torch.Tensor, temb_all: torch.Tensor, B: int, F: int) -> torch.Tensor:
        """ResnetBlockPseudo3D.forward (resnet.py:335-394)."""
        w = self.w
        NB, H, W, Cin = x.shape
        n1 = self._gn_joint(p + ".norm1", x.view(NB, H * W, Cin), w[p + ".norm1.weight"], w[p + ".norm1.bias"], self.eps, F, True)
        a, b = self.temb_slices[p]
        tb = temb_all[a:b].view(1, b - a)
        h = self.conv(p + ".conv1", n1.view(NB, H, W, Cin), B, F, group_bias=tb)
        Cout = h.shape[-1]
        n2 = self._gn_joint(p + ".norm2", h.view(NB, H * W, Cout), w[p + ".norm2.weight"], w[p + ".norm2.bias"], self.eps, F, True)
        if p + ".conv_shortcut.weight" in w:
            sc = ops.gemm(x.view(-1, Cin), w[p + ".conv_shortcut.weight"], bias=w[p + ".conv_shortcut.bias"]).view(NB, H, W, Cout)
        else:
            sc = x
        return self.conv(p + ".conv2", n2.view(NB, H, W, Cout), B, F, residual=sc)

    def transformer(self, p: str, x: torch.Tensor, B: int, F: int, place: str, ctrl) -> torch.Tensor:
        """SpatioTemporalTransformerModel.forward + Block.forward (models/attention.py:95-144,271-337)."""
        w = self.w
        NB, H, W, C = x.shape
        S = H * W
        M = NB * S
        heads = self.heads[p]
        d = C // heads
        scale = d ** -0.5
        bp = p + ".transformer_blocks.0"
        xr = x.view(M, C)
        n = ops.groupnorm(x.view(NB, S, C), w[p + ".norm.weight"], w[p + ".norm.bias"], 1e-6, self.groups, 1, False,
                          images_per_item=self._images_per_item)
        h = ops.gemm(n.view(M, C), w[p + ".proj_in.weight"], bias=w[p + ".proj_in.bias"])
        # ---- attn1: sparse-causal spatio-temporal self-attention (attention_register.py:131-218)
        if "SparseCausalAttention_index" in self.mc:
            index_list = list(self.mc["SparseCausalAttention_index"])
        else:
            index_list = [-1, "first"]
        if "least_sc_channel" in self.mc and C < self.mc["least_sc_channel"]:
            index_list = []
        ln1 = ops.layernorm(h, w[bp + ".norm1.weight"], w[bp + ".norm1.bias"])
        vt = torch.empty((NB, heads, d, S), dtype=f16, device=self.dev)
        qk = ops.gemm(ln1, w[bp + ".attn1.qkv"], vt=dict(out=vt, col_start=2 * C, S=S, d=d, heads=heads))
        k_src, vt_src, n_src = qk[:, C:], vt, NB
        if self.shard is not None and index_list:
            k_src, vt_src, n_src, src_index = self._kv_exchange(p, qk, vt, index_list, B, F, S, C, heads, d)
        else:
            fis = sc_frame_indices(index_list, F) if index_list else [list(range(F))]
            src_index = [[b * F + fi[f] for b in range(B) for f in range(F)] for fi in fis]
        o = torch.empty((M, C), dtype=f16, device=self.dev)
        kw = {}
        if self._foreign is not None:
            self._foreign_attention(False, place, qk[:, :C], k_src, vt_src, o, S_q=S, keys_per_slot=S, n_src=n_src, d=d, heads=heads, F=F,
                                    BF=NB, scale=scale, src_index=src_index)
        else:
            if ctrl is not None and S <= 32 ** 2:
                kw = ctrl.self_attn_args(place, S, len(src_index) * S, heads, NB, F) or {}
            ops.attention(qk[:, :C], k_src, vt_src, o, S_q=S, keys_per_slot=S, n_src=n_src, d=d, heads=heads, F=F, BF=NB, scale=scale,
                          src_index=src_index, **kw)
        h = ops.gemm(o, w[bp + ".attn1.to_out.0.weight"], bias=w[bp + ".attn1.to_out.0.bias"], residual=h)
        # ---- attn2: text cross-attention (attention_register.py:71-128)
        ln2 = ops.layernorm(h, w[bp + ".norm2.weight"], w[bp + ".norm2.bias"])
        q2 = ops.gemm(ln2, w[bp + ".attn2.to_q.weight"])
        kt, vtt = self._text_kv[bp + ".attn2"]
        kw = {}
        o2 = torch.empty((M, C), dtype=f16, device=self.dev)
        if self._foreign is not None:
            self._foreign_attention(True, place, q2, kt, vtt, o2, S_q=S, keys_per_slot=77, n_src=B, d=d, heads=heads, F=F, BF=NB, scale=scale,
                                    src_index=[[b for b in range(B) for _ in range(F)]])
        else:
            if ctrl is not None and S <= 32 ** 2:
                kw = ctrl.cross_attn_args(place, S, heads, NB, F) or {}
            ops.attention(q2, kt, vtt, o2, S_q=S, keys_per_slot=77, n_src=B, d=d, heads=heads, F=F, BF=NB, scale=scale,
                          src_index=[[b for b in range(B) for _ in range(F)]], **kw)
        h = ops.gemm(o2, w[bp + ".attn2.to_out.0.weight"], bias=w[bp + ".attn2.to_out.0.bias"], residual=h)
        # ---- feed-forward (GEGLU)
        ln3 = ops.layernorm(h, w[bp + ".norm3.weight"], w[bp + ".norm3.bias"])
        g = ops.gemm(ln3, w[bp + ".ff.net.0.proj.weight"], bias=w[bp + ".ff.net.0.proj.bias"], geglu=True,
                     force_bn=w[bp + ".ff.net.0.proj.weight#bn"])
        h = ops.gemm(g, w[bp + ".ff.net.2.weight"], bias=w[bp + ".ff.net.2.bias"], residual=h)
        # ---- temporal attention over frames (models/attention.py:327-337), un-hooked
        po_bias = w[p + ".proj_out.bias"]
        if p + ".proj_out.bias#folded" in w:
            po_bias = w[p + ".proj_out.bias#folded"]  # to_out.weight == 0: the layer adds its bias only
        else:
            lnt = ops.layernorm(h, w[bp + ".norm_temporal.weight"], w[bp + ".norm_temporal.bias"])
            qkvt = ops.gemm(lnt, w[bp + ".attn_temporal.qkv"])
            if self.shard is not None:
                ot = self._temporal_attn_sharded(p, qkvt, B, F, S, heads, d, scale)
            else:
                ot = ops.temporal_attn(qkvt, B, F, S, heads, d, scale)
            h = ops.gemm(ot, w[bp + ".attn_temporal.to_out.0.weight"], bias=w[bp + ".attn_temporal.to_out.0.bias"], residual=h)
        out = ops.gemm(h, w[p + ".proj_out.weight"], bias=po_bias, residual=xr)
        return out.view(NB, H, W, C)

    def _foreign_attention(self, is_cross: bool, place: str, q, k, vt, o, **geo):
        """Slow path for a controller that only implements the reference protocol `controller(attn[BF, heads, s, t], is_cross, place)`
        (attention_register.py:49-51): the kernel materialises the fp16 probabilities of EVERY attention layer into a slab (STORE mode on
        all rows), the Python controller sees / edits that tensor, and a second launch multiplies the (possibly edited) slab with V
        (REPLACE mode).  This is the reference's own data flow (one probability tensor per layer in HBM) and costs what it costs there;
        the controllers of fatezero_b200.controllers never take this path."""
        BF, heads, S = geo["BF"], geo["heads"], geo["S_q"]
        T = len(geo["src_index"]) * geo["keys_per_slot"]
        ld = (T + 7) // 8 * 8
        slab = torch.zeros((BF, heads, S, ld), dtype=f16, device=self.dev)
        ops.attention(q, k, vt, o, edit_bf_start=0, row_mode=_lib.ATTN_STORE, store=slab, cache_ld=ld, **geo)
        view = slab[..., :T]
        new = self._foreign(view, is_cross, place)
        if new is not None and (new.data_ptr() != view.data_ptr() or new.shape != view.shape):
            view.copy_(new.reshape(view.shape))
        ops.attention(q, k, vt, o, edit_bf_start=0, row_mode=_lib.ATTN_REPLACE, base=slab, cache_ld=ld, **geo)

    def time_embedding(self, t: float) -> torch.Tensor:
        """time_proj + time_embedding + all time_emb_proj(SiLU(emb)) rows (unet_3d_condition.py:356-362; resnet.py:355)."""
        w = self.w
        c0 = self.ch[0]
        s = ops.timestep_sinusoid(t, c0, bool(self.cfg.get("flip_sin_to_cos", True)), float(self.cfg.get("freq_shift", 0)), self.dev)
        e = ops.rowvec_linear(s, w["time_embedding.linear_1.weight"], w["time_embedding.linear_1.bias"], False)
        emb = ops.rowvec_linear(e, w["time_embedding.linear_2.weight"], w["time_embedding.linear_2.bias"], True)
        return ops.rowvec_linear(emb, w["#temb_proj.weight"], w["#temb_proj.bias"], True)

    # ---------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x: torch.Tensor, t: float, text: torch.Tensor, ctrl=None) -> torch.Tensor:
        """x [B,4,F,H,W] (any float dtype, CUDA), text [B,77,D] -> eps [B,4,F,H,W] fp32."""
        self._foreign = None
        if ctrl is not None and not hasattr(ctrl, "self_attn_args"):
            if type(ctrl).__name__ in ("EmptyControl", "DummyController"):
                ctrl = None
            elif callable(ctrl):
                self._foreign, ctrl = ctrl, None  # reference-protocol controller: materialised-probability slow path
            else:
                raise NotImplementedError(
                    f"controller {type(ctrl).__name__} implements neither the fused-kernel protocol (self_attn_args / cross_attn_args) "
                    "nor the reference protocol __call__(attn, is_cross, place_in_unet)")
        w = self.w
        B, Cl, F, H, W = x.shape
        NB = B * F
        if text.shape[0] != B:
            raise ValueError(f"encoder_hidden_states batch {text.shape[0]} != sample batch {B}")
        self._ensure_text(text)
        groups = getattr(ctrl, "prompt_groups", 1) if ctrl is not None else 1
        if groups > 1 and self.shard is not None:
            raise NotImplementedError("a batched multi-prompt edit does not run frame-sharded")
        if groups > 1 and B % groups:
            raise ValueError(f"batch {B} does not split into {groups} prompt groups")
        self._images_per_item = NB // groups if groups > 1 else None
        if ctrl is not None:
            ctrl.begin_forward(B, F)
        temb_all = self.time_embedding(t)
        xf = x.to(f32).contiguous()
        cols = ops.im2col_latents(xf)
        c0 = self.ch[0]
        h = ops.gemm(cols, w["conv_in.weight"], bias=w["conv_in.bias"]).view(NB, H, W, c0)
        if self._has_temporal("conv_in"):
            h = self._temporal("conv_in", h, B, F)
        skips = [h]
        nblk = len(self.ch)
        lpb = self.cfg["layers_per_block"]
        for i, btype in enumerate(self.cfg["down_block_types"]):
            p = f"down_blocks.{i}"
            for j in range(lpb):
                h = self.resnet(f"{p}.resnets.{j}", h, temb_all, B, F)
                if btype.startswith("CrossAttn"):
                    h = self.transformer(f"{p}.attentions.{j}", h, B, F, "down", ctrl)
                skips.append(h)
            if i != nblk - 1:
                h = self.conv(f"{p}.downsamplers.0.conv", h, B, F, stride=2)
                skips.append(h)
        h = self.resnet("mid_block.resnets.0", h, temb_all, B, F)
        h = self.transformer("mid_block.attentions.0", h, B, F, "mid", ctrl)
        h = self.resnet("mid_block.resnets.1", h, temb_all, B, F)
        for i, btype in enumerate(self.cfg["up_block_types"]):
            p = f"up_blocks.{i}"
            for j in range(lpb + 1):
                h = ops.concat_channels(h, skips.pop())
                h = self.resnet(f"{p}.resnets.{j}", h, temb_all, B, F)
                if btype.startswith("CrossAttn"):
                    h = self.transformer(f"{p}.attentions.{j}", h, B, F, "up", ctrl)
            if i != nblk - 1:
                h = self.conv(f"{p}.upsamplers.0.conv", ops.upsample2x(h), B, F)
        NBh, Hh, Wh, Ch = h.shape
        n = self._gn_joint("conv_norm_out", h.view(NB, Hh * Wh, Ch), w["conv_norm_out.weight"], w["conv_norm_out.bias"], self.eps, F, True)
        co = self.cfg["out_channels"]
        # conv_out as one 16-wide MMA tile (first `co` channels valid); its bias precedes the temporal conv (resnet.py:64 then :76)
        y = ops.conv3x3(n.view(NB, Hh, Wh, Ch), w["conv_out.weight"], bias=w["conv_out.bias"])
        return self._finish(y.view(NB * Hh * Wh, 16), B, co, F, Hh, Wh)

    def _finish(self, y, B, co, F, H, W):
        w = self.w
        kw = {}
        if "conv_out.conv_temporal.down.weight" in w:
            if not self.lora_skip.get("conv_out", False):
                kw = dict(down=w["conv_out.conv_temporal.down.weight#f32"], up=w["conv_out.conv_temporal.up.weight#f32"])
        elif "conv_out.conv_temporal.weight" in w:
            kw = dict(w_full=w["conv_out.conv_temporal.weight#f32"], b_full=w["conv_out.conv_temporal.bias"])
        if self.shard is None or not kw:
            return ops.out_temporal(y, B, co, F, H, W, **kw)
        # frame-sharded: the conv_out tail (a 4-channel Conv1d pair over frames, 2-frame reach) runs on the gathered 16-channel rows of
        # the whole clip (131 KB per frame) and keeps this rank's frames
        rank, world, _ = self.shard
        ar = self.arena
        st = ops._stream()
        fb = H * W * 16 * 2
        Ft = F * world
        site = ar.site(("out_gather", B, F, H, W), B * Ft * fb)
        segs = [(y.data_ptr(), F * fb, r, ar.peer_ptr(r, site, rank * F * fb), Ft * fb, B, F * fb) for r in range(world)]
        ar.exchange(site, segs, range(world), st)
        full = ops.out_temporal(ar.tensor(site, 0, (B * Ft * H * W, 16)), B, co, Ft, H, W, **kw)
        return full[:, :, rank * F:(rank + 1) * F].contiguous()
