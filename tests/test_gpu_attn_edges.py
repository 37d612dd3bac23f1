"""Edge cases of the fused attention (fz_attn.cu) and the temporal attention (fz_elem.cu) against fp64 references of
softmax(scale Q K^T) V built from the same fp16 Q, K and V (tests/_ref64.py).

Code path                                                          reached by
-----------------------------------------------------------------  ----------------------------------------------------------------
3 and 4 K/V slots (kMaxSlots = 4), duplicated source frames,       test_plain_slots
  keys_per_slot in {144, 80, 16} (partial last atom of each slot)
head dims 8, 64, 128, 192 (1-3 chunks), S_q in {16, 65, 129}        test_plain_head_dim
  (S_q < 64: warpgroup 1 idle), one-hot rows whose maximum grows
  by more than 2^8 between key atoms (online-softmax rescale)
STORE: P within 1 ulp of fp16(softmax64), 3-4 slots, hooked and     test_store
  un-hooked rows in one launch (edit_bf_start > 0)
REPLACE / BLEND at d = 192 (tightest shared-memory plan), 3-4       test_replace_blend
  slots, keys_per_slot = 144
causal masking (CLIP: L in {77, 64, 130}, vt_ld padded)             test_causal
host-side refusals: d = 200, 5 slots, cache_ld that does not        test_refusals
  split into n_slots runs of >= keys_per_slot keys
temporal attention: F in {1, 3, 5, 16, 24, 28, 32} x d in           test_temporal_attn, test_temporal_attn_refuses_33_frames
  {40, 80, 160}; F = 33 refused
"""
import pytest
import torch

from _ref64 import check_attn, check_probs, softmax64

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from fatezero_b200 import _lib, ops

dev = "cuda"


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def f32(x: float) -> float:
    """The value the kernel sees for a float argument (passed as a C float)."""
    return torch.tensor(x, dtype=torch.float32).item()


class Case:
    """fp16 inputs of one attention launch and their fp64 reference."""

    def __init__(self, BF, S_q, kps, n_src, heads, d, src_index, seed=0, qscale=1.0, key_ramp=None):
        self.BF, self.S_q, self.kps, self.n_src, self.heads, self.d, self.si = BF, S_q, kps, n_src, heads, d, src_index
        Cc = heads * d
        self.q = (rnd(BF * S_q, Cc, seed=seed) * qscale).half()
        k = rnd(n_src * kps, Cc, seed=seed + 1)
        if key_ramp is not None:  # scale key atom j by key_ramp(j): the row maximum grows from atom to atom
            k = k.view(n_src, kps, Cc)
            for j in range((kps + 63) // 64):
                k[:, 64 * j:64 * (j + 1)] *= key_ramp(j)
            k = k.reshape(n_src * kps, Cc)
        self.k = k.half()
        self.v = rnd(n_src * kps, Cc, seed=seed + 2).half()
        self.vt_ld = (kps + 7) // 8 * 8
        self.vt = torch.zeros(n_src, heads, d, self.vt_ld, dtype=torch.float16, device=dev)
        self.vt[..., :kps] = self.v.view(n_src, kps, heads, d).permute(0, 2, 3, 1)
        self.scale = d ** -0.5
        self.T = len(src_index) * kps

    def kw(self, **extra):
        return dict(S_q=self.S_q, keys_per_slot=self.kps, n_src=self.n_src, d=self.d, heads=self.heads, F=self.BF, BF=self.BF,
                    scale=self.scale, src_index=self.si, **extra)

    def run(self, **extra):
        out = torch.full((self.BF * self.S_q, self.heads * self.d), float("nan"), dtype=torch.float16, device=dev)
        ops.attention(self.q, self.k, self.vt, out, **self.kw(**extra))
        return out.view(self.BF, self.S_q, self.heads, self.d).permute(0, 2, 1, 3)  # [BF, heads, S_q, d]

    def gather(self, x):
        """x [n_src * kps, heads * d] -> [BF, heads, T, d] fp64, keys concatenated slot-major (the kernel's key order)."""
        xx = x.double().view(self.n_src, self.kps, self.heads, self.d)
        g = torch.cat([xx[torch.tensor(row, device=dev)] for row in self.si], dim=1)
        return g.permute(0, 2, 1, 3)

    def probs(self, causal=False):
        q = self.q.double().view(self.BF, self.S_q, self.heads, self.d).permute(0, 2, 1, 3)
        s = q @ self.gather(self.k).transpose(-1, -2) * f32(self.scale)
        if causal:
            s = s.masked_fill(torch.ones(self.S_q, self.T, dtype=torch.bool, device=dev).triu(1), -float("inf"))
        return softmax64(s)


# -------------------------------------------------------------------------------------------------------------- plain (un-hooked) rows
# BF, S_q, keys_per_slot, heads, d, src_index (per slot: K/V source frame per query frame)
SLOT_CASES = [
    (3, 144, 144, 2, 40, [[0, 1, 2], [1, 1, 1], [0, 0, 2]]),
    (2, 80, 80, 2, 64, [[0, 1], [1, 0], [0, 0], [1, 1]]),
    (3, 16, 16, 1, 80, [[0, 1, 2], [2, 2, 2], [1, 0, 1], [0, 0, 0]]),
    (2, 100, 16, 2, 160, [[1, 0], [1, 1], [0, 1]]),
]


@pytest.mark.parametrize("BF,S_q,kps,heads,d,si", SLOT_CASES)
def test_plain_slots(BF, S_q, kps, heads, d, si, report):
    c = Case(BF, S_q, kps, BF, heads, d, si, seed=1, qscale=2.0)
    got = c.run()
    check_attn(got, c.probs(), c.gather(c.v), report, f"plain_{len(si)}slots_kps{kps}_d{d}")


# d, S_q, qscale: qscale 8 with keys scaled up atom by atom makes nearly one-hot rows whose maximum jumps by more than 2^8 (the rescale
# threshold, in log2 units) between atoms
HEAD_DIM_CASES = [(8, 16, 1), (8, 129, 8), (64, 65, 8), (64, 16, 1), (128, 129, 1), (128, 65, 8), (192, 16, 8), (192, 65, 1), (192, 129, 8)]


@pytest.mark.parametrize("d,S_q,qscale", HEAD_DIM_CASES)
def test_plain_head_dim(d, S_q, qscale, report):
    kps = 300
    c = Case(1, S_q, kps, 1, 1, d, [[0]], seed=2, qscale=qscale, key_ramp=(lambda j: 1.0 + 0.5 * j) if qscale > 1 else None)
    got = c.run()
    p = c.probs()
    if qscale > 1:  # the case must actually drive the rescale: a later atom's maximum exceeds the first atom's by > 8 (log2)
        s = torch.log2(p)
        first, rest = s[..., :64].amax(-1), s[..., 64:].amax(-1)
        assert ((rest - first) > 8).float().mean().item() > 0.5
    check_attn(got, p, c.gather(c.v), report, f"plain_d{d}_sq{S_q}_qs{qscale}")


# ----------------------------------------------------------------------------------------------------------------------------- STORE
# BF, S_q, keys_per_slot, heads, d, src_index, edit_bf_start
STORE_CASES = [
    (3, 144, 144, 2, 64, [[0, 1, 2], [1, 1, 1], [0, 0, 2]], 1),
    (2, 65, 80, 1, 192, [[0, 1], [1, 0], [0, 0], [1, 1]], 0),
    (4, 129, 16, 2, 40, [[0, 1, 2, 3], [3, 3, 3, 3], [1, 1, 0, 0]], 2),
]


@pytest.mark.parametrize("BF,S_q,kps,heads,d,si,start", STORE_CASES)
def test_store(BF, S_q, kps, heads, d, si, start, report):
    c = Case(BF, S_q, kps, BF, heads, d, si, seed=3, qscale=2.0)
    cache = torch.full((BF - start, heads, S_q, c.T), 7.0, dtype=torch.float16, device=dev)
    got = c.run(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=cache, cache_ld=c.T)
    p = c.probs()
    tag = f"{len(si)}slots_kps{kps}_d{d}_start{start}"
    check_probs(cache, p[start:], report, f"store_P_{tag}")
    check_attn(got, p, c.gather(c.v), report, f"store_O_{tag}")


# ------------------------------------------------------------------------------------------------------------------- REPLACE and BLEND
@pytest.mark.parametrize("mode", ["replace", "blend"])
@pytest.mark.parametrize("si", [[[0, 1, 2], [1, 1, 1], [2, 0, 0]], [[0, 1, 2], [2, 2, 2], [1, 0, 1], [0, 0, 0]]], ids=["3slots", "4slots"])
def test_replace_blend(si, mode, report):
    BF, S_q, kps, heads, d, start = 3, 130, 144, 1, 192, 1
    c = Case(BF, S_q, kps, BF, heads, d, si, seed=4, qscale=2.0)
    base = torch.softmax(rnd(BF - start, heads, S_q, c.T, seed=5) * 3, -1).half()
    p = c.probs()
    pe = p.clone()
    if mode == "replace":
        got = c.run(edit_bf_start=start, row_mode=_lib.ATTN_REPLACE, base=base, cache_ld=c.T)
        pe[start:] = base.double()
    else:
        mask = (rnd(BF - start, S_q, seed=6) > 0).float()
        got = c.run(edit_bf_start=start, row_mode=_lib.ATTN_BLEND, base=base, cache_ld=c.T, mask=mask)
        m = mask.double()[:, None, :, None]
        pe[start:] = m * p[start:] + (1 - m) * base.double()
    check_attn(got, pe, c.gather(c.v), report, f"{mode}_{len(si)}slots_d{d}")


# ---------------------------------------------------------------------------------------------------------------------------- causal
@pytest.mark.parametrize("L", [77, 64, 130])
def test_causal(L, report):
    """The CLIP text encoder's call: q and k are column slices of one [B L, 2 C] buffer, V^T padded to a multiple of 8 keys."""
    B, heads, d = 2, 2, 64
    Cc = heads * d
    c = Case(B, L, L, B, heads, d, [list(range(B))], seed=7, qscale=2.0)
    qk = torch.cat([c.q, c.k], dim=1)
    out = torch.full((B * L, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(qk[:, :Cc], qk[:, Cc:], c.vt, out, **c.kw(causal=True))
    got = out.view(B, L, heads, d).permute(0, 2, 1, 3)
    check_attn(got, c.probs(causal=True), c.gather(c.v), report, f"causal_L{L}")


# -------------------------------------------------------------------------------------------------------------------------- refusals
def test_refusals():
    """Every refusal fails in the host-side argument checks, before any launch."""
    c = Case(2, 64, 64, 2, 1, 200, [[0, 1]])
    with pytest.raises(RuntimeError, match="head dim 200"):
        c.run()
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1]] * 5)
    with pytest.raises(RuntimeError, match="n_slots=5"):
        c.run()
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1], [1, 0]])
    cache = torch.zeros(2, 1, 64, 128, dtype=torch.float16, device=dev)
    # 2 slots of 64 keys in rows of 112: each slot's run would be cut to 56 keys
    with pytest.raises(RuntimeError, match="cache_ld"):
        c.run(row_mode=_lib.ATTN_STORE, store=cache, cache_ld=112)
    with pytest.raises(RuntimeError, match="cache_ld"):
        c.run(row_mode=_lib.ATTN_REPLACE, base=cache, cache_ld=112)
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1], [1, 0], [0, 0]])
    with pytest.raises(RuntimeError, match="cache_ld"):
        c.run(row_mode=_lib.ATTN_STORE, store=torch.zeros(2, 1, 64, 200, dtype=torch.float16, device=dev), cache_ld=200)
    torch.cuda.synchronize()
    assert torch.all(cache == 0), "a refused call wrote the cache"


# ------------------------------------------------------------------------------------------------------------------ temporal attention
@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("Fr", [1, 3, 5, 16, 24, 28, 32])
def test_temporal_attn(Fr, d, report):
    B, HW, heads = 1, 24, 8
    Cc = heads * d
    qkv = rnd(B * Fr * HW, 3 * Cc, seed=8).half()
    out = ops.temporal_attn(qkv, B, Fr, HW, heads, d, d ** -0.5)
    t = qkv.double().view(B, Fr, HW, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # [3, B, HW, heads, F, d]
    p = softmax64(t[0] @ t[1].transpose(-1, -2) * f32(d ** -0.5))
    got = out.view(B, Fr, HW, heads, d).permute(0, 2, 3, 1, 4)
    check_attn(got, p, t[2], report, f"temporal_F{Fr}_d{d}")


def test_temporal_attn_refuses_33_frames():
    qkv = torch.zeros(33 * 4, 3 * 64, dtype=torch.float16, device=dev)
    with pytest.raises(RuntimeError, match="F=33"):
        ops.temporal_attn(qkv, 1, 33, 4, 1, 64, 0.125)
