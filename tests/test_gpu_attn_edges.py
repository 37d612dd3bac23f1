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
CROSSEDIT (Refine, Replace, pure Reweight; eq in {0, -1, 2.5, 10,   test_cross_edit
  0.5} on alpha = 0 / 1 / fractional words, fractional a, mapper
  -1, M with many-to-one / one-to-many columns and rows >= 64):
  the edited fp16 P read through a one-hot V ("probe") against
  the fp64 edit of the stored P (check_edit), cur == stored P
  bitwise at alpha = 0, O with random V; d in {40, 80, 160, 192},
  S_q in {64, 65, 129, 256, 1024}, keys_per_slot in {77, 16, 80},
  edit_bf_start > 0 (un-hooked rows in the same launch)
fp16 running sums of STORE and CROSSEDIT: bitwise acc + stored P    test_cross_edit, test_running_sum_steps
  (the pre-edit P), pad columns up to acc_ld in {80, 96}
  unchanged, a NaN guard frame after the slab untouched (S_q tails
  65 / 129: no second add onto row S_q - 1); 20 steps replayed in
  fp16 on the host, sums past 8
grouped launches with a slab per group: STORE groups with their     test_cross_edit_grouped
  own cache and running sum, CROSSEDIT groups with their own
  table, source map and running sum, each against its fp64 edit
host-side refusals: d = 200, 5 slots, cache_ld that does not        test_refusals
  split into n_slots runs of >= keys_per_slot keys; CROSSEDIT at
  keys_per_slot = 81, over two slots, without tables; a running
  sum over two slots (nothing written)
temporal attention: F in {1, 3, 5, 16, 24, 28, 32} x d in           test_temporal_attn, test_temporal_attn_refuses_33_frames
  {40, 80, 160} (generic kernel); F = 33 refused
pixel-major temporal attention (F in {2, 4, 8}): head groups hg =   test_temporal_attn
  8 / 4 / 2 (d = 40 / 80 / 160), 1 (d = 320), 6 -> 4 (d = 48),
  5 -> 1 (d = 64, 7 heads), 40 -> 32 (d = 8, 256 rows per warp),
  3 (d = 16); grid stride at B = 2, HW = 4096; F = 8 falling back
  to the generic kernel (d = 20, 328); sharp rows (qscale 4);
  identical frames (O == V bitwise)
"""
import pytest
import torch

from _ref64 import X_ALPHA, check_attn, check_edit, check_probs, check_running_sum, cross_edit_ref, cross_edit_table, softmax64, ulp16

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
        return {**dict(S_q=self.S_q, keys_per_slot=self.kps, n_src=self.n_src, d=self.d, heads=self.heads, F=self.BF, BF=self.BF,
                       scale=self.scale, src_index=self.si), **extra}

    def run(self, vt=None, **extra):
        out = torch.full((self.BF * self.S_q, self.heads * self.d), float("nan"), dtype=torch.float16, device=dev)
        ops.attention(self.q, self.k, self.vt if vt is None else vt, out, **self.kw(**extra))
        return out.view(self.BF, self.S_q, self.heads, self.d).permute(0, 2, 1, 3)  # [BF, heads, S_q, d]

    def gather(self, x):
        """x [n_src * kps, heads * d] -> [BF, heads, T, d] fp64, keys concatenated slot-major (the kernel's key order)."""
        xx = x.double().view(self.n_src, self.kps, self.heads, self.d)
        g = torch.cat([xx[torch.tensor(row, device=dev)] for row in self.si], dim=1)
        return g.permute(0, 2, 1, 3)

    def probe(self, off):
        """V^T whose head-dim column j is one-hot at key off + j: output column j of a row is then that row's fp16 P at key off + j exactly
        (one non-zero product; hooked rows are not rescaled)."""
        vt = torch.zeros_like(self.vt)
        j = torch.arange(min(self.d, self.kps - off), device=dev)
        vt[:, :, j, j + off] = 1.0
        return vt

    def probed(self, **extra):
        """The fp16 P the kernel multiplies with V, [BF, heads, S_q, kps], read through probe launches (one per d keys)."""
        return torch.cat([self.run(vt=self.probe(off), **extra)[..., :min(self.d, self.kps - off)] for off in range(0, self.kps, self.d)], -1)

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


# ------------------------------------------------------------------------------------------------------- CROSSEDIT and running sums
def guarded_acc(Fc, heads, S_q, acc_ld, seed):
    """Running-sum slab acc [Fc, heads, S_q, 80] as a view of big [Fc + 1, heads, S_q, acc_ld]: frame Fc is a NaN guard, every column of
    big[:Fc] (the pad columns past the keys included) starts finite and positive (a -0 pad would legitimately become +0)."""
    big = torch.full((Fc + 1, heads, S_q, acc_ld), float("nan"), dtype=torch.float16, device=dev)
    big[:Fc] = (0.25 + 7.5 * torch.rand(Fc, heads, S_q, acc_ld, generator=torch.Generator().manual_seed(seed))).half()
    return big, big[:Fc, :, :, :80]


def check_acc(big, old, Fc, p16, kps, report, key):
    check_running_sum(big[:Fc], old[:Fc], p16, kps, report, key)
    assert torch.isnan(big[Fc]).all(), f"{key}: the running sum wrote past its slab"


def source_map(Fc, heads, S_q, cache_ld, kps, seed):
    """Cached source map slab as the inversion leaves it: fp16 rows over kps keys, zero pad up to cache_ld."""
    base = torch.zeros(Fc, heads, S_q, cache_ld, dtype=torch.float16, device=dev)
    base[..., :kps] = torch.softmax(rnd(Fc, heads, S_q, kps, seed=seed) * 2, -1).half()
    return base


def check_cross_edit(edited, p_store, base, table, kps, report, tag):
    """edited [Fc, heads, S_q, kps]: the fp16 P a CROSSEDIT launch multiplied with V, p_store the STORE launch's P of the same rows.
    Where alpha = 0 the edit is cur itself, so edited == P_store there proves cur == P_store (both launches take the same two-pass path);
    the fp64 edit is then built from P_store."""
    keep = (table[X_ALPHA:X_ALPHA + kps] == 0).to(dev)
    a, b = edited[..., keep], p_store[..., :kps][..., keep]
    diff = int((a != b).sum().item())
    report[f"xedit_cur_bitwise_{tag}"] = dict(n=a.numel(), mismatches=diff,
                                              max_ulps=((a.double() - b.double()).abs() / ulp16(b.double())).max().item())
    assert diff == 0, f"{tag}: cur differs from the stored P in {diff} elements at alpha = 0"
    ref, terms = cross_edit_ref(p_store, base, table, kps)
    check_edit(edited, ref, terms, report, f"xedit_P_{tag}")
    return ref


# d, S_q, keys_per_slot, heads, BF, edit_bf_start, running-sum row stride (acc_ld)
XEDIT_CASES = [
    (40, 256, 77, 8, 3, 1, 80),    # d = 40: two probe launches (keys 0..39, 40..76)
    (80, 1024, 77, 2, 3, 1, 80),
    (160, 256, 77, 2, 2, 0, 96),   # NCH = 3
    (160, 64, 80, 2, 3, 1, 80),    # keys_per_slot = 80: the CROSSEDIT limit
    (192, 65, 77, 1, 3, 1, 96),    # S_q tail in warpgroup 1
    (192, 129, 77, 1, 2, 1, 80),   # S_q tail in warpgroup 0 of the second CTA
    (80, 129, 16, 2, 3, 2, 80),    # one masked key atom
    (40, 65, 80, 2, 2, 0, 96),
]


@pytest.mark.parametrize("kind", ["refine", "replace", "reweight"])
@pytest.mark.parametrize("d,S_q,kps,heads,BF,start,acc_ld", XEDIT_CASES)
def test_cross_edit(d, S_q, kps, heads, BF, start, acc_ld, kind, report):
    """STORE (+ running sum) and CROSSEDIT (+ running sum) on the same Q / K: the stored P within 1 ulp of fp16(softmax64), both running
    sums bitwise acc + P_store (the pre-edit P), the edited P (probe V) against the fp64 edit of P_store, O (random V) against P_edit V."""
    Fc, cache_ld = BF - start, (kps + 7) // 8 * 8
    c = Case(BF, S_q, kps, 2, heads, d, [[bf % 2 for bf in range(BF)]], seed=10, qscale=2.0)
    tag = f"{kind}_d{d}_sq{S_q}_kps{kps}_start{start}_ld{acc_ld}"
    p = c.probs()
    store = torch.full((Fc, heads, S_q, cache_ld), 7.0, dtype=torch.float16, device=dev)
    big, acc = guarded_acc(Fc, heads, S_q, acc_ld, seed=1)
    old = big.clone()
    c.run(edit_bf_start=start, row_mode=_lib.ATTN_STORE, store=store, cache_ld=cache_ld, acc=acc)
    check_probs(store[..., :kps], p[start:], report, f"xedit_store_P_{tag}")
    check_acc(big, old, Fc, store, kps, report, f"xedit_store_acc_{tag}")

    base = source_map(Fc, heads, S_q, cache_ld, kps, seed=11)
    table = cross_edit_table(kind, kps)
    hook = dict(edit_bf_start=start, row_mode=_lib.ATTN_CROSSEDIT, base=base, cache_ld=cache_ld, xedit=table.to(dev))
    pe = p.clone()
    pe[start:] = check_cross_edit(c.probed(**hook)[start:], store, base, table, kps, report, tag)

    big, acc = guarded_acc(Fc, heads, S_q, acc_ld, seed=2)
    old = big.clone()
    got = c.run(**hook, acc=acc)
    check_acc(big, old, Fc, store, kps, report, f"xedit_acc_{tag}")
    check_attn(got, pe, c.gather(c.v), report, f"xedit_O_{tag}")


def test_cross_edit_grouped(report):
    """The batched inversion and edit of several clips: one launch of STORE groups, each with its own cache and running-sum slab, then one
    of CROSSEDIT groups, each with its own table, cached source slab and running sum; every group checked against its own fp64 reference."""
    d, S_q, kps, heads, Fr, start = 80, 129, 77, 2, 2, 1
    kinds = ["refine", "replace", "reweight"]
    G = len(kinds)
    BF = start + G * Fr
    c = Case(BF, S_q, kps, G + 1, heads, d, [[0] + [1 + g for g in range(G) for _ in range(Fr)]], seed=12, qscale=2.0)
    p = c.probs()
    rows = [slice(start + g * Fr, start + (g + 1) * Fr) for g in range(G)]
    geo = dict(edit_bf_start=start, cache_ld=80, F=Fr)

    stores = [torch.full((Fr, heads, S_q, 80), 7.0, dtype=torch.float16, device=dev) for _ in range(G)]
    accs = [guarded_acc(Fr, heads, S_q, 80, seed=20 + g) for g in range(G)]
    olds = [big.clone() for big, _ in accs]
    c.run(**geo, groups=[dict(row_mode=_lib.ATTN_STORE, store=s, acc=a) for s, (_, a) in zip(stores, accs)])
    for g in range(G):
        check_probs(stores[g][..., :kps], p[rows[g]], report, f"grouped_store_P_{g}")
        check_acc(accs[g][0], olds[g], Fr, stores[g], kps, report, f"grouped_store_acc_{g}")

    bases = [source_map(Fr, heads, S_q, 80, kps, seed=30 + g) for g in range(G)]
    tables = [cross_edit_table(k, kps) for k in kinds]
    groups = [dict(row_mode=_lib.ATTN_CROSSEDIT, xedit=t.to(dev), base=b) for t, b in zip(tables, bases)]
    edited = c.probed(**geo, groups=groups)
    pe = p.clone()
    for g in range(G):
        pe[rows[g]] = check_cross_edit(edited[rows[g]], stores[g], bases[g], tables[g], kps, report, f"grouped_{kinds[g]}")

    accs = [guarded_acc(Fr, heads, S_q, 80, seed=40 + g) for g in range(G)]
    olds = [big.clone() for big, _ in accs]
    got = c.run(**geo, groups=[dict(gr, acc=a) for gr, (_, a) in zip(groups, accs)])
    for g in range(G):
        check_acc(accs[g][0], olds[g], Fr, stores[g], kps, report, f"grouped_xedit_acc_{g}")
    check_attn(got, pe, c.gather(c.v), report, "grouped_xedit_O")


def test_running_sum_steps(report):
    """20 STORE steps into one running sum, fresh Q / K each step (sharp rows), replayed on the host in fp16: bitwise equal, with sums past 8
    so the coarse binades round too."""
    BF, S_q, kps, heads, d = 2, 65, 77, 2, 64
    big, acc = guarded_acc(BF, heads, S_q, 80, seed=3)
    host = big[:BF].cpu()
    store = torch.empty(BF, heads, S_q, 80, dtype=torch.float16, device=dev)
    for step in range(20):
        c = Case(BF, S_q, kps, BF, heads, d, [[0, 1]], seed=100 + step, qscale=4.0)
        c.run(row_mode=_lib.ATTN_STORE, store=store, cache_ld=80, acc=acc)
        host[..., :kps] = host[..., :kps] + store[..., :kps].cpu()
    got = big[:BF].cpu()
    report["running_sum_20_steps"] = dict(n=got.numel(), mismatches=int((got != host).sum().item()), max=host.max().item(),
                                          above_8=int((host[..., :kps] > 8).sum().item()))
    assert torch.equal(got, host), "running sum after 20 steps differs from the fp16 replay"
    assert torch.isnan(big[BF]).all()
    assert report["running_sum_20_steps"]["above_8"] > 100


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
    # CROSSEDIT past 80 keys, over two slots, without tables; a running sum over two slots
    xe = cross_edit_table("refine", 64).to(dev)
    acc = torch.zeros(2, 1, 64, 88, dtype=torch.float16, device=dev)
    c = Case(2, 64, 81, 2, 1, 64, [[0, 1]])
    with pytest.raises(RuntimeError, match="CROSSEDIT needs tables, one slot, <= 80 keys"):
        c.run(row_mode=_lib.ATTN_CROSSEDIT, base=torch.zeros(2, 1, 64, 88, dtype=torch.float16, device=dev), cache_ld=88, xedit=xe, acc=acc)
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1], [1, 0]])
    with pytest.raises(RuntimeError, match="CROSSEDIT needs tables, one slot, <= 80 keys"):
        c.run(row_mode=_lib.ATTN_CROSSEDIT, base=cache, cache_ld=128, xedit=xe)
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1]])
    with pytest.raises(RuntimeError, match="CROSSEDIT needs tables, one slot, <= 80 keys"):
        c.run(row_mode=_lib.ATTN_CROSSEDIT, base=cache, cache_ld=128, acc=acc)
    c = Case(2, 64, 64, 2, 1, 64, [[0, 1], [1, 0]])
    with pytest.raises(RuntimeError, match="running sum only for single-slot maps"):
        c.run(row_mode=_lib.ATTN_STORE, store=cache, cache_ld=128, acc=acc)
    torch.cuda.synchronize()
    assert torch.all(cache == 0), "a refused call wrote the cache"
    assert torch.all(acc == 0), "a refused call wrote the running sum"


# ------------------------------------------------------------------------------------------------------------------ temporal attention
# B, F, HW, heads, d, qscale, frames ("rnd", or "same": every frame of a pixel identical).  F in {2, 4, 8} with d % 8 == 0 and d <= 320
# runs the pixel-major kernel, whose warp takes hg heads (hg = min(heads, 320 / d), decremented until it divides heads); the rest the
# generic one.
TEMPORAL_CASES = {f"{Fr}-{d}": (1, Fr, 24, 8, d, 1.0, "rnd") for Fr in (1, 2, 3, 4, 5, 8, 16, 24, 28, 32) for d in (40, 80, 160)}
TEMPORAL_CASES.update({f"F{Fr}-h{heads}-d{d}": (1, Fr, 24, heads, d, 1.0, "rnd") for Fr in (2, 4, 8)
                       for heads, d in ((2, 320), (8, 48), (7, 64), (64, 8), (3, 16))})  # hg = 1, 6 -> 4, 5 -> 1, 40 -> 32, 3
TEMPORAL_CASES.update({
    "grid-stride": (2, 8, 4096, 8, 40, 1.0, "rnd"),  # 8192 warp items, more than the launch's grid x 4 warps
    "F8-generic-d20": (1, 8, 24, 8, 20, 1.0, "rnd"),
    "F8-generic-d328": (1, 8, 24, 2, 328, 1.0, "rnd"),
    **{f"sharp-F{Fr}": (1, Fr, 24, 8, 80, 4.0, "rnd") for Fr in (2, 4, 8)},
    **{f"same-F{Fr}": (1, Fr, 24, 8, 40, 1.0, "same") for Fr in (2, 4, 8)},
})


@pytest.mark.parametrize("B,Fr,HW,heads,d,qscale,frames", TEMPORAL_CASES.values(), ids=TEMPORAL_CASES.keys())
def test_temporal_attn(B, Fr, HW, heads, d, qscale, frames, report):
    Cc = heads * d
    qkv = rnd(B * Fr * HW, 3 * Cc, seed=8)
    qkv[:, :Cc] *= qscale
    if frames == "same":
        qkv = qkv.view(B, Fr, HW, 3 * Cc)[:, :1].expand(B, Fr, HW, 3 * Cc).reshape(-1, 3 * Cc)
    qkv = qkv.half()
    out = ops.temporal_attn(qkv, B, Fr, HW, heads, d, d ** -0.5)
    t = qkv.double().view(B, Fr, HW, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # [3, B, HW, heads, F, d]
    p = softmax64(t[0] @ t[1].transpose(-1, -2) * f32(d ** -0.5))
    got = out.view(B, Fr, HW, heads, d).permute(0, 2, 3, 1, 4)
    check_attn(got, p, t[2], report, f"temporal_B{B}_F{Fr}_HW{HW}_h{heads}_d{d}_qs{qscale}_{frames}")
    if frames == "same":  # every score is the row maximum: P = fp16(1 / F) = 1 / F exactly (__expf(0) = 1), so O = V bitwise
        assert torch.equal(out, qkv[:, 2 * Cc:]), "identical frames: O differs from V"


def test_temporal_attn_refuses_33_frames():
    qkv = torch.zeros(33 * 4, 3 * 64, dtype=torch.float16, device=dev)
    with pytest.raises(RuntimeError, match="F=33"):
        ops.temporal_attn(qkv, 1, 33, 4, 1, 64, 0.125)
