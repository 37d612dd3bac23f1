"""GPU parity of the fused attention kernel (all controller modes) against a PyTorch fp32 restatement of
prompt_attention/attention_register.py:23-59 + the controller arithmetic of attention_util.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from fatezero_b200 import _lib, ops

dev = "cuda"


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def make_inputs(BF, S, Sk, n_src, heads, d, seed=0, qscale=1.0):
    C_ = heads * d
    q = (rnd(BF * S, C_, seed=seed) * qscale).half()
    k = rnd(n_src * Sk, C_, seed=seed + 1).half()
    v = rnd(n_src * Sk, C_, seed=seed + 2).half()
    vt_ld = (Sk + 7) // 8 * 8
    vt = torch.zeros(n_src, heads, d, vt_ld, dtype=torch.float16, device=dev)
    vt[..., :Sk] = v.reshape(n_src, Sk, heads, d).permute(0, 2, 3, 1)
    return q, k, v, vt


def ref_probs(q, k, BF, S, Sk, heads, d, src_index, scale):
    """[BF, heads, S, n_slots*Sk] fp32 softmax probabilities, keys concatenated slot-major."""
    qh = q.float().reshape(BF, S, heads, d).permute(0, 2, 1, 3)
    kk = k.float().reshape(-1, Sk, heads, d)
    ks = torch.cat([kk[torch.tensor(si, device=dev)] for si in src_index], dim=1)  # [BF, slots*Sk, heads, d]
    s = torch.einsum("bhsd,bthd->bhst", qh, ks) * scale
    return torch.softmax(s, dim=-1)


def gather_v(v, Sk, heads, d, src_index):
    vv = v.float().reshape(-1, Sk, heads, d)
    return torch.cat([vv[torch.tensor(si, device=dev)] for si in src_index], dim=1)  # [BF, T, heads, d]


def pv(p, vs):
    o = torch.einsum("bhst,bthd->bshd", p, vs)
    return o.reshape(o.shape[0] * o.shape[1], -1)


def check(got, ref, report, key, atol, rtol=0.0):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs().max().item()
    report[key] = dict(max_abs=err, ref_max=ref.abs().max().item(), nan=bool(torch.isnan(got).any().item()))
    assert not torch.isnan(got).any(), f"{key}: NaN"
    assert err <= atol + rtol * ref.abs().max().item(), f"{key}: max_abs {err:.4g} (ref_max {ref.abs().max().item():.3g})"


SELF_CASES = [
    # BF, F, S, heads, d, index-list (per slot: source frame per query frame)
    (2, 2, 64, 8, 40, "own"),
    (2, 2, 256, 8, 160, "mid"),
    (3, 3, 1024, 8, 80, "mid"),
    (2, 2, 4096, 2, 40, "own"),
    (4, 4, 256, 4, 16, "prev_first"),
    (2, 2, 144, 4, 80, "prev_first"),
    (2, 2, 576, 2, 64, "mid"),
    # no hook, d <= 64, multiples of 128 keys: 1, 3, 5 and 10 128-key blocks, odd / even, one and two K/V frames
    (2, 2, 128, 2, 40, "own"),
    (3, 3, 384, 2, 48, "mid"),
    (2, 2, 640, 1, 40, "own"),
    (2, 2, 640, 2, 64, "prev_first"),
    (2, 2, 1024, 8, 40, "prev_first"),
]


def index_list(kind, F_, BF):
    B = BF // F_
    rows = []
    if kind == "own":
        rows.append([b * F_ + f for b in range(B) for f in range(F_)])
    elif kind == "mid":
        rows.append([b * F_ + (F_ - 1) // 2 for b in range(B) for f in range(F_)])
    else:
        rows.append([b * F_ + max(f - 1, 0) for b in range(B) for f in range(F_)])
        rows.append([b * F_ for b in range(B) for f in range(F_)])
    return rows


@pytest.mark.parametrize("BF,F_,S,heads,d,kind", SELF_CASES)
def test_self_plain(BF, F_, S, heads, d, kind, report):
    q, k, v, vt = make_inputs(BF, S, S, BF, heads, d, qscale=2.0)
    si = index_list(kind, F_, BF)
    out = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si)
    p = ref_probs(q, k, BF, S, S, heads, d, si, d ** -0.5)
    check(out, pv(p, gather_v(v, S, heads, d, si)), report, f"self_plain_{S}_{d}_{kind}", atol=4e-3, rtol=4e-3)


@pytest.mark.parametrize("ramp", ["up", "down", "spike"])
def test_self_plain_online_rescale(ramp, report):
    """Key blocks with growing / shrinking / one spiking scale: the row maximum sits in a late, an early or a single 128-key block, which
    random inputs alone never produce."""
    BF, F_, S, heads, d = 2, 2, 640, 2, 40
    q, k, v, vt = make_inputs(BF, S, S, BF, heads, d, seed=21, qscale=2.0)
    kk = k.float().reshape(BF, S, heads * d)
    for t in range(S // 128):
        f = {"up": 1.0 + 2.5 * t, "down": 1.0 + 2.5 * (S // 128 - 1 - t), "spike": 9.0 if t == 3 else 1.0}[ramp]
        kk[:, 128 * t:128 * (t + 1)] *= f
    k = kk.reshape(BF * S, heads * d).half()
    si = index_list("own", F_, BF)
    out = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si)
    p = ref_probs(q, k, BF, S, S, heads, d, si, d ** -0.5)
    check(out, pv(p, gather_v(v, S, heads, d, si)), report, f"self_plain_rescale_{ramp}", atol=4e-3, rtol=4e-3)


@pytest.mark.parametrize("BF,F_,S,heads,d,kind", [c for c in SELF_CASES if c[2] <= 1024])
def test_self_store_replace_blend(BF, F_, S, heads, d, kind, report):
    q, k, v, vt = make_inputs(BF, S, S, BF, heads, d, seed=3, qscale=2.0)
    si = index_list(kind, F_, BF)
    T = len(si) * S
    tag = f"{S}_{d}_{kind}"
    p = ref_probs(q, k, BF, S, S, heads, d, si, d ** -0.5)
    vs = gather_v(v, S, heads, d, si)
    # STORE (inversion: all rows)
    cache = torch.full((BF, heads, S, T), 7.0, dtype=torch.float16, device=dev)
    out = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si,
                  row_mode=_lib.ATTN_STORE, store=cache, cache_ld=T)
    check(cache, p, report, f"store_P_{tag}", atol=1.5e-3)
    check(out, pv(p.half().float(), vs), report, f"store_O_{tag}", atol=4e-3, rtol=4e-3)
    # REPLACE on the last half of the rows (edit_bf_start = BF//2), first half stays plain
    base = torch.softmax(rnd(BF - BF // 2, heads, S, T, seed=9) * 2, -1).half()
    out2 = torch.zeros_like(out)
    ops.attention(q, k, vt, out2, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si,
                  edit_bf_start=BF // 2, row_mode=_lib.ATTN_REPLACE, base=base, cache_ld=T)
    pe = p.clone()
    pe[BF // 2:] = base.float()
    check(out2, pv(pe, vs), report, f"replace_O_{tag}", atol=4e-3, rtol=4e-3)
    # BLEND
    mask = (rnd(BF - BF // 2, S, seed=11) > 0).float()
    out3 = torch.zeros_like(out)
    ops.attention(q, k, vt, out3, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si,
                  edit_bf_start=BF // 2, row_mode=_lib.ATTN_BLEND, base=base, cache_ld=T, mask=mask)
    pb = p.clone()
    m4 = mask[:, None, :, None]
    pb[BF // 2:] = m4 * p[BF // 2:].half().float() + (1 - m4) * base.float()
    check(out3, pv(pb, vs), report, f"blend_O_{tag}", atol=4e-3, rtol=4e-3)


def make_xedit(mode, alpha, eq, a, mapper, M):
    t = torch.zeros(_lib.XEDIT_FLOATS)
    t[0] = mode
    t[8:8 + 77] = alpha
    t[88:88 + 80] = 1.0
    t[88:88 + 77] = eq
    t[168:168 + 77] = a
    t[248:248 + 77] = mapper.float()
    mm = torch.zeros(80, 80)
    mm[:77, :77] = M
    t[328:] = mm.reshape(-1)
    return t.to(dev)


# (1, 4096, 8, 40) / (8, 4096, 8, 40): the step's own text cross-attention shapes at the 64x64 latents
@pytest.mark.parametrize("F_,S,heads,d", [(2, 64, 8, 160), (3, 256, 8, 40), (2, 1024, 8, 80), (2, 4096, 2, 40), (2, 144, 4, 16),
                                        (1, 4096, 8, 40), (8, 4096, 8, 40), (4, 1024, 8, 32)])
def test_cross(F_, S, heads, d, report):
    B = 2
    BF = B * F_
    q, k, v, vt = make_inputs(BF, S, 77, B, heads, d, seed=5, qscale=2.0)
    si = [[b for b in range(B) for f in range(F_)]]
    kw = dict(S_q=S, keys_per_slot=77, n_src=B, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si)
    p = ref_probs(q, k, BF, S, 77, heads, d, si, d ** -0.5)
    vs = gather_v(v, 77, heads, d, si)
    tag = f"{S}_{d}"
    out = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, **kw)
    check(out, pv(p, vs), report, f"cross_plain_{tag}", atol=4e-3, rtol=4e-3)
    if S > 1024:
        return
    # inversion-style STORE of all rows + running sum
    cache = torch.full((BF, heads, S, 80), 7.0, dtype=torch.float16, device=dev)
    acc = torch.zeros(BF, heads, S, 80, dtype=torch.float16, device=dev)
    acc[..., :77] = 0.25
    out1 = torch.zeros_like(out)
    ops.attention(q, k, vt, out1, **kw, row_mode=_lib.ATTN_STORE, store=cache, cache_ld=80, acc=acc)
    check(cache[..., :77], p, report, f"cross_store_P_{tag}", atol=1.5e-3)
    check(cache[..., 77:], torch.zeros_like(cache[..., 77:]), report, f"cross_store_pad_{tag}", atol=0)
    check(acc[..., :77], 0.25 + p.half().float(), report, f"cross_acc_{tag}", atol=1e-3)
    check(out1, pv(p.half().float(), vs), report, f"cross_store_O_{tag}", atol=4e-3, rtol=4e-3)
    # CROSSEDIT on cond rows (edit_bf_start = F)
    base = torch.zeros(F_, heads, S, 80, dtype=torch.float16, device=dev)
    base[..., :77] = torch.softmax(rnd(F_, heads, S, 77, seed=13) * 2, -1).half()
    alpha = (torch.arange(77) % 5 != 0).float()
    eq = torch.ones(77)
    eq[3] = 10.0
    a = (torch.arange(77) % 7 != 0).float()
    mapper = torch.cat([torch.tensor([0, 1, -1, 2, 3]), torch.arange(4, 76)])
    M = torch.eye(77)
    M[2, 2] = 0
    M[2, 3] = 0.5
    M[2, 4] = 0.5
    M[5, 5] = 0
    M[5, 6] = 1
    cur = p[F_:].half().float()
    bs = base[..., :77].float()
    for mode, name in ((0, "refine"), (1, "replace")):
        xe = make_xedit(mode, alpha, eq, a, mapper, M)
        acc2 = torch.zeros(F_, heads, S, 80, dtype=torch.float16, device=dev)
        out2 = torch.zeros_like(out)
        ops.attention(q, k, vt, out2, **kw, edit_bf_start=F_, row_mode=_lib.ATTN_CROSSEDIT, base=base, cache_ld=80, acc=acc2, xedit=xe)
        if mode == 0:
            R = bs[..., mapper.to(dev)] * a.to(dev) + cur * (1 - a.to(dev))
        else:
            R = torch.einsum("thpw,wn->thpn", bs, M.to(dev))
        R = R * eq.to(dev)
        new = (R * alpha.to(dev) + (1 - alpha.to(dev)) * cur).half().float()
        pe = p.clone()
        pe[F_:] = new
        check(out2, pv(pe, vs), report, f"cross_{name}_O_{tag}", atol=6e-3, rtol=6e-3)
        check(acc2[..., :77], cur, report, f"cross_{name}_acc_{tag}", atol=1e-3)


def test_limits_bf64_and_over(report):
    """The kernel's frame table holds kMaxBF = 64 (frame, batch) rows: 32 frames x CFG 2 is exactly the edge (it must work), 65 must be
    refused with an error (never a silent truncation)."""
    BF, F_, S, heads, d = 64, 32, 128, 2, 40
    q, k, v, vt = make_inputs(BF, S, S, BF, heads, d, qscale=2.0)
    si = index_list("mid", F_, BF)
    out = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si)
    p = ref_probs(q, k, BF, S, S, heads, d, si, d ** -0.5)
    check(out, pv(p, gather_v(v, S, heads, d, si)), report, "self_plain_bf64", atol=4e-3, rtol=4e-3)
    cache = torch.zeros(BF, heads, S, S, dtype=torch.float16, device=dev)
    out2 = torch.zeros_like(out)
    ops.attention(q, k, vt, out2, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F_, BF=BF, scale=d ** -0.5, src_index=si,
                  row_mode=_lib.ATTN_STORE, store=cache, cache_ld=S)
    check(cache, p, report, "store_bf64", atol=1.5e-3)
    BF = 65
    q, k, v, vt = make_inputs(BF, S, S, BF, heads, d)
    with pytest.raises(RuntimeError, match="BF=65"):
        ops.attention(q, k, vt, torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev), S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads,
                      F=65, BF=BF, scale=d ** -0.5, src_index=[list(range(BF))])
