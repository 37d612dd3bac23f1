"""Batch invariance of the multi-prompt edit: for every prompt, the batched pass computes bit for bit what editing that prompt alone
computes.  Kernel level: the grouped attention (fz_attention_grouped_f16) against one fz_attention_f16 launch per group, the batched
GroupNorm and CFG/DDIM step against per-item calls, and the tap-GEMM against every BLOCK_N (pick_block_n depends on the row count, so
the text K/V projections of a batch of K prompts may pick another BLOCK_N than a single prompt's).  Pipeline level:
p2preplace_edit_batch against the single-prompt pipe(edit_type="swap") runs against the same inversion store."""
import tempfile

import pytest
import torch

from _ref64 import check_attn, softmax64

pytestmark = pytest.mark.gpu

from _helpers import GOLDEN_DIR, build_product, case_inputs, run_product_case  # noqa: E402
from oracle.cases import CASES, SRC  # noqa: E402

if torch.cuda.is_available():
    from fatezero_b200 import _lib, controllers, ops

dev = "cuda"


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def src_rows(kind, F, B):
    if kind == "mid":
        return [[b * F + (F - 1) // 2 for b in range(B) for f in range(F)]]
    return [[b * F + max(f - 1, 0) for b in range(B) for f in range(F)], [b * F for b in range(B) for f in range(F)]]  # [-1, 'first']


def group_rows(K, F, g):
    """rows of prompt g in the batch [uncond_1..K ; cond_1..K]: its uncond block and its cond block"""
    return list(range(g * F, (g + 1) * F)) + list(range((K + g) * F, (K + g + 1) * F))


def rows_of(t, rows, S):
    return torch.cat([t[r * S:(r + 1) * S] for r in rows])


# ------------------------------------------------------------------------------------------------ grouped self-attention
SELF_MODES = ["replace", "none", "blend", "replace"]


@pytest.mark.parametrize("kind", ["mid", "prev_first"])
@pytest.mark.parametrize("S", [256, 1024])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_grouped_self_bitwise(d, S, kind, report):
    K, F, heads = len(SELF_MODES), 2, 2
    BF = 2 * K * F
    si = src_rows(kind, F, 2 * K)
    T = len(si) * S
    Cc = heads * d
    q, k, v = rnd(BF * S, Cc, seed=1, scale=2.0).half(), rnd(BF * S, Cc, seed=2).half(), rnd(BF * S, Cc, seed=3).half()
    vt = v.view(BF, S, heads, d).permute(0, 2, 3, 1).contiguous()
    base = torch.softmax(rnd(F, heads, S, T, seed=4) * 3, -1).half()
    masks = [(rnd(F, S, seed=10 + g) > 0.3 * g).float().contiguous() for g in range(K)]
    mode = {"none": _lib.ATTN_NONE, "replace": _lib.ATTN_REPLACE, "blend": _lib.ATTN_BLEND}
    groups = [dict(row_mode=mode[m], mask=masks[g] if m == "blend" else None) for g, m in enumerate(SELF_MODES)]
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    geo = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, scale=d ** -0.5)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, edit_bf_start=K * F, base=base, cache_ld=T, groups=groups, **geo)
    plain = torch.full_like(out, float("nan"))
    ops.attention(q, k, vt, plain, F=F, BF=BF, src_index=si, **geo)
    assert torch.equal(out[:K * F * S], plain[:K * F * S])  # uncond rows: a plain launch
    for g, m in enumerate(SELF_MODES):
        rows = group_rows(K, F, g)
        one = torch.full((2 * F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        kw = dict(row_mode=mode[m], base=base, cache_ld=T, mask=masks[g]) if m != "none" else {}
        if m == "replace":
            kw.pop("mask")
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=2 * F, src_index=[[row[r] for r in rows] for row in si], edit_bf_start=F,
                      **kw, **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"group {g} ({m})"
    report[f"grouped_self_d{d}_S{S}_{kind}"] = "bitwise"


def make_xedit(mode, eq_word=None):
    t = torch.zeros(_lib.XEDIT_FLOATS)
    t[0] = mode
    t[8:8 + 77] = (torch.arange(77) % 5 != 0).float()
    t[88:88 + 80] = 1.0
    if eq_word is not None:
        t[88 + eq_word] = 10.0
    t[168:168 + 77] = (torch.arange(77) % 7 != 0).float()
    t[248:248 + 77] = torch.cat([torch.tensor([0, 1, -1, 2, 3]), torch.arange(4, 76)]).float()
    M = torch.eye(80)
    M[2, 2], M[2, 3], M[2, 4], M[5, 5], M[5, 6] = 0, 0.5, 0.5, 0, 1
    t[328:] = M.reshape(-1)
    return t.to(dev)


@pytest.mark.parametrize("S,d", [(256, 40), (1024, 80), (256, 160)])
def test_grouped_cross_bitwise(S, d, report):
    """CROSSEDIT groups with refine, replace and reweight tables (+ a NONE group), each with its own running-sum slab."""
    tabs = [make_xedit(0), make_xedit(1), make_xedit(1, eq_word=3), None]
    K, F, heads = len(tabs), 2, 2
    BF, Cc = 2 * K * F, heads * d
    si = [[b for b in range(2 * K) for _ in range(F)]]
    q = rnd(BF * S, Cc, seed=5, scale=2.0).half()
    k, v = rnd(2 * K * 77, Cc, seed=6).half(), rnd(2 * K * 77, Cc, seed=7).half()
    vt = torch.zeros(2 * K, heads, d, 80, dtype=torch.float16, device=dev)
    vt[..., :77] = v.view(2 * K, 77, heads, d).permute(0, 2, 3, 1)
    base = torch.zeros(F, heads, S, 80, dtype=torch.float16, device=dev)
    base[..., :77] = torch.softmax(rnd(F, heads, S, 77, seed=8) * 2, -1).half()
    accs = [torch.full((F, heads, S, 80), 0.125 * g, dtype=torch.float16, device=dev) for g in range(K)]
    acc_ref = [a.clone() for a in accs]
    groups = [dict(row_mode=_lib.ATTN_CROSSEDIT if t is not None else _lib.ATTN_NONE, xedit=t, acc=accs[g] if t is not None else None)
              for g, t in enumerate(tabs)]
    geo = dict(S_q=S, keys_per_slot=77, n_src=2 * K, d=d, heads=heads, scale=d ** -0.5)
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, edit_bf_start=K * F, base=base, cache_ld=80, groups=groups, **geo)
    for g, t in enumerate(tabs):
        rows = group_rows(K, F, g)
        one = torch.full((2 * F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        kw = dict(row_mode=_lib.ATTN_CROSSEDIT, base=base, cache_ld=80, acc=acc_ref[g], xedit=t) if t is not None else {}
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=2 * F, src_index=[[si[0][r] for r in rows]], edit_bf_start=F, **kw, **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"group {g}"
        assert torch.equal(accs[g], acc_ref[g]), f"group {g} running sum"
    report[f"grouped_cross_S{S}_d{d}"] = "bitwise"


def test_grouped_mixed_fp64(report):
    """[REPLACE, NONE, BLEND] groups in one launch against the fp64 attention bound of tests/_ref64.py."""
    K, F, S, heads, d = 3, 2, 256, 2, 80
    BF = 2 * K * F
    si = src_rows("mid", F, 2 * K)
    q, k, v = rnd(BF * S, heads * d, seed=11, scale=2.0).half(), rnd(BF * S, heads * d, seed=12).half(), rnd(BF * S, heads * d, seed=13).half()
    vt = v.view(BF, S, heads, d).permute(0, 2, 3, 1).contiguous()
    base = torch.softmax(rnd(F, heads, S, S, seed=14) * 3, -1).half()
    mask = (rnd(F, S, seed=15) > 0).float()
    groups = [dict(row_mode=_lib.ATTN_REPLACE), dict(row_mode=_lib.ATTN_NONE), dict(row_mode=_lib.ATTN_BLEND, mask=mask)]
    out = torch.full((BF * S, heads * d), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F, BF=BF, scale=d ** -0.5, src_index=si,
                  edit_bf_start=K * F, base=base, cache_ld=S, groups=groups)
    idx = torch.tensor(si[0], device=dev)
    qh = q.double().view(BF, S, heads, d).permute(0, 2, 1, 3)
    kh = k.double().view(BF, S, heads, d)[idx].permute(0, 2, 1, 3)
    vh = v.double().view(BF, S, heads, d)[idx].permute(0, 2, 1, 3)
    p = softmax64(qh @ kh.transpose(-1, -2) * torch.tensor(d ** -0.5, dtype=torch.float32).item())
    r0, r2 = K * F, (K + 2) * F
    p[r0:r0 + F] = base.double()
    m = mask.double()[:, None, :, None]
    p[r2:r2 + F] = m * p[r2:r2 + F] + (1 - m) * base.double()
    check_attn(out.view(BF, S, heads, d).permute(0, 2, 1, 3), p, vh, report, "grouped_mixed_fp64")


def test_grouped_refusals():
    F, S, heads, d = 2, 64, 1, 40
    def call(BF, start, groups, n_src=None):
        q = torch.zeros(BF * S, heads * d, dtype=torch.float16, device=dev)
        vt = torch.zeros(BF, heads, d, S, dtype=torch.float16, device=dev)
        base = torch.zeros(F, heads, S, S, dtype=torch.float16, device=dev)
        ops.attention(q, q, vt, torch.empty_like(q), S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=F, BF=BF, scale=1.0,
                      src_index=[list(range(BF))], edit_bf_start=start, base=base, cache_ld=S, groups=groups)
    rep = dict(row_mode=_lib.ATTN_REPLACE)
    with pytest.raises(RuntimeError, match="n_groups"):
        call(8, 4, [rep] * 3)                       # 4 rows after edit_bf_start, 3 groups of F = 2
    with pytest.raises(RuntimeError, match="STORE"):
        call(8, 4, [rep, dict(row_mode=_lib.ATTN_STORE)])
    with pytest.raises(RuntimeError, match="BF=130"):
        call(130, 114, [rep] * 8)                   # over the grouped limit of 128 rows
    with pytest.raises(ValueError, match="groups"):
        call(36, 18, [rep] * 9)
    with pytest.raises(RuntimeError, match="BLEND needs a mask"):
        call(8, 4, [rep, dict(row_mode=_lib.ATTN_BLEND)])


# --------------------------------------------------------------------------------------------------------- GroupNorm / CFG
@pytest.mark.parametrize("HW,C,fps", [(4096, 320, 8), (1024, 640, 1), (64, 1280, 8), (256, 1280, 1)])
def test_groupnorm_batched_bitwise(HW, C, fps):
    K, per = 4, 16  # 4 prompts x CFG 2 x 8 frames
    x = rnd(K * per, HW, C, seed=21).half()
    gamma, beta = rnd(C, seed=22), rnd(C, seed=23)
    got = ops.groupnorm(x, gamma, beta, 1e-5, 32, fps, True, images_per_item=per)
    for k in range(K):
        one = ops.groupnorm(x[k * per:(k + 1) * per].contiguous(), gamma, beta, 1e-5, 32, fps, True)
        assert torch.equal(got[k * per:(k + 1) * per], one), f"item {k}"
    with pytest.raises(RuntimeError, match="images_per_item"):
        ops.groupnorm(x, gamma, beta, 1e-5, 32, 8, True, images_per_item=12)


def test_cfg_ddim_batched_bitwise():
    K, F, h = 4, 8, 64
    x = rnd(K, 4, F, h, h, seed=31)
    eps2 = rnd(2 * K, 4, F, h, h, seed=32)
    x_inv = rnd(1, 4, F, h, h, seed=33)
    mk = lambda s: (rnd(F, h, h, seed=s) > 0).float()  # noqa: E731
    blends = [dict(x_inv=x_inv, mask_a=mk(40), mask_b=mk(41), apply_blend=True), None,
              dict(x_inv=x_inv, mask_a=mk(42), mask_b=mk(43), apply_blend=False), dict(x_inv=x_inv, mask_a=mk(44), mask_b=mk(45), apply_blend=True)]
    got = x.clone()
    ops.cfg_ddim_step_batched(got, eps2, 7.5, 0.3, 0.5, x_inv=x_inv, blends=blends)
    for k, b in enumerate(blends):
        one = x[k:k + 1].clone()
        e = torch.cat([eps2[k:k + 1], eps2[K + k:K + k + 1]]).contiguous()
        if b is None:
            ops.cfg_ddim_step(one, e, 7.5, 0.3, 0.5)
        else:
            ops.cfg_ddim_step(one, e, 7.5, 0.3, 0.5, x_inv=x_inv, mask_a=b["mask_a"], mask_b=b["mask_b"], apply_blend=b["apply_blend"])
        assert torch.equal(got[k:k + 1], one), f"item {k}"


# ------------------------------------------------------------------------------------------------------------ tap-GEMM
@pytest.mark.parametrize("M,N,K", [(154, 640, 768), (616, 1280, 768), (4096, 320, 320), (512, 2560, 1280)])
def test_tapgemm_independent_of_block_n(M, N, K, report):
    """Every output element is one tile's fp32 wgmma accumulation over K in the same k order whatever BLOCK_N: the result must not
    depend on it (so the automatic choice, which depends on the number of row tiles, cannot make a batch differ from a single prompt)."""
    a, w = rnd(M, K, seed=51).half(), (rnd(N, K, seed=52) * 0.05).half()
    bias, res = rnd(N, seed=53), rnd(M, N, seed=54).half()
    outs = {bn: ops.gemm(a, w, bias=bias, residual=res, force_bn=bn) for bn in (16, 32, 64, 128, 160, 256)}
    ref = ops.gemm(a, w, bias=bias, residual=res)
    for bn, o in outs.items():
        assert torch.equal(o, ref), f"BLOCK_N={bn}"
    x = rnd(4, 16, 16, 320, seed=55).half()
    w9 = (rnd(9, 640, 320, seed=56) * 0.02).half()
    cref = ops.conv3x3(x, w9)
    for bn in (32, 64, 128, 160, 256):
        assert torch.equal(ops.conv3x3(x, w9, force_bn=bn), cref), f"conv BLOCK_N={bn}"
    report[f"tapgemm_bn_{M}_{N}_{K}"] = "bitwise"


# ------------------------------------------------------------------------------------------------------------ pipeline
MC = CASES["mini_replace_blend"]["model_config"]
PROMPTS = [
    (SRC, dict(is_replace_controller=True, cross_replace_steps={"default_": 0.8}, self_replace_steps=0.8)),  # reconstruction (prompt 0)
    (CASES["mini_refine"]["target"], CASES["mini_refine"]["p2p"]),
    (CASES["mini_replace_blend"]["target"], CASES["mini_replace_blend"]["p2p"]),
    (CASES["mini_reweight_next"]["target"], CASES["mini_reweight_next"]["p2p"]),
]


def _invert(pipe, x0, N, twice=False):
    pipe.scheduler.set_timesteps(N)
    emb = pipe._encode_prompt(SRC, dev, 1, True, None)
    pipe.prepare_before_train_loop()
    for _ in range(2 if twice else 1):  # the second pass replays a captured inversion: its store can back a captured edit
        pipe.store_controller = controllers.AttentionStore()
        controllers.register_attention_control(pipe, pipe.store_controller)
        pipe.store_controller.LOW_RESOURCE = True
        inv = pipe.ddim_clean2noisy_loop(x0, emb, pipe.store_controller)
        pipe.store_controller.LOW_RESOURCE = False
    return inv[-1]


def _single(pipe, xT, prompt, p2p, N, save_path):
    trace = []
    res = pipe(prompt=prompt, source_prompt=SRC, edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5,
               output_type="latent", callback=lambda i, t, l: trace.append(l.detach().clone()), use_inversion_attention=True,
               save_self_attention=False, save_path=save_path, **p2p)
    return dict(trace=trace, final=res["sdimage_output"].images, masks=res["mask_list"], sums=pipe.last_edit_controller.attention_store)


def _batch(pipe, xT, prompts, N, save_path):
    trace = []
    res = pipe.p2preplace_edit_batch([p for p, _ in prompts], [dict(c, use_inversion_attention=True, save_self_attention=False) for _, c in prompts],
                                     SRC, xT, N, 7.5, save_path=save_path, output_type="latent",
                                     callback=lambda i, t, l: trace.append(l.detach().clone()))
    return trace, res


def _assert_same(single, trace, res, k, ctrl, tag):
    for i, (a, b) in enumerate(zip(single["trace"], trace)):
        assert torch.equal(a[0], b[k]), f"{tag}: prompt {k} step {i}"
    assert torch.equal(single["final"][0], res[k]["sdimage_output"].images[0]), f"{tag}: prompt {k} final latents"
    if single["masks"] is None:
        assert res[k]["mask_list"] is None
    else:
        assert len(single["masks"]) == len(res[k]["mask_list"]) > 0
        for a, b in zip(single["masks"], res[k]["mask_list"]):
            assert torch.equal(a, b), f"{tag}: prompt {k} mask"
    sums = ctrl.attention_store
    assert set(sums) == set(single["sums"])
    for key in sums:
        for a, b in zip(single["sums"][key], sums[key]):
            assert torch.equal(a, b), f"{tag}: prompt {k} {key} running sum"


@pytest.mark.parametrize("graph_mode", ["off", "auto"])
def test_pipeline_batch_equals_single_prompt_runs(graph_mode, report):
    case = CASES["mini_replace_blend"]
    N = case["steps"]
    pipe = build_product(case["unet"], MC)
    x0 = case_inputs(case).to(dev)
    xT = _invert(pipe, x0, N, twice=graph_mode == "auto")
    save = tempfile.mkdtemp()
    pipe.graph_mode = "off"
    singles = [_single(pipe, xT, p, c, N, save) for p, c in PROMPTS]
    pipe.graph_mode = graph_mode
    trace, res = _batch(pipe, xT, PROMPTS, N, save)
    if graph_mode == "auto":  # the first batched call ran eagerly: the second one captures and replays
        assert not any(isinstance(k[0], tuple) for k in pipe._plans)  # inversion plans only
        trace, res = _batch(pipe, xT, PROMPTS, N, save)
        assert any(k[0][0] == "edit" and k[0][5][0] == "edit_batch" for k in pipe._plans if isinstance(k[0], tuple))
    assert len(trace) == N and trace[0].shape[0] == len(PROMPTS)
    for k, ctrl in enumerate(pipe.last_edit_controllers):
        _assert_same(singles[k], trace, res, k, ctrl, graph_mode)
    report[f"pipeline_batch_{graph_mode}"] = dict(prompts=len(PROMPTS), steps=N, bitwise=True)


def test_pipeline_batch_of_one_equals_existing_path():
    case = CASES["mini_refine"]
    N = case["steps"]
    pipe = build_product(case["unet"], case["model_config"])
    pipe.graph_mode = "off"
    xT = _invert(pipe, case_inputs(case).to(dev), N)
    single = _single(pipe, xT, case["target"], case["p2p"], N, None)
    trace, res = _batch(pipe, xT, [(case["target"], case["p2p"])], N, None)
    _assert_same(single, trace, res, 0, pipe.last_edit_controllers[0], "K=1")


def test_sd14_batched_group0_matches_golden_and_single():
    import os
    from test_gpu_golden_sd14 import BOUNDS
    name = "sd14_replace_blend"
    path = os.path.join(GOLDEN_DIR, f"{name}.pt")
    if not os.path.exists(path):
        pytest.skip(f"{path} missing")
    g = torch.load(path)
    case = CASES[name]
    pipe = build_product(case["unet"], case["model_config"])
    pipe.graph_mode = "off"
    single = run_product_case(case, pipe=pipe)
    xT = single["inv_latents"][-1:].to(dev)[0]
    refine = ("watercolor painting of " + SRC, CASES["sd14_config1"]["p2p"])
    trace, res = _batch(pipe, xT, [(case["target"], case["p2p"]), refine], case["steps"], tempfile.mkdtemp())
    got = res[0]["sdimage_output"].images[0].float().cpu()
    assert torch.equal(got, single["edit_latents"][-1][0])
    d = (got - g["edit_latents"][-1].reshape(got.shape).float()).abs().flatten()
    assert torch.quantile(d[::7], 0.99).item() < BOUNDS[name]["free_edit"]
