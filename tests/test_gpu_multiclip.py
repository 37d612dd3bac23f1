"""Batch invariance of the multi-clip inversion and edit: every clip of a batch gets, bit for bit, what its own single-clip run computes.
Kernel level: grouped STORE and per-group cached maps (fz_attention_grouped_slabs_f16) against one fz_attention_f16 launch per group, and
fz_cfg_ddim_step_multi against per-item fz_cfg_ddim_step.  Pipeline level: prepare_latents_ddim_inverted_batch against
prepare_latents_ddim_inverted per clip, p2preplace_edit_clips against p2preplace_edit against each clip's own store, eager and replayed
from CUDA graphs."""
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

from _helpers import build_product, case_inputs  # noqa: E402
from oracle.cases import CASES, SRC  # noqa: E402
from test_gpu_edit_batch import make_xedit, rnd, rows_of, src_rows  # noqa: E402

if torch.cuda.is_available():
    from fatezero_b200 import _lib, controllers, ops

dev = "cuda"


def clip_rows(F, k, start=0):
    return list(range(start + k * F, start + (k + 1) * F))


# --------------------------------------------------------------------------------------------------- grouped STORE (inversion)
@pytest.mark.parametrize("kind", ["mid", "prev_first"])
@pytest.mark.parametrize("S", [256, 1024])
@pytest.mark.parametrize("d", [40, 80, 160])
def test_grouped_store_self_bitwise(d, S, kind, report):
    K, F, heads = 3, 2, 2
    BF, Cc = K * F, heads * d
    si = src_rows(kind, F, K)
    T = len(si) * S
    q, k, v = rnd(BF * S, Cc, seed=61, scale=2.0).half(), rnd(BF * S, Cc, seed=62).half(), rnd(BF * S, Cc, seed=63).half()
    vt = v.view(BF, S, heads, d).permute(0, 2, 3, 1).contiguous()
    slabs = [torch.full((F, heads, S, T), float("nan"), dtype=torch.float16, device=dev) for _ in range(K)]
    geo = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, scale=d ** -0.5)
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, cache_ld=T, groups=[dict(row_mode=_lib.ATTN_STORE, store=s) for s in slabs], **geo)
    for c in range(K):
        rows = clip_rows(F, c)
        one = torch.full((F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        ref = torch.full_like(slabs[c], float("nan"))
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=F, src_index=[[row[r] for r in rows] for row in si], row_mode=_lib.ATTN_STORE,
                      store=ref, cache_ld=T, **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"clip {c} output"
        assert torch.equal(slabs[c], ref), f"clip {c} stored maps"
    report[f"grouped_store_self_d{d}_S{S}_{kind}"] = "bitwise"


@pytest.mark.parametrize("S,d", [(256, 40), (1024, 80), (256, 160)])
def test_grouped_store_cross_bitwise(S, d, report):
    K, F, heads = 3, 2, 2
    BF, Cc = K * F, heads * d
    si = [[b for b in range(K) for _ in range(F)]]
    q = rnd(BF * S, Cc, seed=71, scale=2.0).half()
    k, v = rnd(K * 77, Cc, seed=72).half(), rnd(K * 77, Cc, seed=73).half()
    vt = torch.zeros(K, heads, d, 80, dtype=torch.float16, device=dev)
    vt[..., :77] = v.view(K, 77, heads, d).permute(0, 2, 3, 1)
    slabs = [torch.full((F, heads, S, 80), float("nan"), dtype=torch.float16, device=dev) for _ in range(K)]
    accs = [torch.full((F, heads, S, 80), 0.25 * c, dtype=torch.float16, device=dev) for c in range(K)]
    acc_ref = [a.clone() for a in accs]
    geo = dict(S_q=S, keys_per_slot=77, n_src=K, d=d, heads=heads, scale=d ** -0.5)
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, cache_ld=80,
                  groups=[dict(row_mode=_lib.ATTN_STORE, store=s, acc=a) for s, a in zip(slabs, accs)], **geo)
    for c in range(K):
        rows = clip_rows(F, c)
        one = torch.full((F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        ref = torch.full_like(slabs[c], float("nan"))
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=F, src_index=[[si[0][r] for r in rows]], row_mode=_lib.ATTN_STORE, store=ref,
                      cache_ld=80, acc=acc_ref[c], **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"clip {c} output"
        assert torch.equal(slabs[c][..., :77], ref[..., :77]), f"clip {c} stored maps"
        assert torch.equal(accs[c], acc_ref[c]), f"clip {c} running sum"
    report[f"grouped_store_cross_S{S}_d{d}"] = "bitwise"


# --------------------------------------------------------------------------------------------------- per-group cached maps (edit)
@pytest.mark.parametrize("kind", ["mid", "prev_first"])
@pytest.mark.parametrize("S,d", [(256, 40), (1024, 80), (256, 160)])
def test_per_group_base_self_bitwise(S, d, kind, report):
    """REPLACE / BLEND / NONE / REPLACE groups, three of them reading their own clip's map, the last sharing group 0's."""
    modes = [_lib.ATTN_REPLACE, _lib.ATTN_BLEND, _lib.ATTN_NONE, _lib.ATTN_REPLACE]
    K, F, heads = len(modes), 2, 2
    BF, Cc = 2 * K * F, heads * d
    si = src_rows(kind, F, 2 * K)
    T = len(si) * S
    q, k, v = rnd(BF * S, Cc, seed=81, scale=2.0).half(), rnd(BF * S, Cc, seed=82).half(), rnd(BF * S, Cc, seed=83).half()
    vt = v.view(BF, S, heads, d).permute(0, 2, 3, 1).contiguous()
    bases = [torch.softmax(rnd(F, heads, S, T, seed=84 + g) * 3, -1).half() for g in range(3)]
    bases.append(bases[0])
    mask = (rnd(F, S, seed=90) > 0).float()
    groups = [dict(row_mode=m, base=b, mask=mask if m == _lib.ATTN_BLEND else None) for m, b in zip(modes, bases)]
    geo = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, scale=d ** -0.5)
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, edit_bf_start=K * F, cache_ld=T, groups=groups, **geo)
    for g, m in enumerate(modes):
        rows = clip_rows(F, g) + clip_rows(F, g, K * F)
        one = torch.full((2 * F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        kw = {} if m == _lib.ATTN_NONE else dict(row_mode=m, base=bases[g], cache_ld=T)
        if m == _lib.ATTN_BLEND:
            kw["mask"] = mask
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=2 * F, src_index=[[row[r] for r in rows] for row in si], edit_bf_start=F,
                      **kw, **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"group {g}"
    report[f"per_group_base_self_S{S}_d{d}_{kind}"] = "bitwise"


@pytest.mark.parametrize("S,d", [(256, 40), (1024, 80), (256, 160)])
def test_per_group_base_cross_bitwise(S, d, report):
    tabs = [make_xedit(0), make_xedit(1), make_xedit(1, eq_word=3)]
    K, F, heads = len(tabs), 2, 2
    BF, Cc = 2 * K * F, heads * d
    si = [[b for b in range(2 * K) for _ in range(F)]]
    q = rnd(BF * S, Cc, seed=91, scale=2.0).half()
    k, v = rnd(2 * K * 77, Cc, seed=92).half(), rnd(2 * K * 77, Cc, seed=93).half()
    vt = torch.zeros(2 * K, heads, d, 80, dtype=torch.float16, device=dev)
    vt[..., :77] = v.view(2 * K, 77, heads, d).permute(0, 2, 3, 1)
    bases = []
    for g in range(K):
        b = torch.zeros(F, heads, S, 80, dtype=torch.float16, device=dev)
        b[..., :77] = torch.softmax(rnd(F, heads, S, 77, seed=94 + g) * 2, -1).half()
        bases.append(b)
    accs = [torch.full((F, heads, S, 80), 0.125 * g, dtype=torch.float16, device=dev) for g in range(K)]
    acc_ref = [a.clone() for a in accs]
    groups = [dict(row_mode=_lib.ATTN_CROSSEDIT, xedit=t, acc=a, base=b) for t, a, b in zip(tabs, accs, bases)]
    geo = dict(S_q=S, keys_per_slot=77, n_src=2 * K, d=d, heads=heads, scale=d ** -0.5)
    out = torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev)
    ops.attention(q, k, vt, out, F=F, BF=BF, src_index=si, edit_bf_start=K * F, cache_ld=80, groups=groups, **geo)
    for g, t in enumerate(tabs):
        rows = clip_rows(F, g) + clip_rows(F, g, K * F)
        one = torch.full((2 * F * S, Cc), float("nan"), dtype=torch.float16, device=dev)
        ops.attention(rows_of(q, rows, S), k, vt, one, F=F, BF=2 * F, src_index=[[si[0][r] for r in rows]], edit_bf_start=F,
                      row_mode=_lib.ATTN_CROSSEDIT, base=bases[g], cache_ld=80, acc=acc_ref[g], xedit=t, **geo)
        assert torch.equal(rows_of(out, rows, S), one), f"group {g}"
        assert torch.equal(accs[g], acc_ref[g]), f"group {g} running sum"
    report[f"per_group_base_cross_S{S}_d{d}"] = "bitwise"


def test_null_slabs_mean_the_launch_slab():
    """A NULL per-group pointer means the slab of the launch arguments: NULL slabs give bitwise what per-group pointers to that same slab
    give.  (That the grouped launch without slabs still computes what it computed before is guarded by the unchanged
    tests/test_gpu_edit_batch.py.)"""
    K, F, S, heads, d = 3, 2, 256, 2, 80
    BF, Cc = 2 * K * F, heads * d
    si = src_rows("prev_first", F, 2 * K)
    T = len(si) * S
    q, k, v = rnd(BF * S, Cc, seed=101, scale=2.0).half(), rnd(BF * S, Cc, seed=102).half(), rnd(BF * S, Cc, seed=103).half()
    vt = v.view(BF, S, heads, d).permute(0, 2, 3, 1).contiguous()
    base = torch.softmax(rnd(F, heads, S, T, seed=104) * 3, -1).half()
    mask = (rnd(F, S, seed=105) > 0).float()
    modes = [dict(row_mode=_lib.ATTN_REPLACE), dict(row_mode=_lib.ATTN_NONE), dict(row_mode=_lib.ATTN_BLEND, mask=mask)]
    kw = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, scale=d ** -0.5, F=F, BF=BF, src_index=si, edit_bf_start=K * F, cache_ld=T)
    null = ops.attention(q, k, vt, torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev), base=base, groups=modes, **kw)
    explicit = ops.attention(q, k, vt, torch.full((BF * S, Cc), float("nan"), dtype=torch.float16, device=dev),
                             groups=[dict(g, base=base) for g in modes], **kw)
    assert torch.equal(null, explicit)
    # STORE: NULL store pointers write the launch's slab (one group here, so the slab is the group's)
    slab_a = torch.full((F, heads, S, T), float("nan"), dtype=torch.float16, device=dev)
    slab_b = torch.full_like(slab_a, float("nan"))
    kw1 = dict(kw, BF=F, edit_bf_start=0, src_index=[row[:F] for row in si])
    o1 = ops.attention(q, k, vt, torch.empty((F * S, Cc), dtype=torch.float16, device=dev), store=slab_a,
                       groups=[dict(row_mode=_lib.ATTN_STORE)], **kw1)
    o2 = ops.attention(q, k, vt, torch.empty((F * S, Cc), dtype=torch.float16, device=dev), groups=[dict(row_mode=_lib.ATTN_STORE, store=slab_b)],
                       **kw1)
    assert torch.equal(o1, o2) and torch.equal(slab_a, slab_b)


# ------------------------------------------------------------------------------------------------------------------ CFG step
@pytest.mark.parametrize("shared", [False, True])
def test_cfg_ddim_multi_bitwise(shared):
    K, F, h = 4, 4, 32
    x = rnd(K, 4, F, h, h, seed=111)
    eps2 = rnd(2 * K, 4, F, h, h, seed=112)
    invs = [rnd(1, 4, F, h, h, seed=113 + k) for k in range(K)]
    if shared:  # items of one clip: the same device pointer
        invs = [invs[0]] * K
    mk = lambda s: (rnd(F, h, h, seed=s) > 0).float()  # noqa: E731
    blends = [dict(x_inv=invs[0], mask_a=mk(120), mask_b=mk(121), apply_blend=True), None,
              dict(x_inv=invs[2], mask_a=mk(122), mask_b=None, apply_blend=True), dict(x_inv=invs[3], mask_a=mk(124), mask_b=mk(125), apply_blend=False)]
    got = x.clone()
    ops.cfg_ddim_step_multi(got, eps2, 7.5, 0.3, 0.5, blends=blends)
    for k, b in enumerate(blends):
        one = x[k:k + 1].clone()
        e = torch.cat([eps2[k:k + 1], eps2[K + k:K + k + 1]]).contiguous()
        if b is None:
            ops.cfg_ddim_step(one, e, 7.5, 0.3, 0.5)
        else:
            ops.cfg_ddim_step(one, e, 7.5, 0.3, 0.5, x_inv=b["x_inv"], mask_a=b["mask_a"], mask_b=b["mask_b"], apply_blend=b["apply_blend"])
        assert torch.equal(got[k:k + 1], one), f"item {k}"
    plain = x.clone()
    ops.cfg_ddim_step_multi(plain, eps2, 7.5, 0.3, 0.5)
    ref = x.clone()
    ops.cfg_ddim_step_batched(ref, eps2, 7.5, 0.3, 0.5)
    assert torch.equal(plain, ref)


# ------------------------------------------------------------------------------------------------------------------ pipeline
CASE = CASES["mini_replace_blend"]
N = CASE["steps"]
SOURCES = [SRC, "a red car driving down a curvy road in the countryside", "a silver jeep driving down a snowy road in the countryside"]


def clip_latents(k):
    """distinct content per clip: the case's latents mirrored / shifted / rescaled"""
    x0 = case_inputs(CASE).to(dev)
    return [x0, -x0.flip(-1), 0.8 * x0.roll(3, -2)][k]


def single_inversion(pipe, x0, source):
    pipe.scheduler.set_timesteps(N)
    emb = pipe._encode_prompt(source, dev, 1, True, None)
    pipe.prepare_before_train_loop()
    store = controllers.AttentionStore()
    pipe.store_controller = store
    controllers.register_attention_control(pipe, store)
    store.LOW_RESOURCE = True
    inv = pipe.ddim_clean2noisy_loop(x0, emb, store)
    store.LOW_RESOURCE = False
    controllers.register_attention_control(pipe, pipe.empty_controller)
    return inv, store


def batch_inversion(pipe, clips, sources):
    pipe.scheduler.set_timesteps(N)
    return pipe.prepare_latents_ddim_inverted_batch(sources, latents=clips), pipe.store_controllers


def assert_store_equal(a, b, tag):
    assert a.cur_step == b.cur_step == N, tag
    assert len(a.latents_store) == len(b.latents_store) == N
    for i, (x, y) in enumerate(zip(a.latents_store, b.latents_store)):
        assert torch.equal(x, y), f"{tag}: latents_store[{i}]"
    assert len(a.attention_store_all_step) == len(b.attention_store_all_step) == N
    for i, (sa, sb) in enumerate(zip(a.attention_store_all_step, b.attention_store_all_step)):
        assert set(sa) == set(sb)
        for key in sa:
            assert len(sa[key]) == len(sb[key]), f"{tag}: step {i} {key}"
            for j, (x, y) in enumerate(zip(sa[key], sb[key])):
                assert torch.equal(x, y), f"{tag}: step {i} {key}[{j}]"
    sa, sb = a.attention_store, b.attention_store
    assert set(sa) == set(sb)
    for key in sa:
        assert len(sa[key]) == len(sb[key]) > 0
        for x, y in zip(sa[key], sb[key]):
            assert torch.equal(x, y), f"{tag}: attention_store {key}"


@pytest.fixture(scope="module")
def pipe_and_singles():
    pipe = build_product(CASE["unet"], CASE["model_config"])
    pipe.graph_mode = "off"
    singles = [single_inversion(pipe, clip_latents(k), SOURCES[k]) for k in range(3)]
    return pipe, singles


@pytest.mark.parametrize("K", [1, 2, 3])
def test_batched_inversion_equals_single_clip_runs(pipe_and_singles, K, report):
    pipe, singles = pipe_and_singles
    pipe.graph_mode = "off"
    lats, stores = batch_inversion(pipe, [clip_latents(k) for k in range(K)], SOURCES[:K])
    assert len(lats) == len(stores) == K
    for k in range(K):
        inv, store = singles[k]
        assert len(lats[k]) == N + 1
        for i, (x, y) in enumerate(zip(inv, lats[k])):
            assert torch.equal(x, y), f"clip {k} latent {i}"
        assert_store_equal(store, stores[k], f"K={K} clip {k}")
    report[f"batched_inversion_K{K}"] = "bitwise"


JOBS = [  # (clip, target prompt, p2p config)
    (0, CASES["mini_refine"]["target"], CASES["mini_refine"]["p2p"]),                 # Refine + Reweight
    (1, CASE["target"], CASE["p2p"]),                                                   # Replace + self-attention blend + latent blend
    (0, CASES["mini_reweight_next"]["target"], CASES["mini_reweight_next"]["p2p"]),   # a second prompt on clip 0: Replace + Reweight
]


def edit_single(pipe, store, xT, prompt, p2p, save):
    pipe.store_controller = store
    res = pipe(prompt=prompt, source_prompt=SRC, edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5, output_type="latent",
               use_inversion_attention=True, save_self_attention=False, save_path=save, **p2p)
    return dict(final=res["sdimage_output"].images, masks=res["mask_list"], sums=pipe.last_edit_controller.attention_store)


def edit_clips(pipe, stores, xTs, jobs, save):
    js = [dict(p2p, store=stores[c], latents=xTs[c], prompt=p, source_prompt=SRC, use_inversion_attention=True, save_self_attention=False)
          for c, p, p2p in jobs]
    return pipe.p2preplace_edit_clips(js, N, 7.5, output_type="latent", save_path=save)


def assert_job_equal(single, res, ctrl, tag):
    assert torch.equal(single["final"], res["sdimage_output"].images), f"{tag}: final latents"
    if single["masks"] is None:
        assert res["mask_list"] is None
    else:
        assert len(single["masks"]) == len(res["mask_list"]) > 0
        for a, b in zip(single["masks"], res["mask_list"]):
            assert torch.equal(a, b), f"{tag}: mask"
    sums = ctrl.attention_store
    assert set(sums) == set(single["sums"]) and sums
    for key in sums:
        for a, b in zip(single["sums"][key], sums[key]):
            assert torch.equal(a, b), f"{tag}: {key} running sum"


def test_batched_clip_edit_equals_single_edits(report):
    pipe = build_product(CASE["unet"], CASE["model_config"])
    pipe.graph_mode = "off"
    save = tempfile.mkdtemp()
    lats, stores = batch_inversion(pipe, [clip_latents(0), clip_latents(1)], [SRC, SRC])
    xTs = [l[-1] for l in lats]
    singles = [edit_single(pipe, stores[c], xTs[c], p, p2p, save) for c, p, p2p in JOBS]
    res = edit_clips(pipe, stores, xTs, JOBS, save)
    for j, (s, r, ctrl) in enumerate(zip(singles, res, pipe.last_edit_controllers)):
        assert_job_equal(s, r, ctrl, f"job {j}")
    assert singles[1]["masks"]  # the latent blend ran
    report["batched_clip_edit"] = dict(jobs=len(JOBS), clips=2, steps=N, bitwise=True)


def test_graph_replay_equals_eager(report):
    """Both batched loops under graph_mode='auto' (eager, capture + replay, replay with new clips / prompts) against eager runs."""
    pipe = build_product(CASE["unet"], CASE["model_config"])
    save = tempfile.mkdtemp()
    sets = [([clip_latents(0), clip_latents(1)], SOURCES[:2]), ([clip_latents(2), clip_latents(0)], [SOURCES[2], SOURCES[0]])]
    pipe.graph_mode = "off"
    eager = [batch_inversion(pipe, c, s) for c, s in sets]
    pipe.graph_mode = "auto"
    for rnd_i, (c, s) in enumerate([sets[0], sets[0], sets[1]]):  # eager, captured + replayed, replayed with other clips
        lats, stores = batch_inversion(pipe, c, s)
        ref_lats, ref_stores = eager[1 if rnd_i == 2 else 0]
        for k in range(2):
            for i, (x, y) in enumerate(zip(ref_lats[k], lats[k])):
                assert torch.equal(x, y), f"inversion round {rnd_i} clip {k} latent {i}"
            assert_store_equal(ref_stores[k], stores[k], f"inversion round {rnd_i} clip {k}")
    assert any(k[0] == "inv" and k[5][0] == "store_batch" for k in pipe._plans)
    assert stores[0]._graph_plan_id[1] == 0 and stores[1]._graph_plan_id[1] == 1
    # second call: new latents and new target prompts with the same edit structure (the captured edit is replayed, not re-captured)
    runs = dict(a=(JOBS, [l[-1] for l in lats]),
                b=([(0, "watercolor painting of a silver jeep driving down a snowy road in the countryside", JOBS[0][2]),
                    (1, "a Porsche car driving down a snowy road in the countryside", JOBS[1][2]),
                    (0, "a silver jeep driving down a snowy road in the mountains", JOBS[2][2])], [0.9 * l[-1] for l in lats]))
    pipe.graph_mode = "off"
    ref = {name: (edit_clips(pipe, stores, xTs, jobs, save), list(pipe.last_edit_controllers)) for name, (jobs, xTs) in runs.items()}
    pipe.graph_mode = "auto"
    n_plans = None
    for rnd_i, name in enumerate(["a", "a", "b"]):
        jobs, xTs = runs[name]
        res = edit_clips(pipe, stores, xTs, jobs, save)
        if rnd_i == 1:
            n_plans = len(pipe._plans)
        ref_res, ref_ctrls = ref[name]
        for j, (r0, r1, c0, c1) in enumerate(zip(ref_res, res, ref_ctrls, pipe.last_edit_controllers)):
            single = dict(final=r0["sdimage_output"].images, masks=r0["mask_list"], sums=c0.attention_store)
            assert_job_equal(single, r1, c1, f"edit round {rnd_i} job {j}")
    assert any(isinstance(k[0], tuple) and k[0][0] == "edit" and k[0][5][0] == "edit_clips" for k in pipe._plans)
    assert len(pipe._plans) == n_plans  # the third call replayed the plan captured by the second
    report["graph_replay_multiclip"] = "bitwise"


def test_single_clip_replay_recomputes_self_sums():
    """A store filled by replaying a captured inversion does not inherit the self-attention sums the capture's store had computed: they
    are rebuilt from the replayed maps (the single-clip path; the batched one is covered above)."""
    pipe = build_product(CASE["unet"], CASE["model_config"])
    pipe.graph_mode = "off"
    _, ref = single_inversion(pipe, clip_latents(1), SOURCES[1])
    pipe.graph_mode = "auto"
    single_inversion(pipe, clip_latents(0), SOURCES[0])                  # eager
    _, captured = single_inversion(pipe, clip_latents(0), SOURCES[0])    # captured + replayed
    assert captured.attention_store["down_self"]                          # computes (and caches) the sums of clip 0
    _, replayed = single_inversion(pipe, clip_latents(1), SOURCES[1])    # replayed with another clip
    assert replayed._graph_plan_id is not None
    assert_store_equal(ref, replayed, "single-clip replay")
