"""Runners for the non-square parity tests (oracle/nonsquare.py's cases): the CPU oracle and the CUDA product on h x w latents.
_helpers.run_oracle_case / run_product_case build square clips; these take the clip from the case's (h, w)."""
import os
import tempfile

import torch

import _sd2_golden
from _helpers import GOLDEN_DIR, build_oracle, build_product  # noqa: F401  (build_product: used by the GPU tests)
from fatezero_b200 import synth
from oracle import nonsquare as ns


def load(name: str) -> dict:
    """The golden with the samples of every step (oracle/sd2.py's compact format, teacher latents kept in full)."""
    assert os.path.exists(os.path.join(GOLDEN_DIR, f"{name}.pt")), f"missing golden fixture {name} (python -m oracle.make_nonsquare_golden)"
    return _sd2_golden.load(name)


def run_oracle(case: dict, ou=None):
    """Inversion + edit with the CPU oracle (oracle.nonsquare.OracleEditNS). Returns dict(inv_latents, edit_latents, store, ctrl)."""
    from oracle import fz_oracle as fo
    cfg = synth.UNET_CONFIGS[case["unet"]]
    ou = ou or build_oracle(case["unet"], case["model_config"])
    tok, te = synth.ToyTokenizer(), synth.ToyTextEncoder(cfg["cross_attention_dim"])
    emb_src = fo.encode_prompts(tok, te, case["source"])
    emb_tgt = fo.encode_prompts(tok, te, case["target"])
    N = case["steps"]
    store = fo.OracleStore()
    inv = fo.invert(ou, ns.case_inputs(case), emb_src[1:], N, store)
    p = case["p2p"]
    plan = fo.EditPlan(tok, case["source"], case["target"], N, p["cross_replace_steps"], p["self_replace_steps"],
                       p.get("is_replace_controller", True), p.get("eq_params"), p.get("blend_words"),
                       bool(p.get("blend_self_attention")), bool(p.get("blend_latents")), p.get("blend_th", (0.3, 0.3)))
    ctrl = ns.OracleEditNS(plan, store, (case["h"], case["w"]))
    tr = fo.edit(ou, inv[-1], emb_tgt, N, ctrl)
    return dict(inv_latents=torch.stack(inv), edit_latents=torch.stack(tr), store=store, ctrl=ctrl)


def run_product(case: dict, pipe=None, device="cuda", teacher=None, output_type="latent", shard=None):
    """Inversion + edit through the reference-facing API of the CUDA product on the case's h x w clip.  teacher: dict(inv_latents,
    edit_latents) of reference latents every forward starts from (teacher forcing).  shard = (rank, world): this process holds a
    contiguous block of the clip's frames (pipe.unet.set_frame_shard done by the caller)."""
    from fatezero_b200 import controllers
    pipe = pipe or build_product(case["unet"], case["model_config"], device)
    N = case["steps"]
    pipe.scheduler.set_timesteps(N)
    x0 = ns.case_inputs(case).to(device)
    if shard is not None:
        from fatezero_b200 import dist as fzdist
        x0 = fzdist.frame_slice(x0, shard[0], shard[1])
    emb = pipe._encode_prompt(case["source"], device, 1, True, None)
    pipe.prepare_before_train_loop()
    pipe.store_controller = controllers.AttentionStore()
    controllers.register_attention_control(pipe, pipe.store_controller)
    pipe.store_controller.LOW_RESOURCE = True
    inv = pipe.ddim_clean2noisy_loop(x0, emb, pipe.store_controller,
                                     teacher_latents=None if teacher is None else list(teacher["inv_latents"]))
    pipe.store_controller.LOW_RESOURCE = False
    trace = []
    p = dict(case["p2p"])
    if teacher is not None:
        p["teacher_latents"] = list(teacher["edit_latents"])
    res = pipe(prompt=case["target"], source_prompt=case["source"], edit_type="swap", image=None, strength=None, generator=None,
               num_inference_steps=N, clip_length=x0.shape[2], guidance_scale=7.5, num_images_per_prompt=1,
               latents=inv[-1] if teacher is None else teacher["inv_latents"][-1].to(device), uncond_embeddings_list=None,
               save_path=tempfile.mkdtemp() if p.get("blend_words") else None, height=8 * case["h"], width=8 * case["w"],
               output_type=output_type, callback=lambda i, t, l: trace.append(l.detach().float().cpu().clone()),
               use_inversion_attention=True, save_self_attention=False, **p)
    return dict(inv_latents=torch.stack([l.float().cpu() for l in inv]), edit_latents=torch.stack(trace), pipe=pipe, result=res)
