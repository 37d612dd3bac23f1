"""SD-2-base against SD-1.4 geometry on the flagship workload: a style edit (Refine + Reweight, 512x512x8 frames, 50 inversion + 50 edit
DDIM steps, synthetic weights, graph-captured loops) through the reference-facing API, one geometry after the other, alternating.

Per round and geometry the UNet is built on the GPU from a seeded state dict, two clips warm it up (eager, then captured) and --clips clips
are timed, wall clock around a device synchronise; the pipe is then freed, so the two map caches (36 GiB and 49 GiB at 8 frames) never
coexist.  Reported per geometry: frames/s (frames / median clip seconds), the map-cache bytes per frame and DDIM step
(controllers.map_cache_bytes) and the peak HBM allocated while timing.  The card name, power limit and max SM clock are printed first.

    python tools/bench_sd2.py [--rounds 2] [--clips 3] [--frames 8]
Prints one JSON line per (round, geometry) and a summary line.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

GEOMETRIES = ("sd2", "sd14")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:  # noqa: BLE001
        out = "unknown"
    return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out, query=q)


def build_pipe(name, sd, device):
    from fatezero_b200 import DDIMScheduler, P2pDDIMSpatioTemporalPipeline, UNetPseudo3DConditionModel, synth
    cfg = synth.UNET_CONFIGS[name]
    unet = UNetPseudo3DConditionModel(**cfg, **bench.CFG["model_config"])
    unet.load_state_dict(sd)
    unet.to(device)
    te = synth.ToyTextEncoder(cfg["cross_attention_dim"]).to(device)
    pipe = P2pDDIMSpatioTemporalPipeline(synth.VaeStub(), te, synth.ToyTokenizer(), unet, DDIMScheduler())
    pipe.scheduler.set_timesteps(bench.DDIM_STEPS)
    pipe.prepare_before_train_loop()
    return pipe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--clips", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sd2 measures on a CUDA device; none is visible")
    from fatezero_b200 import controllers, synth
    from fatezero_b200.unet import unet_param_spec
    bench.select_config("style")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    F, size = args.frames, bench.CFG["size"]
    mc = bench.CFG["model_config"]
    sds = {}
    for name in GEOMETRIES:
        spec = unet_param_spec(dict(synth.UNET_CONFIGS[name]), mc)
        sds[name] = synth.synth_state_dict({k: v[0] for k, v in spec.items()}, seed=0)
    x0 = (synth.synth_latents(F, size, size) * 0.5).to(dev)
    rows = {n: [] for n in GEOMETRIES}
    for rnd in range(args.rounds):
        for name in GEOMETRIES:
            pipe = build_pipe(name, sds[name], dev)
            emb = pipe._encode_prompt(bench.SRC, dev, 1, True, None)
            for _ in range(2):  # eager, then captured: the timed clips replay graphs
                bench.edit_clip(pipe, x0, emb)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            ts = []
            for _ in range(args.clips):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                bench.edit_clip(pipe, x0, emb)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            per_step, once = controllers.map_cache_bytes(dict(pipe.unet.config), mc, size, size)
            med = sorted(ts)[len(ts) // 2]
            row = dict(round=rnd, geometry=name, frames=F, latent=f"{size}x{size}", ddim_steps=bench.DDIM_STEPS, clip_s=[round(t, 3) for t in ts],
                       frames_per_s=round(F / med, 3), map_cache_bytes_per_frame_step=per_step, map_cache_mib_per_frame_step=round(per_step / 2 ** 20, 2),
                       peak_hbm_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), graph_plans=len(pipe._plans))
            rows[name].append(row)
            print(json.dumps(row), flush=True)
            if hasattr(pipe, "store_controller"):
                pipe.store_controller.reset()
            del pipe
            gc.collect()
            torch.cuda.empty_cache()
    summary = {n: dict(frames_per_s=[r["frames_per_s"] for r in rs], map_cache_mib_per_frame_step=rs[0]["map_cache_mib_per_frame_step"],
                       peak_hbm_gib=max(r["peak_hbm_gib"] for r in rs)) for n, rs in rows.items()}
    print(json.dumps(dict(summary=summary, workload=bench.CFG["workload"].replace("SD-1.4 UNet geometry", "SD-2-base / SD-1.4 UNet geometry"),
                          card=info)), flush=True)


if __name__ == "__main__":
    main()
