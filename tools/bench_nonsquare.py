"""Edited frames per second on non-square clips against the square flagship workload: a style edit (Refine + Reweight, 8 frames, 50 inversion
+ 50 edit DDIM steps, SD-1.4 UNet geometry with synthetic weights, graph-captured loops) through the reference-facing API at 512x512,
512x768 and 512x896 pixels, the sizes alternating within every round.

One UNet serves every size.  Per round and size, two clips warm the size up (eager, then captured) and --clips clips are timed, wall clock
around a device synchronise; the size's graphs are then released, so only one size's map cache is held at a time.  Reported per size:
frames/s (frames / median clip seconds), the ratio to 512x512 in the same round, the map-cache bytes per frame and DDIM step
(controllers.map_cache_bytes: the non-square sizes store no 32x48 / 32x56 level, which holds more than 32**2 pixels) and the peak HBM
allocated while timing.  The card name, power limit and max SM clock are printed first.

    python tools/bench_nonsquare.py [--rounds 2] [--clips 3] [--frames 8]
Prints one JSON line per (round, size) and a summary line.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_sd2 import build_pipe, card  # noqa: E402

SIZES = ((512, 512), (512, 768), (512, 896))  # (height, width) in pixels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--clips", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nonsquare measures on a CUDA device; none is visible")
    from fatezero_b200 import controllers, synth
    from fatezero_b200.unet import unet_param_spec
    bench.select_config("style")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    F, mc = args.frames, bench.CFG["model_config"]
    spec = unet_param_spec(dict(synth.UNET_CONFIGS["sd14"]), mc)
    pipe = build_pipe("sd14", synth.synth_state_dict({k: v[0] for k, v in spec.items()}, seed=0), dev)
    emb = pipe._encode_prompt(bench.SRC, dev, 1, True, None)
    rows = {s: [] for s in SIZES}
    for rnd in range(args.rounds):
        square_fps = None
        for H, W in SIZES:
            h, w = H // 8, W // 8
            x0 = (synth.synth_latents(F, h, w) * 0.5).to(dev)
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
            med = sorted(ts)[len(ts) // 2]
            fps = F / med
            square_fps = fps if (H, W) == SIZES[0] else square_fps
            per_step, _ = controllers.map_cache_bytes(dict(pipe.unet.config), mc, h, w)
            row = dict(round=rnd, size=f"{H}x{W}", latent=f"{h}x{w}", frames=F, ddim_steps=bench.DDIM_STEPS, clip_s=[round(t, 3) for t in ts],
                       frames_per_s=round(fps, 3), vs_512x512=round(fps / square_fps, 3),
                       map_cache_mib_per_frame_step=round(per_step / 2 ** 20, 2), peak_hbm_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                       graph_plans=len(pipe._plans))
            rows[(H, W)].append(row)
            print(json.dumps(row), flush=True)
            pipe.store_controller.reset()
            pipe.release_graphs()
            del x0
            gc.collect()
            torch.cuda.empty_cache()
    summary = {f"{H}x{W}": dict(frames_per_s=[r["frames_per_s"] for r in rs], vs_512x512=[r["vs_512x512"] for r in rs],
                                map_cache_mib_per_frame_step=rs[0]["map_cache_mib_per_frame_step"], peak_hbm_gib=max(r["peak_hbm_gib"] for r in rs))
               for (H, W), rs in rows.items()}
    print(json.dumps(dict(summary=summary, workload=bench.CFG["workload"].replace("512x512", "512x512 / 512x768 / 512x896"), card=info)),
          flush=True)


if __name__ == "__main__":
    main()
