"""K source clips: K sequential (inversion + edit) runs against one batched inversion plus one batched edit
(prepare_latents_ddim_inverted_batch + p2preplace_edit_clips).

Workload: bench.py's `style` geometry (SD-1.4 UNet, non-degenerate synthetic weights, 512x512, Refine+Reweight, one target prompt per clip),
K distinct synthetic clips of F frames, for (F, steps) in --shapes and K in --ks.  A (F, K) point whose map caches the HBM admission check
of the batched inversion refuses is reported as refused.  Both paths run with CUDA graphs (first call eager, second captured, later calls
replayed) and are timed alternately, --rounds times each (the median is reported), wall clock around a device synchronise; the VAE is not part of either path
(latents in, latents out).  Reports the peak HBM of each path, whether every clip's final latents are bitwise equal between the two paths,
and the card name and power limit read in the same run.

    python tools/bench_multiclip.py [--shapes 1:50,2:50,4:50,8:10] [--ks 1,2,4,8] [--rounds 3]
Prints one JSON line per point and a summary line.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from bench_edit_batch import card  # noqa: E402

SRC = bench.SRC


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1:50,2:50,4:50,8:10")
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from fatezero_b200 import controllers, synth
    bench.select_config("style")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = bench.build_pipe(dev)
    size, tgt, p2p = bench.CFG["size"], bench.CFG["tgt"], dict(bench.CFG["p2p"], use_inversion_attention=True, save_self_attention=False)
    emb = pipe._encode_prompt(SRC, dev, 1, True, None)
    info = card()
    rows = []
    for shape in args.shapes.split(","):
        F, N = (int(v) for v in shape.split(":"))
        base = (synth.synth_latents(F, size, size) * 0.5).to(dev)
        for K in [int(k) for k in args.ks.split(",")]:
            clips = [base.roll(7 * k, -1) * (1.0 - 0.05 * k) for k in range(K)]
            # drop everything the previous point kept alive (captured plans, stores, edit controllers) before admitting this one
            out_s = out_b = None
            pipe.release_graphs()
            controllers.register_attention_control(pipe, pipe.empty_controller)
            pipe.store_controller = controllers.AttentionStore()
            pipe.store_controllers = pipe.last_edit_controller = pipe.last_edit_controllers = None
            torch.cuda.empty_cache()

            def sequential():
                outs = []
                for x0 in clips:
                    pipe.scheduler.set_timesteps(N)
                    pipe.store_controller = pipe.last_edit_controller = None  # the previous clip's cache is released before this clip's
                    pipe.store_controller = controllers.AttentionStore()
                    controllers.register_attention_control(pipe, pipe.store_controller)
                    pipe.store_controller.LOW_RESOURCE = True
                    xT = pipe.ddim_clean2noisy_loop(x0, emb, pipe.store_controller)[-1]
                    pipe.store_controller.LOW_RESOURCE = False
                    r = pipe(prompt=tgt, source_prompt=SRC, edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5,
                             output_type="latent", **p2p)
                    outs.append(r["sdimage_output"].images)
                return outs

            def batched():
                pipe.scheduler.set_timesteps(N)
                # the previous call's stores (and the edit controllers that read them) are released before the batched inversion is admitted
                pipe.store_controllers = pipe.last_edit_controllers = None
                lats = pipe.prepare_latents_ddim_inverted_batch([SRC] * K, latents=clips)
                jobs = [dict(p2p, store=s, latents=l[-1], prompt=tgt, source_prompt=SRC) for s, l in zip(pipe.store_controllers, lats)]
                res = pipe.p2preplace_edit_clips(jobs, N, 7.5, output_type="latent")
                return [r["sdimage_output"].images for r in res]

            def timed(fn):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                return time.perf_counter() - t0, torch.cuda.max_memory_allocated(), out

            ts, tb, ms, mb, bitwise = [], [], 0, 0, True
            try:
                for _ in range(2):  # warm-up: eager, then capture
                    sequential()
                    batched()
                for _ in range(args.rounds):
                    t, m, out_s = timed(sequential)
                    ts.append(t)
                    ms = max(ms, m)
                    t, m, out_b = timed(batched)
                    tb.append(t)
                    mb = max(mb, m)
                    bitwise = bitwise and all(torch.equal(a, b) for a, b in zip(out_s, out_b))
            except (ValueError, torch.OutOfMemoryError) as e:
                # ValueError: the batched inversion's HBM admission check refused the batch
                row = dict(K=K, frames=F, ddim_steps=N, refused=f"{type(e).__name__}: {str(e).splitlines()[0]}", card=info)
                rows.append(row)
                print(json.dumps(row), flush=True)
                continue
            row = dict(K=K, frames=F, latent=f"{size}x{size}", ddim_steps=N, sequential_s=statistics.median(ts),
                       batched_s=statistics.median(tb), sequential_all_s=[round(t, 3) for t in ts], batched_all_s=[round(t, 3) for t in tb],
                       peak_hbm_gib=dict(sequential=round(ms / 2 ** 30, 2), batched=round(mb / 2 ** 30, 2)), bitwise_equal=bitwise, card=info)
            row["speedup"] = round(row["sequential_s"] / row["batched_s"], 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(dict(summary=[(r["frames"], r["ddim_steps"], r["K"], round(r["sequential_s"], 3), round(r["batched_s"], 3), r["speedup"],
                                    r["peak_hbm_gib"]["sequential"], r["peak_hbm_gib"]["batched"], r["bitwise_equal"])
                                   for r in rows if "refused" not in r],
                          refused=[(r["frames"], r["ddim_steps"], r["K"]) for r in rows if "refused" in r],
                          columns=["frames", "ddim_steps", "K", "sequential_s", "batched_s", "speedup", "peak_seq_gib", "peak_batch_gib",
                                   "bitwise_equal"], card=info)), flush=True)


if __name__ == "__main__":
    main()
