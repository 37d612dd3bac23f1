"""K target prompts of ONE inverted clip: K sequential single-prompt edits against one batched edit (p2preplace_edit_batch).

Workload: bench.py's geometry (SD-1.4 UNet, non-degenerate synthetic weights, 512x512x8 frames, 50 DDIM steps), one inversion with STORE
(captured, so that the edit loops can be captured too), then for K in --ks: K prompts taken in order from PROMPTS (Refine+Reweight,
Replace + self-attention blend + latent blend, Refine, Replace).  Both paths are warmed (first call eager, second call captured) and then
timed alternately, --rounds times each, wall clock around a device synchronise.  Also reports the peak HBM use of each path, the card
name and its power limit, and checks that every prompt's final latents are bitwise equal between the two paths.

    python tools/bench_edit_batch.py [--ks 1,2,4] [--rounds 3] [--frames 8]
Prints one JSON line per K and a summary line; the VAE decode is not part of either path (output_type='latent').
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

SRC = bench.SRC
PROMPTS = [
    (bench.CONFIGS["style"]["tgt"], bench.CONFIGS["style"]["p2p"]),
    (bench.CONFIGS["attribute"]["tgt"], bench.CONFIGS["attribute"]["p2p"]),
    ("a silver jeep driving down a curvy road in the snowy countryside",
     dict(is_replace_controller=False, cross_replace_steps={"default_": 0.8}, self_replace_steps=0.8)),
    ("a silver tank driving down a curvy road in the countryside",
     dict(is_replace_controller=True, cross_replace_steps={"default_": 0.7}, self_replace_steps=0.6)),
]


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:  # noqa: BLE001
        out = "unknown"
    return dict(name=name, power_limit=out, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    args = ap.parse_args()
    from fatezero_b200 import controllers, synth
    bench.select_config("style")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pipe = bench.build_pipe(dev)
    F, size = args.frames, bench.CFG["size"]
    x0 = (synth.synth_latents(F, size, size) * 0.5).to(dev)
    emb = pipe._encode_prompt(SRC, dev, 1, True, None)
    for _ in range(2):  # eager, then captured + replayed: the store then lives in a captured plan and the edit loops can be captured
        pipe.store_controller = controllers.AttentionStore()
        controllers.register_attention_control(pipe, pipe.store_controller)
        pipe.store_controller.LOW_RESOURCE = True
        xT = pipe.ddim_clean2noisy_loop(x0, emb, pipe.store_controller)[-1]
        pipe.store_controller.LOW_RESOURCE = False
    save = tempfile.mkdtemp()
    N = bench.DDIM_STEPS

    def sequential(prompts):
        outs = []
        for p, c in prompts:
            r = pipe(prompt=p, source_prompt=SRC, edit_type="swap", latents=xT, num_inference_steps=N, guidance_scale=7.5, output_type="latent",
                     use_inversion_attention=True, save_self_attention=False, save_path=save, **c)
            outs.append(r["sdimage_output"].images)
        return outs

    def batched(prompts):
        res = pipe.p2preplace_edit_batch([p for p, _ in prompts], [dict(c, use_inversion_attention=True, save_self_attention=False) for _, c in prompts],
                                         SRC, xT, N, 7.5, save_path=save, output_type="latent")
        return [r["sdimage_output"].images for r in res]

    def timed(fn, prompts):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = fn(prompts)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, torch.cuda.max_memory_allocated(), out

    info = card()
    rows = []
    for K in [int(k) for k in args.ks.split(",")]:
        prompts = PROMPTS[:K]
        for _ in range(2):  # warm-up: eager, then capture
            sequential(prompts)
            batched(prompts)
        ts, tb, ms, mb = [], [], 0, 0
        for _ in range(args.rounds):
            t, m, out_s = timed(sequential, prompts)
            ts.append(t)
            ms = max(ms, m)
            t, m, out_b = timed(batched, prompts)
            tb.append(t)
            mb = max(mb, m)
        bitwise = all(torch.equal(a, b) for a, b in zip(out_s, out_b))
        row = dict(K=K, frames=F, latent=f"{size}x{size}", ddim_steps=N, sequential_s=sorted(ts)[len(ts) // 2], batched_s=sorted(tb)[len(tb) // 2],
                   sequential_all_s=[round(t, 3) for t in ts], batched_all_s=[round(t, 3) for t in tb],
                   peak_hbm_gib=dict(sequential=round(ms / 2 ** 30, 2), batched=round(mb / 2 ** 30, 2)), bitwise_equal=bitwise, card=info)
        row["speedup"] = round(row["sequential_s"] / row["batched_s"], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(summary=[(r["K"], round(r["sequential_s"], 3), round(r["batched_s"], 3), r["speedup"], r["bitwise_equal"]) for r in rows],
                          columns=["K", "sequential_s", "batched_s", "speedup", "bitwise_equal"], card=info)), flush=True)


if __name__ == "__main__":
    main()
