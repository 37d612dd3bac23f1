"""Text-to-video sampling (SpatioTemporalStableDiffusionPipeline.__call__): 512x512, 8 frames, 50 DDIM steps, CFG 7.5, SD-1.4 UNet geometry
with synthetic weights, graph-captured loop, for 1 / 2 / 4 clips per call at eta = 0 and eta = 1.

The configurations are measured in alternating rounds (every round visits each of them once); per round and configuration the pipeline has
already run the configuration twice (eager, then captured) and one call is timed, wall clock around a device synchronise.  Reported per
configuration: the median call seconds over rounds, frames/s (clips x frames / median seconds) and the peak HBM allocated while timing.  The
card name, power limit and max SM clock are read in the same run and printed first.

    python tools/bench_sample.py [--rounds 3] [--steps 50] [--frames 8]
Prints one JSON line per (round, configuration) and a summary line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [(clips, eta) for clips in (1, 2, 4) for eta in (0.0, 1.0)]
PROMPT = "a silver jeep driving down a curvy road in the countryside"


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:  # noqa: BLE001
        out = "unknown"
    return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out, query=q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--frames", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample measures on a CUDA device; none is visible")
    from fatezero_b200 import DDIMScheduler, SpatioTemporalStableDiffusionPipeline, UNetPseudo3DConditionModel, synth
    from fatezero_b200.unet import unet_param_spec
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    cfg, mc = synth.SD14_UNET_CONFIG, synth.DEFAULT_MODEL_CONFIG
    unet = UNetPseudo3DConditionModel(**cfg, **mc)
    unet.load_state_dict(synth.synth_state_dict({k: v[0] for k, v in unet_param_spec(dict(cfg), mc).items()}, seed=0))
    unet.to(dev)
    pipe = SpatioTemporalStableDiffusionPipeline(synth.VaeStub(), synth.ToyTextEncoder(cfg["cross_attention_dim"]).to(dev), synth.ToyTokenizer(),
                                                 unet, DDIMScheduler())

    def call(clips, eta):
        gen = torch.Generator(device=dev).manual_seed(0)
        return pipe(prompt=[PROMPT] * clips, height=512, width=512, num_inference_steps=args.steps, clip_length=args.frames,
                    guidance_scale=7.5, eta=eta, generator=gen, output_type="latent").images

    for c in CONFIGS:  # eager (configuration seen), then captured: the timed calls replay graphs
        call(*c)
        call(*c)
    times = {c: [] for c in CONFIGS}
    peaks = {c: 0 for c in CONFIGS}
    for rnd in range(args.rounds):
        for clips, eta in CONFIGS:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out = call(clips, eta)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert torch.isfinite(out).all()
            times[(clips, eta)].append(dt)
            peaks[(clips, eta)] = max(peaks[(clips, eta)], torch.cuda.max_memory_allocated())
            print(json.dumps(dict(round=rnd, clips=clips, eta=eta, seconds=round(dt, 3))), flush=True)
    rows = []
    for (clips, eta), ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        rows.append(dict(clips=clips, eta=eta, frames=args.frames, steps=args.steps, median_s=round(med, 3), s_per_clip=round(med / clips, 3),
                         frames_per_s=round(clips * args.frames / med, 3), peak_hbm_gib=round(peaks[(clips, eta)] / 2 ** 30, 2)))
    print(json.dumps(dict(summary=rows, graph_plans=len(pipe._plans),
                          workload="text-to-video 512x512, CFG 7.5, SD-1.4 UNet geometry, synthetic weights", card=info)), flush=True)


if __name__ == "__main__":
    main()
