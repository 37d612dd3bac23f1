"""Time the CLIP scoring of K edited clips of 8 frames at 512x512 (frame accuracy + temporal consistency, CLIP/frame_acc_tem_con.py):
  ours : device uint8 frames -> ClipEvaluator.score_batch (one image-tower pass over all frames, one text-tower pass over the prompts);
  ref  : the reference's shape: per frame a PIL crop + Resize + CenterCrop + ToTensor + Normalize on the host, then an fp16 CLIP ViT-B/32
         (oracle/clip_oracle.py cast to fp16, torch on the GPU) with encode_image and model(image, text): two image encodes and two text
         encodes of the (source, target) pair per frame, then the consistency from the features.
Synthetic ViT-B/32 weights (same FLOPs as the real model).  Host clock around work that ends in a device synchronise; the two paths are
timed alternately.  Prints one JSON line with the card's name, power limit and max SM clock.
Usage: python tools/bench_clip_eval.py [--ks 1,4,8] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fatezero_b200 import clip_eval  # noqa: E402
from oracle import clip_oracle as co  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,4,8")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from PIL import Image
    dev = torch.device("cuda")
    sd = co.synth_clip_state_dict(0)
    ev = clip_eval.ClipEvaluator.from_state_dict(sd, dev)
    ref = co.ClipOracle(*co.VITB32)
    ref.load_state_dict(sd)
    ref = ref.half().eval().requires_grad_(False).to(dev)
    rng = np.random.default_rng(0)
    base = co.synth_clip_frames()["clip512"]
    src = torch.randint(1, 49406, (1, 77), generator=torch.Generator().manual_seed(1))
    src[0, 0], src[0, 12], src[0, 13:] = 49406, 49407, 0
    out = dict(gpu=torch.cuda.get_device_name(), frames_per_clip=8, size=512, results={})
    for K in [int(k) for k in a.ks.split(",")]:
        clips = [np.ascontiguousarray(base[rng.permutation(8)]) for _ in range(K)]
        tg = src.repeat(K, 1)
        tg[:, 5] = torch.arange(K) + 100
        dclips = [torch.from_numpy(c).to(dev) for c in clips]

        def ours():
            r = ev.score_batch(dclips, src[0], list(tg))
            torch.cuda.synchronize()
            return r

        @torch.no_grad()
        def reference():
            res = []
            for k, c in enumerate(clips):
                text = torch.cat([src, tg[k:k + 1]]).to(dev)
                feats, count = [], 0
                for f in c:
                    image = co.preprocess(co.crop_read(Image.fromarray(f)))[None].to(dev).half()
                    feats.append(ref.encode_image(image))
                    ref.encode_text(text)
                    probs = ref(image, text)[0].softmax(dim=-1).cpu().numpy()
                    count += float(probs[0, 1] >= probs[0, 0])
                nf = [f / torch.sqrt(torch.sum(f ** 2, axis=1, keepdims=True)) for f in feats]
                cons = sum(torch.sum(nf[i] * nf[i + 1], axis=1) for i in range(len(nf) - 1)) / (len(nf) - 1)
                res.append((count / len(c), float(cons)))
            torch.cuda.synchronize()
            return res

        ours(), reference()  # warm-up: every shape of the timed window
        t_ours, t_ref = [], []
        for _ in range(a.reps):
            for fn, acc in ((ours, t_ours), (reference, t_ref)):
                t0 = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t0)
        r_ours, r_ref = ours(), reference()
        out["results"][K] = dict(ours_s=[round(t, 4) for t in t_ours], reference_shaped_s=[round(t, 4) for t in t_ref],
                                 speedup_median=round(float(np.median(t_ref) / np.median(t_ours)), 2),
                                 ours_frames_per_s=round(8 * K / float(np.median(t_ours)), 1),
                                 consistency_ours=[round(r["consistency"], 5) for r in r_ours],
                                 consistency_ref_fp16=[round(c, 5) for _, c in r_ref],
                                 accuracy_ours=[r["accuracy"] for r in r_ours], accuracy_ref_fp16=[acc for acc, _ in r_ref])
        print(json.dumps({K: out["results"][K]}), flush=True)
    # the card's power limit and max SM clock belong beside its timings (read-only query)
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    out["power_limit_and_max_sm_clock"] = q.stdout.strip()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
