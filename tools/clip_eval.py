"""CLIP frame accuracy and temporal consistency of edited clips (the CLI of CLIP/frame_acc_tem_con.py) on the sm_90a kernels.

  python tools/clip_eval.py --checkpoint ~/.cache/clip/ViT-B-32.pt --results DIR --prompts CLIP/bench_clean_prompt.yaml

--results holds one subfolder of PNG frames per edit; each subfolder's name is a key of the --prompts YAML, whose entries carry `source`
and `target`.  All folders are scored in one batched pass.  Prints one JSON line per folder, then the dataset averages.  String prompts are
tokenized with OpenAI `clip.tokenize` (installed, or from $FATEZERO_REFERENCE_ROOT/CLIP)."""
import argparse
import glob
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checkpoint", required=True, help="OpenAI CLIP ViT TorchScript archive or state-dict file")
    ap.add_argument("--results", required=True, help="directory with one subfolder of PNG frames per edit")
    ap.add_argument("--prompts", required=True, help="YAML {folder name: {source: ..., target: ...}}")
    ap.add_argument("--device", default="cuda")
    a = ap.parse_args()
    import yaml
    from fatezero_b200.clip_eval import ClipEvaluator
    prompts = yaml.safe_load(open(a.prompts))
    folders = sorted(p for p in glob.glob(os.path.join(a.results, "*")) if os.path.isdir(p))
    missing = [os.path.basename(f) for f in folders if os.path.basename(f) not in prompts]
    if missing:
        raise SystemExit(f"no prompts for {missing} in {a.prompts}")
    if not folders:
        raise SystemExit(f"no result folders under {a.results}")
    ev = ClipEvaluator.load(a.checkpoint, a.device)
    by_source = {}
    for f in folders:
        by_source.setdefault(prompts[os.path.basename(f)]["source"], []).append(f)
    rows = {}
    for source, fs in by_source.items():
        res = ev.score_batch(fs, source, [prompts[os.path.basename(f)]["target"] for f in fs])
        for f, r in zip(fs, res):
            rows[os.path.basename(f)] = dict(folder_success_rate=r["accuracy"], folder_temporal_consistency=r["consistency"],
                                             frames=len(r["success"]))
    for name in sorted(rows):
        print(json.dumps(dict(folder=name, **rows[name])))
    print(json.dumps(dict(dataset_average_rate=float(np.mean([r["folder_success_rate"] for r in rows.values()])),
                          dataset_average_tempconst=float(np.mean([r["folder_temporal_consistency"] for r in rows.values()])),
                          folders=len(rows))))


if __name__ == "__main__":
    main()
