"""Frame-sharding parity on non-square clips: the frames of ONE 32x48-latent clip over the ranks of this job.
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29531 tools/shard_check_nonsquare.py
Checks (rank 0 prints one JSON line, exit code 1 on failure):
  * one CFG-batch UNet forward, sharded vs the same product on one GPU — tools/shard_check.py's bound, 4e-3 of max|eps|;
  * the non-square golden cases of the unmodified reference (oracle/nonsquare.py) whose frame count divides over the ranks, through the
    reference-facing pipeline API on the rank's frames — tests/test_gpu_nonsquare.py's bounds (inversion 2e-2, final edit 8e-2 relative);
  * CUDA-graph replay of the sharded loops (third run of a case) equals the eager sharded run bit for bit."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("FZ_P2P_ARENA_MB", "3072")
import _nonsquare as nsr  # noqa: E402
from fatezero_b200 import dist as fzdist, synth  # noqa: E402
from oracle import nonsquare as ns  # noqa: E402
from oracle import sd2  # noqa: E402


def gmax(v: float, dev) -> float:
    t = torch.tensor([float(v)], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    rank, world, local = fzdist.env_world()
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    fzdist.init("nccl", dev)
    out, ok = dict(world=world), True
    mc = dict(lora=160, SparseCausalAttention_index=["mid", -1, "first"], least_sc_channel=64)
    pipe = nsr.build_product("mini", mc, device=dev)
    x0 = (synth.synth_latents(2 * world, 32, 48) * 0.5).to(dev)
    x2 = torch.cat([x0, 0.7 * x0])
    emb = torch.randn(2, 77, synth.UNET_CONFIGS["mini"]["cross_attention_dim"], generator=torch.Generator().manual_seed(2)).to(dev)
    full = pipe.unet(x2, 481, emb).sample
    pipe.unet.set_frame_shard(rank, world)
    got = fzdist.gather_frames(pipe.unet(fzdist.frame_slice(x2, rank, world), 481, emb).sample, world)
    pipe.unet.set_frame_shard(0, 1)
    out["forward_max_abs"] = (got - full).abs().max().item()
    out["forward_ref_max"] = full.abs().max().item()
    ok &= out["forward_max_abs"] <= 4e-3 * max(out["forward_ref_max"], 1.0)
    del pipe
    for name in ns.NONSQUARE_REF_CASES:
        case = ns.NONSQUARE_CASES[name]
        if case["frames"] % world:
            continue
        g = nsr.load(name)
        pipe = nsr.build_product(case["unet"], case["model_config"], device=dev)
        pipe.unet.set_frame_shard(rank, world)
        runs = [nsr.run_product(case, pipe=pipe, device=dev, shard=(rank, world)) for _ in range(3)]  # eager, captured, replayed
        p = runs[0]
        inv = fzdist.gather_frames(p["inv_latents"].to(dev), world, dim=3).cpu()
        ed = fzdist.gather_frames(p["edit_latents"][-1:].to(dev), world, dim=3).cpu()
        e_inv = (torch.stack([sd2.sample(v, g["lat_stride"]) for v in inv]) - g["inv_sample"]).abs().max().item() / g["inv_sample"].abs().max().item()
        e_ed = (sd2.sample(ed[0], g["lat_stride"]) - g["edit_sample"][-1]).abs().max().item() / g["edit_sample"][-1].abs().max().item()
        same = all(torch.equal(r["inv_latents"], p["inv_latents"]) and torch.equal(r["edit_latents"], p["edit_latents"]) for r in runs[1:])
        same = gmax(0.0 if same else 1.0, dev) == 0.0
        out[name] = dict(inv_err=e_inv, edit_err=e_ed, graph_replay_equal=same, plans=len(pipe._plans))
        ok &= e_inv <= 2e-2 and e_ed <= 8e-2 and same and len(pipe._plans) == 2
        del pipe, runs
        torch.cuda.empty_cache()
    out["ok"] = bool(ok)
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
