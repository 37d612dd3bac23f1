"""The HBM-bound kernels for `ncu --set full` (one launch each, inputs produced right before, i.e. L2-warm like in the step), or, with
--time N, the mean device time per call of each over N back-to-back calls (CUDA events):
GroupNorm+SiLU 16x4096x320 (joint over 8 frames), GroupNorm 16x4096x960, LayerNorm 65536x320, temporal attention r=64 / r=32 / r=16,
plus small tap-GEMMs (to_out 65536x320x320 with bias+residual, r=8 conv 1280->1280)."""
import argparse, json, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fatezero_b200 import _lib, ops
ap = argparse.ArgumentParser()
ap.add_argument("--time", type=int, default=0, metavar="N", help="time N calls of each kernel instead of one profiled launch")
args = ap.parse_args()
dev = "cuda"
x320 = torch.randn(16, 4096, 320, device=dev).half(); x960 = torch.randn(16, 4096, 960, device=dev).half()
g320, b320 = torch.ones(320, device=dev), torch.zeros(320, device=dev)
g960, b960 = torch.ones(960, device=dev), torch.zeros(960, device=dev)
xl = torch.randn(65536, 320, device=dev).half()
qkv64 = torch.randn(2 * 8 * 4096, 960, device=dev).half(); qkv32 = torch.randn(2 * 8 * 1024, 1920, device=dev).half()
qkv16 = torch.randn(2 * 8 * 256, 3840, device=dev).half()
a = torch.randn(65536, 320, device=dev).half(); w = torch.randn(320, 320, device=dev).half() * 0.05; bias = torch.zeros(320, device=dev)
res = torch.randn(65536, 320, device=dev).half()
x8 = torch.randn(16, 8, 8, 1280, device=dev).half(); w8 = torch.randn(9, 1280, 1280, device=dev).half() * 0.01
fns = {"gn_silu_16x4096x320": lambda: ops.groupnorm(x320, g320, b320, 1e-5, 32, 8, True),
       "gn_silu_16x4096x960": lambda: ops.groupnorm(x960, g960, b960, 1e-5, 32, 8, True),
       "ln_65536x320": lambda: ops.layernorm(xl, g320, b320),
       "tattn_r64": lambda: ops.temporal_attn(qkv64, 2, 8, 4096, 8, 40, 40 ** -0.5),
       "tattn_r32": lambda: ops.temporal_attn(qkv32, 2, 8, 1024, 8, 80, 80 ** -0.5),
       "tattn_r16": lambda: ops.temporal_attn(qkv16, 2, 8, 256, 8, 160, 160 ** -0.5),
       "to_out_gemm": lambda: ops.gemm(a, w, bias=bias, residual=res), "conv_r8": lambda: ops.conv3x3(x8, w8)}
for _ in range(2):
    for f in fns.values(): f()
torch.cuda.synchronize()
if args.time:
    out = {}
    for name, f in fns.items():
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.time): f()
        t1.record()
        torch.cuda.synchronize()
        out[name] = round(1000 * t0.elapsed_time(t1) / args.time, 2)
    # the card's power limit and max SM clock belong beside its timings (read-only query)
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps(dict(lib=os.path.basename(_lib.LIB_PATH), gpu=torch.cuda.get_device_name(), power_limit_and_max_sm_clock=q.stdout.strip(),
                          us_per_call=out)), flush=True)
else:
    torch.cuda.profiler.start()
    for f in fns.values(): f()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
