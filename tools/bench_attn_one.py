"""Single attention configurations (S=4096 d=40 without a controller hook by default). MODE=none|store|replace S=.. D=.."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fatezero_b200 import _lib, ops
dev = "cuda"
S, d, heads, BF = int(os.environ.get("S", 4096)), int(os.environ.get("D", 40)), 8, int(os.environ.get("BF", 16))
mode = os.environ.get("MODE", "none")
C_ = heads * d
q = torch.randn(BF * S, C_, device=dev).half(); k = torch.randn(BF * S, C_, device=dev).half()
vt = torch.randn(BF, heads, d, S, device=dev).half(); out = torch.empty(BF * S, C_, device=dev, dtype=torch.float16)
si = [[(b * 8 + 3) for b in range(BF // 8) for f in range(8)]] if BF >= 8 else [list(range(BF))]
if os.environ.get("SLOTS", "1") == "2":  # the real sparse-causal pattern: [previous frame, first frame]
    si = [[b * 8 + max(f - 1, 0) for b in range(BF // 8) for f in range(8)], [b * 8 for b in range(BF // 8) for f in range(8)]]
kw = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=min(8, BF), BF=BF, scale=d ** -0.5, src_index=si)
cache = torch.empty(BF, heads, S, S, device=dev, dtype=torch.float16) if mode != "none" else None
if mode == "replace":
    cache.copy_(torch.softmax(torch.randn(BF, heads, S, S, device=dev), -1))
def fn():
    if mode == "store": ops.attention(q, k, vt, out, **kw, row_mode=_lib.ATTN_STORE, store=cache, cache_ld=S)
    elif mode == "replace": ops.attention(q, k, vt, out, **kw, row_mode=_lib.ATTN_REPLACE, base=cache, cache_ld=S)
    else: ops.attention(q, k, vt, out, **kw)
for _ in range(3): fn()
torch.cuda.synchronize()
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
for _ in range(5): fn()
e.record(); torch.cuda.synchronize()
ms = s.elapsed_time(e) / 5
print(dict(S=S, d=d, mode=mode, ms=ms, tflops=4 * BF * heads * S * S * len(si) * d / ms / 1e9))
