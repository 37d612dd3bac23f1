"""Representative launches of the two tensor-core kernels for `ncu --set full`:
  1) 3x3 conv 320->320 at 64x64, B*F=16     (tapgemm<160>, 9 taps)      2) linear 65536 x 960 x 320 (QKV, V^T epilogue off)
  3) GEGLU linear 65536 x 2560 x 320         (tapgemm<256>)              4) ST-attention r=64 d=40 (no hook)
  5) ST-attention r=32 d=80 STORE            6) ST-attention r=32 d=80 REPLACE"""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fatezero_b200 import _lib, ops
dev = "cuda"
x = torch.randn(16, 64, 64, 320, device=dev).half(); w9 = torch.randn(9, 320, 320, device=dev).half() * 0.02
a = torch.randn(65536, 320, device=dev).half(); w = torch.randn(960, 320, device=dev).half() * 0.05
wg = torch.randn(2560, 320, device=dev).half() * 0.05; bg = torch.zeros(2560, device=dev)
wp, bp, bn = ops.pack_geglu(wg.float(), bg)
wp = wp.half()
def attn(S, d, mode):
    BF, heads = 16, 8
    C_ = heads * d
    q = torch.randn(BF * S, C_, device=dev).half(); k = torch.randn(BF * S, C_, device=dev).half()
    vt = torch.randn(BF, heads, d, S, device=dev).half(); out = torch.empty(BF * S, C_, device=dev, dtype=torch.float16)
    si = [[(b * 8 + 3) for b in range(2) for f in range(8)]]
    kw = dict(S_q=S, keys_per_slot=S, n_src=BF, d=d, heads=heads, F=8, BF=BF, scale=d ** -0.5, src_index=si)
    cache = torch.empty(BF, heads, S, S, device=dev, dtype=torch.float16) if mode != "none" else None
    if mode == "replace":
        cache.copy_(torch.softmax(torch.randn(BF, heads, S, S, device=dev), -1))
    if mode == "store": return lambda: ops.attention(q, k, vt, out, **kw, row_mode=_lib.ATTN_STORE, store=cache, cache_ld=S)
    if mode == "replace": return lambda: ops.attention(q, k, vt, out, **kw, row_mode=_lib.ATTN_REPLACE, base=cache, cache_ld=S)
    return lambda: ops.attention(q, k, vt, out, **kw)
vt_out = torch.empty(16, 8, 40, 4096, device=dev, dtype=torch.float16)


def cross(S, d):
    BF, heads = 16, 8
    C_ = heads * d
    q = torch.randn(BF * S, C_, device=dev).half(); k = torch.randn(2 * 77, C_, device=dev).half()
    vt = torch.zeros(2, heads, d, 80, device=dev, dtype=torch.float16); vt[..., :77] = torch.randn(2, heads, d, 77, device=dev).half()
    out = torch.empty(BF * S, C_, device=dev, dtype=torch.float16)
    return lambda: ops.attention(q, k, vt, out, S_q=S, keys_per_slot=77, n_src=2, d=d, heads=heads, F=8, BF=BF, scale=d ** -0.5,
                                 src_index=[[b for b in range(2) for _ in range(8)]])


# 7) QKV linear 65536 x 960 x 320 with the V^T third written transposed (staged TMA store)   8) text cross-attention r=64 d=40 (streaming kernel)
fns = [lambda: ops.conv3x3(x, w9), lambda: ops.gemm(a, w), lambda: ops.gemm(a, wp, bias=bp, geglu=True, force_bn=bn),
       attn(4096, 40, "none"), attn(1024, 80, "store"), attn(1024, 80, "replace"),
       lambda: ops.gemm(a, w, vt=dict(out=vt_out, col_start=640, S=4096, d=40, heads=8)), cross(4096, 40)]
for _ in range(2):
    for f in fns: f()
torch.cuda.synchronize()
torch.cuda.profiler.start()
for f in fns: f()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
