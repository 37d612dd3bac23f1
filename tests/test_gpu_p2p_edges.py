"""The peer-memory exchange of the frame-sharded forward (fz_p2p.cu) on ONE GPU: every rank is a plain buffer on the same device, so the
copies, flags, inboxes and epochs of fz_p2p_push / fz_p2p_wait / fz_gn_combine are checked bit for bit without IPC, torch.distributed or
a second process.  The fp64 reference of the statistics fold is gn_combine_ref / check_gn_combine in tests/_ref64.py.

Code path                                                          reached by
-----------------------------------------------------------------  ----------------------------------------------------------------
fz_p2p_push 2-D copies: rows = 1 / row_bytes = 16, source and       test_push_copies
  destination pitches > row_bytes, one segment past the host's
  cap on gx (grid-stride loop, 8 passes per thread), 96 segments
  of mixed sizes at gx = 4 (CTAs that copy nothing still arrive),
  local copies only (dst_slot = -1, n_dst = 0); sentinel-filled
  destinations with guard bytes, every byte outside the segments
  untouched; two launches bitwise equal
last-CTA epilogue: the arrival counter back at 0 after every        test_push_copies
  launch; 16 destination flags (the maximum) exactly 1 with their
  neighbours unchanged; wait_flags with wait_mask bits (bit 31,
  all 32) pre-raised by the test: cleared, other words unchanged
host refusals (error, nothing written): src / dst / pitch /         test_push_refusals
  row_bytes not a multiple of 16, n_segs 0 / 97, n_dst 17, a null
  flag, a null counter
fz_p2p_wait: pre-raised flags of the mask cleared, other words      test_wait, test_wait_mask_zero_launches_nothing
  kept; mask = 0 launches no kernel
fz_gn_combine: {value, epoch + 1} words sent to every peer (not to  test_gn_combine
  slot me, nothing past n), the fp64 fold over ranks and frames
  bitwise against the replay and within the summation bound of
  fsum, non-first slots of every set zeroed, the sums left
  unchanged, nothing past n of the totals written, the epoch word
  advanced; a second call
  on the same site at epoch + 2; the epoch wrapping from 2^32 - 1
  to 0; one CUDA-graph capture replayed twice.  world in {1, 2, 3,
  8, 32}, me first / middle / last, F_loc in {1, 2, 3, 8}, G = 32
  and odd G (1, 5, 7, 11), n = NB G = 1024, 1023, 63, 40
fz_gn_combine host refusals: n = 1025, NB % F_loc != 0, world 0 /  test_gn_combine_refusals
  33, me out of range, a null peer pointer, null totals (nothing
  written)
the engine's exchange helpers with the real kernels on simulated   test_sim_halo, test_sim_kv_exchange, test_sim_temporal_attn,
  ranks (one thread and one slab per rank, world 2 / 4 / 8):         test_sim_conv_out_gather, test_sim_gn_joint
  _halo_ext, _kv_exchange (constant-index and all-gather paths),
  _temporal_attn_sharded, the conv_out gather of _finish and
  _gn_joint (random and constant groups, SiLU on and off; 6 and
  12 frames of 1023 pixels, whose constant-group totals are exact
  in fp64 but not in fp32), every flag word and arrival counter 0
  afterwards

No launch here can spin.  spin_until_raised and the combine's polling loop trap after 30 s, so every flag a launch waits on and every
inbox word a combine reads is written in stream order before the launch and read back on the host, after a synchronize, before the launch
is issued: a staging mistake fails as a Python assertion.  For the same reason nothing here tests that a stale epoch or a missing flag is
ignored: such a test can only end in a spin or a trap.

The simulated ranks share one stream, on which the production exchange (push, then wait inside the same launch) would wait for a push
that is queued behind it.  SimArena therefore overrides exchange() alone: the real push with no sources, a barrier (every rank's push is
queued), a host check that exactly the expected flags are raised, fz_p2p_wait on them, and a second barrier so that no rank queues the
next push to a site before every rank has queued its wait for the previous one.  _gn_joint's combine is wrapped in the same way: each rank
stages its words into the peers' inboxes first, and ops.groupnorm_stats (a view into the workspace every rank shares) runs under a lock
and returns a clone."""
import ctypes as C
import threading

import pytest
import torch

from _ref64 import check_attn, check_gn_combine, f32, gn_check, softmax64
from fatezero_b200 import _lib, ops, p2p
from fatezero_b200._lib import P2PSeg
from fatezero_b200.engine import UNetEngine, sc_frame_indices

pytestmark = pytest.mark.gpu

dev = "cuda"
f16 = torch.float16
i32 = torch.int32
SENT = 0xA5          # destination byte sentinel
SENT32 = 0x5A5A5A5A  # word sentinel


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed * 7919 + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def raw(ptr: int, nbytes: int, dtype=torch.uint8) -> torch.Tensor:
    """Device memory at ptr as a tensor (the arena and inbox words the kernels address by pointer)."""
    return torch.as_tensor(p2p._Raw(ptr, nbytes), device=dev).view(dtype)


def s32(v: int) -> int:
    """A uint32 value as the int32 a tensor stores."""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def push(segs, flags, counter, wait_flags=None, wait_mask=0, n_segs=None, n_dst=None):
    """fz_p2p_push; segs = (src, src_pitch, dst, dst_pitch, rows, row_bytes, dst_slot) with raw pointers."""
    arr = (P2PSeg * max(1, len(segs)))()
    for i, (src, sp, dst, dp, rows, rb, slot) in enumerate(segs):
        arr[i].src, arr[i].src_pitch, arr[i].dst, arr[i].dst_pitch, arr[i].rows, arr[i].row_bytes, arr[i].dst_slot = src, sp, dst, dp, rows, rb, slot
    fl = (C.c_void_p * max(1, len(flags)))(*flags)
    _lib.call("fz_p2p_push", arr, len(segs) if n_segs is None else n_segs, fl, C.c_void_p(counter), len(flags) if n_dst is None else n_dst,
              C.c_void_p(wait_flags) if wait_flags else None, wait_mask, ops._stream())


def push_gx(specs):
    """The host's grid x of fz_p2p_push (about 8 vectors per thread, capped at 296 / n_segs + 1)."""
    max_vec = max(rows * (rb // 16) for rows, rb, _, _ in specs)
    return max(1, min(296 // len(specs) + 1, (max_vec + 2047) // 2048))


# ------------------------------------------------------------------------------------------------------------------ fz_p2p_push
class CopyCase:
    """Sources, a sentinel-filled destination pool with 64 guard bytes around every region, flag words, an arrival counter and wait
    words, all on the device, plus the host's expectation of each after one push.  specs: (rows, row_bytes, src_pitch, dst_pitch)."""

    GUARD = 64

    def __init__(self, specs, n_dst=0, wait_mask=0, seed=0):
        self.specs, self.n_dst, self.wait_mask = specs, n_dst, wait_mask
        so = do = self.GUARD
        self.offs = []
        for rows, rb, sp, dp in specs:
            self.offs.append((so, do))
            so += ((rows - 1) * sp + rb + 15) // 16 * 16 + self.GUARD
            do += ((rows - 1) * dp + rb + 15) // 16 * 16 + self.GUARD
        g = torch.Generator().manual_seed(seed)
        self.src = torch.randint(0, 256, (so,), generator=g, dtype=torch.uint8).to(dev)
        self.dst = torch.empty(do, dtype=torch.uint8, device=dev)
        # 16 flag slots at the odd words, their neighbours hold distinct non-zero values; the counter sits between two guard words
        self.flag_init = torch.tensor([0 if (i % 2 and i < 2 * n_dst) else s32(0x3C000000 + i) for i in range(40)], dtype=i32)
        self.flags = torch.empty(40, dtype=i32, device=dev)
        self.cnt_init = torch.tensor([s32(0x7E000000), 0, s32(0x7E000002)], dtype=i32)
        self.counter = torch.empty(3, dtype=i32, device=dev)
        # wait words: mask bits pre-raised with non-zero values, the other words (and 8 guard words past 32) non-zero and not in the mask
        self.wait_init = torch.tensor([(i + 1) * 977 if i < 32 and (wait_mask >> i) & 1 else s32(0x2B000000 + i) for i in range(40)], dtype=i32)
        self.wait = torch.empty(40, dtype=i32, device=dev)
        exp = torch.full((do,), SENT, dtype=torch.uint8)
        src_h = self.src.cpu()
        for (rows, rb, sp, dp), (s0, d0) in zip(specs, self.offs):
            exp.as_strided((rows, rb), (dp, 1), d0).copy_(src_h.as_strided((rows, rb), (sp, 1), s0))
        self.exp = exp

    def stage(self):
        self.dst.fill_(SENT)
        self.flags.copy_(self.flag_init)
        self.counter.copy_(self.cnt_init)
        self.wait.copy_(self.wait_init)
        torch.cuda.synchronize()
        assert torch.equal(self.wait.cpu(), self.wait_init) and torch.equal(self.counter.cpu(), self.cnt_init)
        raised = [i for i in range(32) if (self.wait_mask >> i) & 1]
        assert all(int(self.wait_init[i]) != 0 for i in raised), "a waited-on flag was not raised before the launch"

    def segs(self):
        fb = self.flags.data_ptr()
        return [(self.src.data_ptr() + s0, sp, self.dst.data_ptr() + d0, dp, rows, rb, (i % self.n_dst) if self.n_dst else -1)
                for i, ((rows, rb, sp, dp), (s0, d0)) in enumerate(zip(self.specs, self.offs))], [fb + 4 * (2 * k + 1) for k in range(self.n_dst)]

    def run(self):
        self.stage()
        segs, flags = self.segs()
        push(segs, flags, self.counter.data_ptr() + 4, self.wait.data_ptr() if self.wait_mask else None, self.wait_mask)
        torch.cuda.synchronize()
        return self.dst.cpu()

    def check_state(self, dst):
        diff = int((dst != self.exp).sum().item())
        assert diff == 0, f"{diff} destination bytes differ from the expected copy (segments, gaps or guards)"
        want_flags = self.flag_init.clone()
        want_flags[1:2 * self.n_dst:2] = 1
        assert torch.equal(self.flags.cpu(), want_flags), "destination flags not exactly 1, or a neighbouring word changed"
        assert torch.equal(self.counter.cpu(), torch.tensor([s32(0x7E000000), 0, s32(0x7E000002)], dtype=i32)), "arrival counter not back at 0"
        want_wait = self.wait_init.clone()
        for i in range(32):
            if (self.wait_mask >> i) & 1:
                want_wait[i] = 0
        assert torch.equal(self.wait.cpu(), want_wait), "wait flags: a raised flag not cleared, or a word outside the mask changed"


def _mixed96():
    specs = [(100, 1024, 1024, 1040)]  # 6400 vectors: gx = min(296 / 96 + 1, 4) = 4
    for i in range(95):
        rows, rb = 1 + i % 3, 16 * (1 + i % 4)
        specs.append((rows, rb, rb + 16 * (i % 2), rb + 16 * (i % 3)))
    return specs


PUSH_CASES = {
    "rows1_16B": dict(specs=[(1, 16, 16, 16)]),
    "pitched": dict(specs=[(37, 48, 80, 48), (5, 32, 32, 4096), (9, 160, 176, 192)], n_dst=2),
    "grid_stride": dict(specs=[(4097, 2400, 2416, 2432)], n_dst=1),
    "96_segs_16_flags": dict(specs=_mixed96(), n_dst=16),
    "local_only": dict(specs=[(3, 64, 64, 64), (2, 16, 48, 32)], n_dst=0),
    "wait_bit31": dict(specs=[(2, 32, 32, 48)], n_dst=3, wait_mask=0x800000F1),
    "wait_all32": dict(specs=[(1, 16, 16, 16)], n_dst=16, wait_mask=0xFFFFFFFF),
}


@pytest.mark.parametrize("name", PUSH_CASES)
def test_push_copies(name, report):
    case = CopyCase(**PUSH_CASES[name], seed=len(name))
    gx = push_gx(case.specs)
    vec = max(rows * (rb // 16) for rows, rb, _, _ in case.specs)
    if name == "grid_stride":
        assert gx == 297 and vec > 8 * gx * 256, "the segment no longer needs the grid-stride loop"
    if name == "96_segs_16_flags":
        assert len(case.specs) == 96 and gx == 4
    first = case.run()
    case.check_state(first)
    second = case.run()
    case.check_state(second)
    assert torch.equal(first, second), "two identical launches differ"
    report[name] = dict(segments=len(case.specs), gx=gx, ctas=gx * len(case.specs), max_vectors=vec, n_dst=case.n_dst, wait_mask=hex(case.wait_mask))


def _refusal_variants(case):
    """(what, segs, flags, counter, n_segs, n_dst, message) variants of one valid launch, each refused by the host checks."""
    segs, flags = case.segs()
    cnt = case.counter.data_ptr() + 4

    def seg(i, k, v):
        s = list(segs[i])
        s[k] = s[k] + v if k in (0, 2) else v
        return [tuple(s) if j == i else x for j, x in enumerate(segs)]
    addr = "not 16-byte addressable"
    return [
        ("src+8", seg(1, 0, 8), flags, cnt, None, None, addr),
        ("dst+8", seg(0, 2, 8), flags, cnt, None, None, addr),
        ("src_pitch40", seg(0, 1, 40), flags, cnt, None, None, addr),
        ("dst_pitch40", seg(1, 3, 40), flags, cnt, None, None, addr),
        ("row_bytes24", seg(0, 5, 24), flags, cnt, None, None, addr),
        ("n_segs0", segs, flags, cnt, 0, None, "unsupported"),
        ("n_segs97", segs * 49, flags, cnt, 97, None, "unsupported"),
        ("n_dst17", segs, flags * 9, cnt, None, 17, "unsupported"),
        ("null_flag", segs, [flags[0], None], cnt, None, None, "null flag"),
        ("null_counter", segs, flags, None, None, None, "unsupported"),
    ]


def test_push_refusals():
    case = CopyCase([(3, 64, 80, 96), (2, 32, 32, 48)], n_dst=2, wait_mask=0x3)
    for what, segs, flags, cnt, n_segs, n_dst, msg in _refusal_variants(case):
        case.stage()
        with pytest.raises(RuntimeError, match=msg):
            push(segs, flags, cnt, case.wait.data_ptr(), case.wait_mask, n_segs=n_segs, n_dst=n_dst)
        torch.cuda.synchronize()
        assert torch.all(case.dst.cpu() == SENT), f"{what}: a refused push wrote a destination"
        assert torch.equal(case.flags.cpu(), case.flag_init), f"{what}: a refused push raised a flag"
        assert torch.equal(case.counter.cpu(), case.cnt_init), f"{what}: a refused push touched the counter"
        assert torch.equal(case.wait.cpu(), case.wait_init), f"{what}: a refused push cleared a wait flag"
    case.check_state(case.run())  # the same launch without the defect goes through


# ------------------------------------------------------------------------------------------------------------------ fz_p2p_wait
@pytest.mark.parametrize("mask", [0x1, 0x80000000, 0x8000A5A1, 0xFFFFFFFF])
def test_wait(mask):
    init = torch.tensor([(i + 3) * 131 if i < 32 and (mask >> i) & 1 else s32(0x61000000 + i) for i in range(36)], dtype=i32)
    words = init.to(dev)
    torch.cuda.synchronize()
    assert torch.equal(words.cpu(), init) and all(int(init[i]) != 0 for i in range(32) if (mask >> i) & 1)
    _lib.call("fz_p2p_wait", C.c_void_p(words.data_ptr()), mask, ops._stream())
    torch.cuda.synchronize()
    want = init.clone()
    want[[i for i in range(32) if (mask >> i) & 1]] = 0
    assert torch.equal(words.cpu(), want)


def test_wait_mask_zero_launches_nothing():
    """mask = 0 returns before launching: the profiler sees the kernel of a mask-1 call and none for the mask-0 call."""
    words = torch.tensor([0, 7, 9], dtype=i32, device=dev)
    torch.cuda.synchronize()
    assert int(words[1].item()) == 7
    from torch.profiler import ProfilerActivity, profile

    def kernels(mask, ptr):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _lib.call("fz_p2p_wait", C.c_void_p(ptr), mask, ops._stream())
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if "p2p_wait_kernel" in e.name]
    assert kernels(0, words.data_ptr()) == []
    assert len(kernels(1, words.data_ptr() + 4)) == 1
    assert torch.equal(words.cpu(), torch.tensor([0, 0, 9], dtype=i32))


# ---------------------------------------------------------------------------------------------------------------- fz_gn_combine
class Combine:
    """One rank `me` of a simulated world: its inbox [world][n][2] uint2 (as int32 [world + 1, n, 2, 2], one guard slot), a scratch inbox
    per peer of the same shape (peer_inbox[r] = slot `me` of it), sums [n + 1] float2 and totals [n + 1] double2 (one guard pair each)
    and the epoch word between two guard words."""

    def __init__(self, world, me, NB, F_loc, G, epoch0=0):
        self.world, self.me, self.NB, self.F_loc, self.G = world, me, NB, F_loc, G
        self.n = n = NB * G
        self.inbox = torch.full((world + 1, n, 2, 2), SENT32, dtype=i32, device=dev)
        self.scratch = {r: torch.full((world + 1, n, 2, 2), SENT32, dtype=i32, device=dev) for r in range(world) if r != me}
        self.sums = torch.full((n + 1, 2), -7.25, dtype=torch.float32, device=dev)
        self.totals = torch.full((n + 1, 2), -9.5, dtype=torch.float64, device=dev)
        self.epoch = torch.tensor([s32(0x44000000), s32(epoch0), s32(0x44000002)], dtype=i32, device=dev)
        self.pi = (C.c_void_p * max(1, world))(*[self.scratch[r].data_ptr() + me * n * 16 if r != me else None for r in range(world)])

    def ep(self) -> int:
        """The epoch this use will carry: the device word + 1 (read after a synchronize)."""
        torch.cuda.synchronize()
        return (int(self.epoch[1].item()) + 1) & 0xFFFFFFFF

    def stage(self, seed):
        """Peer values and own sums for the next use, with per-image (sum, sumsq) magnitudes spread over 2^-12 .. 2^12."""
        g = torch.Generator().manual_seed(seed)
        v = torch.randn(self.world, self.NB, self.G, 2, generator=g)
        v = v * torch.pow(2.0, torch.randint(-12, 13, v.shape, generator=g).float())
        v[..., 1] = v[..., 1].abs()
        self.vals, self.own = v, v[self.me].clone()
        ep = self.ep()
        words = torch.stack([v.view(i32).view(self.world, self.n, 2), torch.full((self.world, self.n, 2), s32(ep), dtype=i32)], -1)
        for r in range(self.world):
            if r != self.me:
                self.inbox[r].copy_(words[r])
        self.sums[:self.n].copy_(self.own.view(self.n, 2))
        self.totals.fill_(-9.5)
        torch.cuda.synchronize()
        got = self.inbox.cpu()
        for r in range(self.world):
            if r != self.me:
                assert torch.equal(got[r], words[r]), f"inbox slot {r} not staged"
                assert torch.all(got[r][..., 1] == s32(ep)), "an inbox word the combine reads does not carry its epoch"
        assert torch.equal(self.sums[:self.n].cpu(), self.own.view(self.n, 2))
        self.staged, self.ep_now = got, ep

    def call(self, **over):
        a = dict(epoch=self.epoch.data_ptr() + 4, pi=self.pi, inbox=self.inbox.data_ptr(), sums=self.sums.data_ptr(),
                 totals=self.totals.data_ptr(), NB=self.NB, F_loc=self.F_loc, G=self.G, world=self.world, me=self.me)
        a.update(over)
        _lib.call("fz_gn_combine", C.c_void_p(a["epoch"]), a["pi"], C.c_void_p(a["inbox"]), C.c_void_p(a["sums"]), C.c_void_p(a["totals"]),
                  a["NB"], a["F_loc"], a["G"], a["world"], a["me"], ops._stream())

    def check(self, report, key):
        torch.cuda.synchronize()
        ep, n = self.ep_now, self.n
        assert torch.equal(self.epoch.cpu(), torch.tensor([s32(0x44000000), s32(ep), s32(0x44000002)], dtype=i32)), "epoch word not advanced by one"
        check_gn_combine(self.totals[:n].view(self.NB, self.G, 2), self.own, self.vals, self.me, self.F_loc, report, key)
        assert torch.equal(self.totals[n].cpu(), torch.tensor([-9.5, -9.5], dtype=torch.float64)), "totals written past n"
        assert torch.equal(self.sums[:n].cpu(), self.own.view(n, 2)) and torch.equal(self.sums[n].cpu(), torch.tensor([-7.25, -7.25])), \
            "the combine wrote its input sums"
        assert torch.equal(self.inbox.cpu(), self.staged), "the combine wrote its own inbox"
        sent = torch.stack([self.own.view(i32).view(n, 2), torch.full((n, 2), s32(ep), dtype=i32)], -1)
        for r, s in self.scratch.items():
            got = s.cpu()
            assert torch.equal(got[self.me], sent), f"words sent to peer {r} are not {{bits of the unmodified sums, epoch + 1}}"
            others = torch.cat([got[:self.me], got[self.me + 1:]])
            assert torch.all(others == SENT32), f"the combine wrote peer {r}'s inbox outside slot {self.me}"


# world, me, NB, F_loc, G, first epoch: n = NB G in {1024, 1023 (odd G = 11), 63 and 40 (< 64 threads), 5 (G = 1)}
COMBINE_CASES = [
    (1, 0, 16, 8, 3, 0),
    (2, 0, 32, 2, 32, 0),
    (2, 1, 32, 8, 32, 5),
    (3, 1, 9, 3, 7, 0),
    (3, 2, 5, 1, 1, 0xFFFFFFFE),  # the epoch wraps to 0 at the second call
    (8, 0, 4, 2, 32, 0),
    (8, 3, 8, 8, 5, 17),
    (8, 7, 6, 3, 32, 0),
    (32, 0, 2, 1, 32, 0),
    (32, 16, 93, 3, 11, 1000),
    (32, 31, 32, 8, 32, 0),
]


@pytest.mark.parametrize("world,me,NB,F_loc,G,epoch0", COMBINE_CASES, ids=lambda v: str(v))
def test_gn_combine(world, me, NB, F_loc, G, epoch0, report):
    c = Combine(world, me, NB, F_loc, G, epoch0)
    tag = f"w{world}_me{me}_NB{NB}_F{F_loc}_G{G}"
    for use in range(2):  # the same site twice: words at epoch + 1, then epoch + 2
        c.stage(seed=10 * world + use)
        c.call()
        c.check(report, f"{tag}_use{use}")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c.call()
    for rep in range(2):  # restaged before each replay: the captured launch reads the epoch from device memory
        c.stage(seed=10 * world + 5 + rep)
        g.replay()
        c.check(report, f"{tag}_graph{rep}")
    assert c.ep_now == (epoch0 + 4) & 0xFFFFFFFF


def test_gn_combine_refusals():
    c = Combine(4, 1, 4, 2, 8)
    c.stage(seed=3)
    bad_pi = (C.c_void_p * 4)(*list(c.pi))
    bad_pi[2] = None
    wide = (C.c_void_p * 33)(*(list(c.pi) + [c.scratch[0].data_ptr()] * 29))
    for what, over, msg in [("n1025", dict(NB=41, G=25, F_loc=1), "1025"), ("NB%F_loc", dict(NB=5), "bad args"),
                            ("world0", dict(world=0, me=0), "bad args"), ("world33", dict(world=33, pi=wide), "bad args"),
                            ("me-1", dict(me=-1), "bad args"), ("me=world", dict(me=4), "bad args"), ("null_peer", dict(pi=bad_pi), "null peer"),
                            ("null_totals", dict(totals=0), "bad args")]:
        with pytest.raises(RuntimeError, match=msg):
            c.call(**over)
        torch.cuda.synchronize()
        assert int(c.epoch[1].item()) == 0, f"{what}: a refused combine advanced the epoch"
        assert torch.equal(c.inbox.cpu(), c.staged), f"{what}: a refused combine wrote the inbox"
        assert torch.equal(c.sums[:c.n].cpu(), c.own.view(c.n, 2)), f"{what}: a refused combine wrote the sums"
        assert torch.all(c.totals == -9.5), f"{what}: a refused combine wrote the totals"
        assert all(torch.all(s == SENT32) for s in c.scratch.values()), f"{what}: a refused combine wrote a peer's inbox"
    c.call()
    c.check(None, "")


# ------------------------------------------------------------------------------------------- engine helpers on simulated ranks
class SimArena(p2p.Arena):
    """p2p.Arena over one CUDA slab per rank of the same device; site / tensor / peer_ptr / flag_ptr / _counter_block are the real ones."""

    def exchange(self, site, segs, sources, stream):
        p2p.Arena.exchange(self, site, segs, (), stream)  # push and raise the destinations' flags, wait for nothing
        self.barrier.wait()                                # every rank's push of this exchange is queued
        mask = self.wait_mask(sources)
        torch.cuda.synchronize()
        got = self.flag_words(site).cpu()
        want = torch.tensor([(mask >> i) & 1 for i in range(32)], dtype=i32)
        assert torch.equal(got, want), f"rank {self.rank}: flags {got.tolist()} raised, expected the sources {want.tolist()}"
        _lib.call("fz_p2p_wait", C.c_void_p(self.base + site.flag_offset), mask, stream)
        self.barrier.wait()                                # no rank pushes to a site before every rank has queued its wait

    def flag_words(self, site):
        return self._mem[site.flag_offset:site.flag_offset + 4 * p2p.FLAG_WORDS].view(i32)


def sim_arenas(world, data_bytes=8 << 20):
    slabs = [torch.zeros(p2p.FLAG_REGION + data_bytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    barrier = threading.Barrier(world, timeout=300)  # a rank that fails breaks the barrier (abort); the timeout only guards the host
    out = []
    for r in range(world):
        a = object.__new__(SimArena)
        a.rank, a.world, a.device, a.group, a.nbytes = r, world, torch.device(dev), None, slabs[r].numel()
        a.base, a.peer_base, a._mem = slabs[r].data_ptr(), [s.data_ptr() for s in slabs], slabs[r]
        a._cursor, a._n_sites, a.sites = p2p.FLAG_REGION, 0, {}
        a.counters = torch.zeros(4096, dtype=i32, device=dev)
        a._counter_cursor = 0
        a.barrier = barrier
        out.append(a)
    return out


def run_ranks(world, fn, groups=32, gn_uses=None, arenas=None):
    """fn(rank, engine) in one thread per rank on engines made with object.__new__; then every flag word and arrival counter must be 0
    (the epoch word of a GroupNorm site, flag word 31, must equal its number of uses, gn_uses[key])."""
    arenas = arenas or sim_arenas(world)
    out, err = [None] * world, []

    def work(r):
        try:
            e = object.__new__(UNetEngine)
            e.shard, e.dev, e.arena, e.groups, e._images_per_item = (r, world, None), torch.device(dev), arenas[r], groups, None
            out[r] = fn(r, e)
        except BaseException as ex:  # noqa: BLE001
            err.append(ex)
            arenas[0].barrier.abort()
    ts = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    if err:
        raise err[0]
    torch.cuda.synchronize()
    for a in arenas:
        assert torch.all(a.counters == 0), f"rank {a.rank}: an arrival counter is not back at 0"
        for key, site in a.sites.items():
            w = a.flag_words(site).cpu()
            if key[0] == "gn":
                assert int(w[31]) == gn_uses[key], f"rank {a.rank} site {key}: epoch {int(w[31])} after {gn_uses[key]} uses"
                w = w[:31]
            assert torch.all(w == 0), f"rank {a.rank} site {key}: flag words {w.tolist()} left raised"
    return out


@pytest.mark.parametrize("world,F", [(2, 4), (4, 2), (8, 1)])
def test_sim_halo(world, F):
    B, HW, Cc = 2, 8, 16
    y = rnd(B, world * F, HW, Cc, seed=1).half()

    def fn(r, e):
        return e._halo_ext(("halo_y", "layer"), y[:, r * F:(r + 1) * F].contiguous()).clone()
    for r, ext in enumerate(run_ranks(world, fn)):
        zero = torch.zeros(B, 1, HW, Cc, dtype=f16, device=dev)
        want = torch.cat([y[:, r * F - 1:r * F] if r > 0 else zero, y[:, r * F:(r + 1) * F],
                          y[:, (r + 1) * F:(r + 1) * F + 1] if r < world - 1 else zero], 1)
        assert torch.equal(ext, want), r


@pytest.mark.parametrize("world,F,index_list", [(2, 2, ["mid"]), (4, 2, ["mid", "first"]), (8, 1, ["last"]), (2, 3, [-1, "first"]), (4, 1, ["mid", 1])])
def test_sim_kv_exchange(world, F, index_list):
    B, S, heads, d = 2, 8, 2, 8
    Cc, Ft = heads * d, world * F
    K, V = rnd(B, Ft, S, Cc, seed=2).half(), rnd(B, Ft, S, Cc, seed=3).half()
    fis = sc_frame_indices(index_list, Ft)

    def fn(r, e):
        qk = torch.zeros(B * F * S, 2 * Cc, dtype=f16, device=dev)
        qk[:, Cc:] = K[:, r * F:(r + 1) * F].reshape(B * F * S, Cc)
        vt = V[:, r * F:(r + 1) * F].reshape(B * F, S, heads, d).permute(0, 2, 3, 1).contiguous()
        k_src, vt_src, n_src, src_index = e._kv_exchange("layer", qk, vt, index_list, B, F, S, Cc, heads, d)
        return k_src.clone(), vt_src.clone(), n_src, src_index
    for r, (k_src, vt_src, n_src, src_index) in enumerate(run_ranks(world, fn)):
        assert len(src_index) == len(index_list) and k_src.shape == (n_src * S, Cc) and vt_src.shape == (n_src, heads, d, S)
        for sl, fi in enumerate(fis):
            for b in range(B):
                for f in range(F):
                    row, g = src_index[sl][b * F + f], fi[r * F + f]
                    assert torch.equal(k_src[row * S:(row + 1) * S], K[b, g]), (r, sl, b, f)
                    assert torch.equal(vt_src[row], V[b, g].reshape(S, heads, d).permute(1, 2, 0)), (r, sl, b, f)


def temporal_plan(Fr, heads, d):
    """fz_temporal_attn_f16's kernel choice: the pixel-major kernel with hg heads per warp, or the generic one (None)."""
    if Fr not in (2, 4, 8) or d % 8 or d > 320:
        return None
    hg = max(1, min(heads, 320 // d))
    while heads % hg:
        hg -= 1
    return hg


@pytest.mark.parametrize("world,F,heads,d", [(2, 2, 2, 8), (4, 1, 2, 8), (8, 1, 2, 8), (2, 4, 8, 40), (4, 3, 8, 40)])
def test_sim_temporal_attn(world, F, heads, d, report):
    B, S = 2, 16
    Cc, Ft, scale = heads * d, world * F, d ** -0.5
    qkv = rnd(B, Ft, S, 3 * Cc, seed=4).half()
    whole = ops.temporal_attn(qkv.reshape(-1, 3 * Cc), B, Ft, S, heads, d, scale)

    def fn(r, e):
        mine = qkv[:, r * F:(r + 1) * F].reshape(B * F * S, 3 * Cc).contiguous()
        return e._temporal_attn_sharded("layer", mine, B, F, S, heads, d, scale).clone()
    got = torch.stack([o.view(B, F, S, Cc) for o in run_ranks(world, fn)], 1).reshape(B, Ft, S, Cc)
    t = qkv.double().view(B, Ft, S, 3, heads, d).permute(3, 0, 2, 4, 1, 5)  # [3, B, S, heads, F, d]
    p = softmax64(t[0] @ t[1].transpose(-1, -2) * f32(scale))
    check_attn(got.view(B, Ft, S, heads, d).permute(0, 2, 3, 1, 4), p, t[2], report, f"sim_temporal_w{world}_F{F}_h{heads}_d{d}")
    # the sharded call attends over S / world pixels of all Ft frames: the kernel plan depends on (Ft, heads, d) only, so it is the
    # whole-clip call's plan, and every pixel's output is computed by the same code in the same order
    report["plan"] = dict(hg=temporal_plan(Ft, heads, d), Ft=Ft)
    assert torch.equal(got, whole.view(B, Ft, S, Cc)), "sharded temporal attention differs from the whole-clip call"


@pytest.mark.parametrize("world,F", [(2, 2), (4, 1), (8, 1)])
def test_sim_conv_out_gather(world, F):
    B, H, W, co, R = 2, 4, 6, 4, 3
    Ft = world * F
    y = rnd(B, Ft, H * W, 16, seed=5).half()
    down, up = (rnd(R, co, 3, seed=6) * 0.5).contiguous(), (rnd(co, R, 3, seed=7) * 0.5).contiguous()
    whole = ops.out_temporal(y.reshape(-1, 16), B, co, Ft, H, W, down=down, up=up)

    def fn(r, e):
        e.w = {"conv_out.conv_temporal.down.weight": down, "conv_out.conv_temporal.down.weight#f32": down,
               "conv_out.conv_temporal.up.weight#f32": up}
        e.lora_skip = {}
        return e._finish(y[:, r * F:(r + 1) * F].reshape(B * F * H * W, 16).contiguous(), B, co, F, H, W)
    for r, got in enumerate(run_ranks(world, fn)):
        assert torch.equal(got, whole[:, :, r * F:(r + 1) * F]), r


def const_groups(shape, G, seed):
    """Every group constant over the whole clip: 0.3, 3 or -150 (the inputs of test_groupnorm_constant_groups)."""
    pick = torch.randint(0, 3, (G,), generator=torch.Generator().manual_seed(seed))
    vals = torch.tensor([0.3, 3.0, -150.0])[pick]
    return vals.repeat_interleave(shape[-1] // G).expand(shape).to(dev)


# world, F (local frames), inputs, C, HW.  Constant groups of 0.3 (fp16 1229 / 4096) over C / 32 * HW * F_total = 5 * 1023 * 12 (or
# 6) elements: every per-image sum is exact in fp32, the set total needs more than 24 bits (exact in fp64)
GN_JOINT_CASES = [(2, 4, "rnd", 320, 64), (4, 2, "rnd", 320, 64), (8, 1, "rnd", 320, 64), (4, 3, "rnd", 320, 1023),
                  (2, 4, "const", 320, 64), (8, 1, "const", 320, 64), (4, 2, "const", 2560, 64), (8, 1, "const", 2560, 64),
                  (4, 3, "const", 320, 1023), (2, 3, "const", 2560, 1023)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("world,F,inputs,C,HW", GN_JOINT_CASES, ids=lambda v: str(v))
def test_sim_gn_joint(world, F, inputs, C, HW, silu, report, monkeypatch):
    B, G = 2, 32
    Ft = world * F
    if inputs == "rnd":
        x = (rnd(B, Ft, HW, C, seed=8) * 1.5 + rnd(B, Ft, 1, C, seed=9)).half()
    else:
        x = const_groups((B, Ft, HW, C), G, 10).half()
    gamma, beta = 1 + 0.3 * rnd(C, seed=11), 0.2 * rnd(C, seed=12) * (0.05 if inputs == "const" else 1.0)
    xw = x.reshape(B * Ft, HW, C)
    tag = f"w{world}_F{F}_{inputs}_C{C}_HW{HW}_silu{int(silu)}"
    gn_check(ops.groupnorm(xw, gamma, beta, 1e-5, G, Ft, silu), xw, gamma, beta, 1e-5, G, Ft, silu, report, f"unsharded_{tag}")

    lock = threading.Lock()
    real_stats, real_call = ops.groupnorm_stats, _lib.call

    def stats(x3, groups):
        with lock:
            return real_stats(x3, groups).clone()
    arenas = sim_arenas(world)
    barrier = arenas[0].barrier  # the exchange barrier: run_ranks aborts it when a rank fails
    staged, uses = {}, {}

    def call(name, *args):
        if name != "fz_gn_combine":
            return real_call(name, *args)
        epoch_p, pi, inbox_p, sums_p, totals_p, NB, F_loc, G_, world_, me, st = args
        n, ar = NB * G_, arenas[me]
        off = epoch_p.value - ar.base
        torch.cuda.synchronize()
        epochs = {int(raw(a.base + off, 4, i32).item()) & 0xFFFFFFFF for a in arenas}
        assert len(epochs) == 1, f"the ranks' epochs disagree: {epochs}"
        ep = s32(epochs.pop() + 1)
        sums = raw(sums_p.value, n * 8, i32).view(n, 2)
        words = torch.stack([sums, torch.full_like(sums, ep)], -1)
        for r in range(world_):
            if r != me:
                raw(pi[r], n * 16, i32).view(n, 2, 2).copy_(words)
        torch.cuda.synchronize()
        for r in range(world_):
            if r != me:
                staged[pi[r]] = words.cpu()
                assert torch.equal(raw(pi[r], n * 16, i32).view(n, 2, 2).cpu(), staged[pi[r]]), f"rank {me}: words for rank {r} not staged"
        uses[(me, off)] = uses.get((me, off), 0) + 1
        barrier.wait()  # every rank has staged its words into every peer's inbox
        mine = raw(inbox_p.value, world_ * n * 16, i32).view(world_, n, 2, 2).cpu()
        assert all(torch.all(mine[r][..., 1] == ep) for r in range(world_) if r != me), f"rank {me}: an inbox word is not staged"
        real_call(name, *args)
        barrier.wait()  # every combine of this use is queued before any rank stages the next use of the site
    monkeypatch.setattr(ops, "groupnorm_stats", stats)
    monkeypatch.setattr(_lib, "call", call)

    def fn(r, e):
        mine = x[:, r * F:(r + 1) * F].reshape(B * F, HW, C).contiguous()
        a = e._gn_joint("norm", mine, gamma, beta, 1e-5, F, silu).clone()
        b = e._gn_joint("norm", mine, gamma, beta, 1e-5, F, silu).clone()  # the same site again, one epoch later
        return a, b
    out = run_ranks(world, fn, groups=G, gn_uses={("gn", "norm", B * F): 2}, arenas=arenas)
    for r, (a, b) in enumerate(out):
        assert torch.equal(a, b), f"rank {r}: the second use of the site differs"
    got = torch.stack([a.view(B, F, HW, C) for a, _ in out], 1).reshape(B * Ft, HW, C)
    gn_check(got, xw, gamma, beta, 1e-5, G, Ft, silu, report, f"gn_joint_{tag}")
    torch.cuda.synchronize()
    for ptr, words in staged.items():
        assert torch.equal(raw(ptr, words.numel() * 4, i32).view(words.shape).cpu(), words), "an inbox differs from the staged words"
    assert set(uses.values()) == {2}
