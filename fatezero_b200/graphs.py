"""CUDA-graph execution of the two DDIM loops: Python leaves the step.

An eager clip edit issues ~58 000 kernel launches through ctypes, each with up to six host-side `cuTensorMapEncodeTiled` calls and a
`torch.empty`: 756 ms of host time per 8-frame clip (tools/ablate.py), hidden behind 2.0 s of GPU work on one GPU but the floor of any
strong-scaling run.  A DDIM step is however a fixed launch sequence for a given (geometry, step index, controller structure): the only
per-step values (timestep, DDIM coefficients, cache slabs of that step, the step's row of the edit tables) are baked per STEP, so each
step is captured once into its own CUDA graph (kernel parameters — tensor maps included — live in the graph nodes, programmatic-
dependent-launch edges are preserved by stream capture) and replayed with one `cudaGraphLaunch`.

`StepGraphs` = an ordered list of per-step graphs sharing ONE private memory pool: activations are recycled inside the pool from step to
step, the objects that must survive (the map-cache slabs, running sums, stored latents, blend masks) stay referenced by the captured
controller and keep their addresses, so a replay refills exactly the tensors the Python-visible controller state points at.

Policy (pipeline.P2pDDIMSpatioTemporalPipeline.graph_mode):
  "auto"  a loop runs eagerly the first time a configuration is seen (which also loads every kernel it needs: lazily loaded modules
          cannot be loaded under capture) and is captured when the same configuration comes again — a one-off edit never pays for a capture;
  "off"   always eager (reference-like ownership: every controller owns freshly allocated maps).
A plan is keyed by everything that shapes the launch sequence; prompt-dependent CONTENT (text embeddings, the edit tables) lives in
static buffers that are refreshed before a replay.
"""
from __future__ import annotations

from typing import Callable, List

import torch

from . import _lib


class StepGraphs:
    def __init__(self, device: torch.device):
        self.device = device
        self.pool = torch.cuda.graph_pool_handle()
        self.stream = torch.cuda.Stream(device=device)
        self.graphs: List[torch.cuda.CUDAGraph] = []
        self.launches: List[int] = []   # kernels of libfatezero_b200 inside each graph (bench.py's gpu_launches accounting)
        self.calls: List[int] = []

    def capture(self, fn: Callable[[], None]):
        """Capture fn() (which must only enqueue work on the current stream) as the next step graph."""
        if not self.graphs:
            # The private pool cannot reuse blocks cached by the ordinary pool, e.g. a previous clip's freed map cache (36 GiB at
            # 512x512x8f): hand them back to the device so that the captured loop fits next to them on an 80 GB card.
            torch.cuda.empty_cache()
        g = torch.cuda.CUDAGraph()
        cur = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(cur)
        k0, c0 = _lib.kernel_launches, _lib.launch_count
        with torch.cuda.stream(self.stream):
            g.capture_begin(pool=self.pool, capture_error_mode="thread_local")
            try:
                fn()
            except BaseException:
                try:
                    g.capture_end()
                except Exception:  # noqa: BLE001
                    pass
                raise
            g.capture_end()
        cur.wait_stream(self.stream)
        self.graphs.append(g)
        self.launches.append(_lib.kernel_launches - k0)
        self.calls.append(_lib.launch_count - c0)
        # nothing ran during capture: take the counts back, replay() adds them when the kernels really run
        _lib.kernel_launches, _lib.launch_count = k0, c0

    def replay(self, i: int):
        self.graphs[i].replay()
        _lib.kernel_launches += self.launches[i]
        _lib.launch_count += self.calls[i]

    def __len__(self):
        return len(self.graphs)


class LoopPlan:
    """One captured DDIM loop: the step graphs plus the static buffers and the controller object they were captured with."""

    def __init__(self, device: torch.device):
        self.steps = StepGraphs(device)
        self.x = None            # fp32 latents, updated in place by the step kernels
        self.text = None         # static text-embedding buffer the captured forwards read
        self.controller = None   # the controller the graphs were captured with (owner of every slab the kernels write)
        self.outputs = []        # per-step output tensors inside the pool (inversion: the N latents)
        self.id = id(self)
