"""CUDA-graph replay of a denoiser's one-call forward, shared by the WaveNet and the ConvNext.

A sampler evaluates the denoiser on the same buffers over and over.  The first call on a set of buffers runs eagerly
(lazy initialisations happen there), the second is captured into a CUDA graph and replayed, and every later one is a
replay, which also removes the per-launch tensor-map encodes from the host path."""
from __future__ import annotations

import torch

from . import _native as N


def run_cached(graphs: dict, key, keep, launch, device, enabled: bool = True):
    """Run `launch()` (one native call that issues its launches on N.stream_ptr(device)) through the graph cache
    `graphs`.  `key` names everything the captured launches read or write (buffer pointers, shapes, weight pack);
    `keep` holds those tensors alive while the graph exists.  With `enabled` False, or while per-launch profiling is
    on, the call runs eagerly."""
    if not enabled or N.prof_is_on():
        launch()
        return
    ent = graphs.get(key)
    if ent is None:                      # first sight of these buffers: run eagerly (lazy inits happen here)
        if len(graphs) >= 4:
            graphs.clear()
        graphs[key] = {"graph": None, "keep": keep}
        launch()
        return
    if ent["graph"] is None:
        # capture on a side stream without torch.cuda.graph()'s device synchronise + empty_cache (the call sits in
        # the middle of a sampler loop); nothing inside allocates
        g = torch.cuda.CUDAGraph()
        cur = torch.cuda.current_stream(device)
        side = torch.cuda.Stream(device=device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            g.capture_begin()
            try:
                launch()
            finally:
                g.capture_end()
        cur.wait_stream(side)
        ent["graph"] = g
    ent["graph"].replay()
