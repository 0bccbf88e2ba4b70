"""CUDA-graph capture of one energy+forces evaluation.

The step is a fixed sequence of ~50 kernel launches from Python/ctypes; at a few ms per step the
launch path matters, so (instead of a tracing compiler) the whole sequence is captured once into a
CUDA graph and replayed: positions are copied into a static buffer, outputs live in static buffers.
Valid as long as the neighbour list (edge_index / shifts / types / cell) is unchanged -- exactly
the interval between neighbour-list rebuilds in MD.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _lib
from . import data as D


class GraphedEnergyForces:
    def __init__(self, model: torch.nn.Module, data: D.Type, warmup: int = 3, stress: bool = False):
        inner = getattr(model, "model", model)  # ForceStressOutput(FusedAllegroEnergy) or the energy model itself
        if not hasattr(inner, "energy_and_forces"):
            raise TypeError("model has no fused energy_and_forces path")
        self.inner = inner
        self.data = dict(data)
        self.static_pos = data[D.POSITIONS_KEY].detach().clone()
        self.data[D.POSITIONS_KEY] = self.static_pos
        kw = {"stress": True} if stress else {}  # stress / virial captured into the graph only on request
        prof = _lib.PROF.enabled
        _lib.PROF.enabled = False
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(warmup):
                self.inner.energy_and_forces(self.data, **kw)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.PROF.launches
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = self.inner.energy_and_forces(self.data, **kw)
        self.launches_per_replay = _lib.PROF.launches - n0
        _lib.PROF.enabled = prof

    def __call__(self, pos: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Replay with new positions (device or pinned-host tensor); returns the static outputs."""
        if pos is not None:
            self.static_pos.copy_(pos, non_blocking=True)
        self.graph.replay()
        _lib.PROF.launches += self.launches_per_replay
        return self.out
