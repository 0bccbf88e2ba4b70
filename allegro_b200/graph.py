"""CUDA-graph capture of one energy+forces evaluation.

The step is a fixed sequence of ~50 kernel launches from Python/ctypes; at a few ms per step the
launch path matters, so (instead of a tracing compiler) the whole sequence is captured once into a
CUDA graph and replayed: positions are copied into a static buffer, outputs live in static buffers.
Valid as long as the neighbour list (edge_index / shifts / types / cell) is unchanged -- exactly
the interval between neighbour-list rebuilds in MD.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch

from . import _lib
from . import data as D


class GraphedEnergyForces:
    def __init__(self, model: torch.nn.Module, data: D.Type, warmup: int = 3, stress: bool = False, atomic_virial: bool = False,
                 heat_current: bool = False, frames: bool = False, before: Optional[Callable[[D.Type], None]] = None):
        """``frames=True``: the evaluation is ``energy_and_forces_frames`` (a batch of frames) instead of ``energy_and_forces``.
        ``before(data)``: launches captured ahead of the evaluation on every replay, given the graph's input dict (its static
        positions), e.g. the in-graph neighbour-list rebuild of calculator.BatchedCalculator."""
        inner = getattr(model, "model", model)  # ForceStressOutput(FusedAllegroEnergy) or the energy model itself
        entry = "energy_and_forces_frames" if frames else "energy_and_forces"
        if not hasattr(inner, entry):
            raise TypeError(f"model has no fused {entry} path")
        self.inner = inner
        self.data = dict(data)
        self.static_pos = data[D.POSITIONS_KEY].detach().clone()
        self.data[D.POSITIONS_KEY] = self.static_pos
        # with the heat current the velocities are an input of the graph as well: a static buffer, like the positions
        self.static_vel = None
        if heat_current:
            v = data.get(D.VELOCITY_KEY)
            self.static_vel = (v.detach().clone() if v is not None
                               else torch.zeros(self.static_pos.shape[0], 3, dtype=self.static_pos.dtype, device=self.static_pos.device))
            self.data[D.VELOCITY_KEY] = self.static_vel
        kw = {"stress": True} if stress else {}  # stress / virial captured into the graph only on request
        if atomic_virial or heat_current:
            kw.update(atomic_virial=bool(atomic_virial), heat_current=bool(heat_current))
        evaluate = getattr(inner, entry)

        def step():
            if before is not None:
                before(self.data)
            return evaluate(self.data, **kw)

        prof = _lib.PROF.enabled
        _lib.PROF.enabled = False
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(warmup):
                step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = _lib.PROF.launches
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = step()
        self.launches_per_replay = _lib.PROF.launches - n0
        # the graph reads the per-list tensors the model derived and cached (types, frame_ptr, volumes, ...) by address; the
        # model keeps one entry per kind, so another call on the same model would free them under the graph: hold them
        self._held = tuple(getattr(inner, "_caches", {}).values())
        _lib.PROF.enabled = prof

    def __call__(self, pos: Optional[torch.Tensor] = None, vel: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Replay with new positions (and, with the heat current, velocities; device or pinned-host tensors); returns the
        static outputs."""
        if pos is not None:
            self.static_pos.copy_(pos, non_blocking=True)
        if vel is not None:
            if self.static_vel is None:
                raise ValueError("velocities are only an input of a graph captured with heat_current=True")
            self.static_vel.copy_(vel, non_blocking=True)
        self.graph.replay()
        _lib.PROF.launches += self.launches_per_replay
        return self.out
