"""MD-side driver: positions in, energy / forces (/ stress) out, with a Verlet-skin neighbour list.

What an ASE calculator or LAMMPS' pair style does around the model (the callers of the hot path,
SURVEY.md section 8 rows f2/f3): keep a neighbour list built with ``r_max + skin``, rebuild it only when an
atom has moved more than ``skin / 2`` since the last build, and evaluate the model on the current
positions.  Between rebuilds the edge list is static, so the whole evaluation is replayed from one
CUDA graph (``allegro_b200.graph.GraphedEnergyForces``); a rebuild re-captures it.

Edges of the skin list that are currently longer than ``r_max`` cost time but contribute exactly
zero: the radial basis carries the polynomial cutoff (zero with zero derivative for r >= r_max,
nequip PolynomialCutoff) and every MLP on the path is bias-free, so such an edge has zero scalar
features, zero tensor features, zero environment weight and zero edge energy (checked in
tests/test_calculator.py against evaluations on exact r_max lists).

``model`` is anything with the reference's ``forward(data) -> data`` contract; CUDA-graph replay is used
when it exposes the fused ``energy_and_forces`` path (allegro_b200.model.AllegroModel).

The same argument holds pair type by pair type.  With ``prune_edges=True`` and a model built with
``per_edge_type_cutoff``, the list is searched at ``r_list = max(rmax_table) + skin`` and pruned to
``rmax_table[t_i, t_j] + skin`` (``data.prune_csr``), so an H-H or Li-Li pair beyond its own cutoff is never evaluated.
The rebuild rule (an atom moved more than ``skin / 2``) covers each pair with its own radius, so no kept-out pair can
come within its cutoff before the next rebuild.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import data as D


def prune_table(model, skin: float) -> Optional[torch.Tensor]:
    """``rmax_table + skin`` [T,T] fp64 on the CPU of a model built with per-edge-type cutoffs, else None."""
    inner = getattr(model, "model", model)
    norm = getattr(inner, "edge_norm", None)
    if norm is None or not getattr(norm, "per_type", False):
        return None
    return norm.rmax_table.detach().to(device="cpu", dtype=torch.float64) + float(skin)


class AllegroCalculator:
    def __init__(self, model, r_max: float, skin: float = 0.5, pbc=(True, True, True), use_graph: bool = True,
                 compute_stress: bool = False, check_every: int = 1, compute_atomic_virial: bool = False,
                 compute_heat_current: bool = False, prune_edges: bool = False):
        assert skin >= 0.0 and check_every >= 1
        self.model, self.r_max, self.skin = model, float(r_max), float(skin)
        # per-type list radii (prune_edges with a per_edge_type_cutoff model), else one radius r_max + skin
        self._cutoffs = prune_table(model, skin) if prune_edges else None
        self.r_list = float(self._cutoffs.max()) if self._cutoffs is not None else self.r_max + self.skin
        self.pbc = tuple(bool(p) for p in (pbc if not isinstance(pbc, bool) else (pbc,) * 3))
        self.compute_stress = bool(compute_stress)
        # per-atom virial / heat current: skin edges have zero gradient, so they add nothing to either
        self.compute_heat_current = bool(compute_heat_current)
        self.compute_atomic_virial = bool(compute_atomic_virial) or self.compute_heat_current
        inner = getattr(model, "model", model)
        if self.compute_atomic_virial and not hasattr(inner, "energy_and_forces"):
            raise NotImplementedError("atomic_virial / heat_current need the fused energy_and_forces path")
        self.use_graph = bool(use_graph) and hasattr(inner, "energy_and_forces")
        self.check_every = int(check_every)
        self.n_rebuilds = 0
        self.n_evaluations = 0
        self._data: Optional[D.Type] = None
        self._pos_ref: Optional[torch.Tensor] = None
        self._graphed = None
        self._since_check = 0

    # ---- neighbour-list management ---------------------------------------------------------
    def _needs_rebuild(self, pos, cell, atom_types) -> bool:
        if self._data is None or pos.shape != self._pos_ref.shape:
            return True
        old_cell = self._data.get(D.CELL_KEY)
        if (cell is None) != (old_cell is None) or (cell is not None and not torch.equal(cell.to(old_cell.dtype).view(3, 3), old_cell.view(3, 3))):
            return True
        if atom_types is not None and not torch.equal(atom_types.reshape(-1), self._data[D.ATOM_TYPE_KEY]):
            return True
        self._since_check += 1
        if self._since_check < self.check_every:
            return False
        self._since_check = 0
        moved = (pos - self._pos_ref).norm(dim=-1).max()
        return bool(moved > 0.5 * self.skin)  # one device->host sync per check

    def _rebuild(self, pos, cell, atom_types):
        if atom_types is None:
            if self._data is None:
                raise ValueError("atom_types are needed for the first evaluation")
            atom_types = self._data[D.ATOM_TYPE_KEY]
        if self.compute_stress and cell is not None:
            if not D.is_regular_cell(cell):
                raise ValueError("compute_stress=True needs a non-singular cell: stress is the virial over the cell volume")
        data = {D.POSITIONS_KEY: pos.clone(), D.ATOM_TYPE_KEY: atom_types.reshape(-1).clone()}
        inner = getattr(self.model, "model", self.model)
        if hasattr(inner, "energy_and_forces") and D.csr_supported(pos, self.r_list, cell, self.pbc):
            # CUDA cell list straight into the kernels' CSR (no int64 COO list, no sort by centre); any cell, or none
            prune = {} if self._cutoffs is None else dict(types=data[D.ATOM_TYPE_KEY], cutoffs=self._cutoffs)
            csr, shift_vec = D.neighbor_csr(pos, self.r_list, cell, self.pbc, **prune)
            data[D.CSR_KEY], data[D.EDGE_SHIFT_VEC_KEY] = csr, shift_vec
            if cell is not None:
                data[D.CELL_KEY] = cell.view(3, 3).clone()
            self._n_edges = csr.num_edges
        elif self._cutoffs is not None and hasattr(inner, "energy_and_forces"):
            # the pair search, then the same pruning on its CSR form
            ei, shift = D.neighbor_list(pos, self.r_list, cell, self.pbc)
            n = pos.shape[0]
            shift_vec = shift @ cell.view(3, 3).to(pos.dtype) if cell is not None else torch.zeros(ei.shape[1], 3, dtype=pos.dtype, device=pos.device)
            csr, shift_vec = D.prune_csr(D.build_csr(ei, n), shift_vec.contiguous(), pos, data[D.ATOM_TYPE_KEY], self._cutoffs, self.r_list)
            data[D.CSR_KEY], data[D.EDGE_SHIFT_VEC_KEY] = csr, shift_vec
            if cell is not None:
                data[D.CELL_KEY] = cell.view(3, 3).clone()
            self._n_edges = csr.num_edges
        else:
            ei, shift = D.neighbor_list(pos, self.r_list, cell, self.pbc)
            data[D.EDGE_INDEX_KEY] = ei
            self._n_edges = int(ei.shape[1])
            if cell is not None:
                data[D.CELL_KEY] = cell.view(3, 3).clone()
                data[D.EDGE_CELL_SHIFT_KEY] = shift
        self._data, self._pos_ref = data, pos.clone()
        self._graphed = None
        self._since_check = 0
        self.n_rebuilds += 1
        if self.use_graph:
            from .graph import GraphedEnergyForces

            self._graphed = GraphedEnergyForces(self.model, data, stress=self.compute_stress, **self._extra_kw())

    def _extra_kw(self):
        if not self.compute_atomic_virial:
            return {}
        return dict(atomic_virial=True, heat_current=self.compute_heat_current)

    # ---- evaluation ----------------------------------------------------------------------------
    def compute(self, pos: torch.Tensor, cell: Optional[torch.Tensor] = None, atom_types: Optional[torch.Tensor] = None,
                velocities: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """-> {"energy" [1,1], "forces" [N,3], "atomic_energy" [N,1]} (+ "stress", "virial" [1,3,3] if asked for and a cell
        is given: with ``cell=None`` no stress is returned, a singular cell (``data.is_regular_cell``) raises ValueError, and
        any other cell, however thin an open axis, divides the virial by its own volume;
        "atomic_virial" [N,3,3] with compute_atomic_virial; "heat_current" [1,3] with compute_heat_current, which needs
        ``velocities`` [N,3]).  The returned tensors are the model's output buffers: with graph replay they are
        overwritten by the next call."""
        if self.compute_heat_current and (velocities is None or tuple(velocities.shape) != (pos.shape[0], 3)):
            raise ValueError(f"compute_heat_current needs velocities [{pos.shape[0]},3]")
        if self._needs_rebuild(pos, cell, atom_types):
            self._rebuild(pos, cell, atom_types)
        if self._graphed is not None:
            out = self._graphed(pos, velocities if self.compute_heat_current else None)
        else:
            d = dict(self._data)
            d[D.POSITIONS_KEY] = pos
            if self.compute_heat_current:
                d[D.VELOCITY_KEY] = velocities
            inner = getattr(self.model, "model", self.model)
            if hasattr(inner, "energy_and_forces"):
                out = inner.energy_and_forces(d, stress=self.compute_stress, **self._extra_kw())
            else:
                out = self.model(d)
        self.n_evaluations += 1
        res = {"energy": out[D.TOTAL_ENERGY_KEY], "forces": out[D.FORCE_KEY], "atomic_energy": out[D.PER_ATOM_ENERGY_KEY]}
        if self.compute_stress and D.STRESS_KEY in out:
            res["stress"], res["virial"] = out[D.STRESS_KEY], out[D.VIRIAL_KEY]
        if self.compute_atomic_virial:
            res["atomic_virial"] = out[D.ATOMIC_VIRIAL_KEY]
        if self.compute_heat_current:
            res["heat_current"] = out[D.HEAT_CURRENT_KEY]
        return res

    @property
    def num_edges(self) -> int:
        return 0 if self._data is None else int(self._n_edges)
