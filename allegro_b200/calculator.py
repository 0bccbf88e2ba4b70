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

import math
from typing import Dict, List, Optional

import torch

from . import _lib
from . import data as D


def prune_table(model, skin: float) -> Optional[torch.Tensor]:
    """``rmax_table + skin`` [T,T] fp64 on the CPU of a model built with per-edge-type cutoffs, else None.  For a
    ``committee.Committee``, the elementwise max over its members, a member without per-edge-type cutoffs counting as
    ``r_max + skin`` everywhere; None when no member has per-edge-type cutoffs."""
    from .committee import Committee

    inner = getattr(model, "model", model)
    if isinstance(inner, Committee):
        tables = [prune_table(m, skin) for m in inner.members]
        if all(t is None for t in tables):
            return None
        T = len(inner.type_names)
        full = [t if t is not None else torch.full((T, T), float(getattr(m, "model", m).r_max) + float(skin), dtype=torch.float64)
                for m, t in zip(inner.members, tables)]
        return torch.stack(full).amax(dim=0)
    norm = getattr(inner, "edge_norm", None)
    if norm is None or not getattr(norm, "per_type", False):
        return None
    return norm.rmax_table.detach().to(device="cpu", dtype=torch.float64) + float(skin)


def _committee_keys(out: D.Type, res: Dict[str, torch.Tensor]):
    """The statistics of a ``committee.Committee`` model (data.COMMITTEE_KEYS), where the model wrote them."""
    for k in D.COMMITTEE_KEYS:
        if k in out:
            res[k] = out[k]


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
        ``velocities`` [N,3]; with a ``committee.Committee`` as the model, also its statistics, data.COMMITTEE_KEYS).  The
        returned tensors are the model's output buffers: with graph replay they are overwritten by the next call."""
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
        _committee_keys(out, res)
        return res

    @property
    def num_edges(self) -> int:
        return 0 if self._data is None else int(self._n_edges)


# Capacity of a frame's edge slot: its edge count at a full build times SLOT_HEADROOM, plus SLOT_MIN_EDGES (so that a
# frame whose atoms have no neighbour yet still has room).  A frame that outgrows its slot makes the calculator rebuild
# every slot and capture its graph again, once; the headroom makes that rare in NVE / NVT runs of solids and liquids.
SLOT_HEADROOM = 1.25
SLOT_MIN_EDGES = 16
# Launches of one in-graph rebuild: check, count, place, fill, transpose (nlist_slots.cu).
SLOT_REBUILD_LAUNCHES = 5


class BatchedCalculator:
    """Molecular dynamics of a batch of small frames from one CUDA graph: energies, forces (and stress) of every frame per
    replay, each frame keeping its own Verlet list at ``r_list = r_max + skin`` and rebuilding it on the device, inside
    the replay, when one of its atoms has moved more than ``skin / 2`` since its last build (the rule of
    ``AllegroCalculator``).

    The batch's list has a fixed layout (include/allegro_b200.h, ab2_slots_*): frame b owns the edges
    [slot_ptr[b], slot_ptr[b+1]), its rows hold their real edges in the order of ``data.neighbor_csr_frames`` followed by
    padding self-edges 2 r_list long, which contribute exactly zero (the argument of the module docstring: x >= 1 zeroes
    the radial basis and every MLP is bias-free).  So the number of edges never changes and one captured graph serves
    every step.  A frame whose list outgrows its slot is never evaluated on a stale list: after each replay the host reads
    the overflow count, and if it is not zero the step is discarded, every slot is re-sized from a full build at the
    current positions, the graph is captured again and the step recomputed.

    ``frames``: single-frame dicts as ``batch.collate`` takes them (``pos`` on the device, ``atom_types``, optional
    ``cell`` / ``pbc``), at most ``data.FRAMES_MAX_ATOMS`` atoms each; cells and types are fixed for the calculator's
    lifetime (NVE / NVT).  ``compute(pos)`` takes the positions of every frame back to back."""

    # The rebuild kernels (``_lib.slots_*``).  A restatement with the same signatures may stand in for them on CPU tensors
    # (``_device = False``: no CUDA check, no graph).
    _kernels = _lib
    _device = True

    def __init__(self, model, frames, r_max: float, skin: float = 0.5, compute_stress: bool = False):
        from .batch import _pbc_of

        if not (float(skin) >= 0.0):
            raise ValueError(f"skin must be >= 0, got {skin}")
        if not (float(r_max) > 0.0):
            raise ValueError(f"r_max must be > 0, got {r_max}")
        self.model, self.r_max, self.skin = model, float(r_max), float(skin)
        self.r_list = self.r_max + self.skin
        self.compute_stress = bool(compute_stress)
        self._inner = getattr(model, "model", model)
        if not hasattr(self._inner, "energy_and_forces_frames"):
            raise TypeError("BatchedCalculator needs a model with the fused energy_and_forces_frames path")
        frames = list(frames)
        if not frames:
            raise ValueError("BatchedCalculator needs at least one frame")
        pos = [f[D.POSITIONS_KEY] for f in frames]
        dtype, dev = pos[0].dtype, pos[0].device
        for b, p in enumerate(pos):
            if not isinstance(p, torch.Tensor) or p.dim() != 2 or p.shape[1] != 3:
                raise ValueError(f"frame {b}: pos must be [n,3]")
            if p.dtype != dtype or p.device != dev:
                raise ValueError(f"frame {b}: every frame's pos must have one dtype and device ({dtype}, {dev})")
            if D.ATOM_TYPE_KEY not in frames[b] or frames[b][D.ATOM_TYPE_KEY].numel() != p.shape[0]:
                raise ValueError(f"frame {b}: atom_types needs one entry per atom")
        if dtype not in (torch.float32, torch.float64):
            raise ValueError(f"positions must be fp32 or fp64, got {dtype}")
        if self._device and not pos[0].is_cuda:
            raise ValueError("BatchedCalculator runs on the GPU: the frames' positions must be CUDA tensors")
        sizes = [int(p.shape[0]) for p in pos]
        if max(sizes) > D.FRAMES_MAX_ATOMS:
            raise ValueError(f"BatchedCalculator takes frames of at most {D.FRAMES_MAX_ATOMS} atoms (got {max(sizes)}); "
                             "larger systems belong to AllegroCalculator")
        if sum(sizes) == 0:
            raise ValueError("BatchedCalculator needs at least one atom")
        B, n = len(frames), sum(sizes)
        pbc = torch.stack([_pbc_of(f) for f in frames])
        with_cell = any(D.CELL_KEY in f for f in frames)
        cell = (torch.stack([f[D.CELL_KEY].reshape(3, 3).to(device=dev, dtype=dtype) if D.CELL_KEY in f
                             else torch.zeros(3, 3, dtype=dtype, device=dev) for f in frames]) if with_cell else None)
        # every refusal of the frames search, before any launch: bad cells, too many images
        rows, nimg = D.frames_geometry(cell, pbc, self.r_list, dtype)
        if self.compute_stress and (cell is None or not bool(D.regular_cells(cell).all())):
            raise ValueError("compute_stress=True needs a non-singular cell on every frame (data.is_regular_cell): stress is "
                             "the virial over the cell volume")
        self.dtype, self.device, self.num_frames, self.num_atoms = dtype, dev, B, n
        self.sizes = sizes
        self._max_atoms = max(sizes)
        fp = [0]
        for s in sizes:
            fp.append(fp[-1] + s)
        self._fp_host = fp
        i32 = dict(dtype=torch.int32, device=dev)
        self.frame_ptr = torch.tensor(fp, **i32)
        # the cell inverse as data.neighbor_csr_frames forms it (fp64, on the device), so the rows are those of that search
        rows = rows.to(dev)
        periodic = pbc.any(dim=1).view(B, 1, 1).to(dev)
        eye = torch.eye(3, dtype=torch.float64, device=dev).expand(B, 3, 3)
        inv = torch.where(periodic, torch.linalg.inv(torch.where(periodic, rows, eye)), torch.zeros_like(rows))
        self._geom = (self.frame_ptr, rows.to(device=dev, dtype=dtype).contiguous(), inv.to(device=dev, dtype=dtype).contiguous(),
                      pbc.to(**i32).contiguous(), nimg.to(**i32).contiguous())
        self.pad = 2.0 * self.r_list  # |shift| of a padding edge: beyond every cutoff
        self._pos = torch.cat(pos, 0).detach().to(dtype).contiguous().clone()
        self._pos_ref = torch.empty_like(self._pos)
        self._flag = torch.zeros(B, **i32)
        self._counts = torch.zeros(n, **i32)
        self._overflow = torch.zeros(1, **i32)
        self._rebuilds = torch.zeros(B, **i32)
        types = torch.cat([f[D.ATOM_TYPE_KEY].reshape(-1).to(dev) for f in frames], 0)
        self._base = {
            D.ATOM_TYPE_KEY: types,
            D.BATCH_KEY: torch.repeat_interleave(torch.arange(B, device=dev), torch.tensor(sizes, device=dev)),
            D.NUM_NODES_KEY: torch.tensor(sizes, dtype=torch.long, device=dev),
        }
        if cell is not None:
            self._base[D.CELL_KEY], self._base[D.PBC_KEY] = cell, pbc.to(dev)
        self.n_captures = 0
        self.n_overflows = 0
        self.n_evaluations = 0
        self._graphed = None
        self._full_build()

    # ---- the list ------------------------------------------------------------------------------
    def _rebuild_launches(self, data: D.Type):
        """One in-graph rebuild of the flagged frames' slots at the positions of ``data``."""
        K, pos = self._kernels, data[D.POSITIONS_KEY]
        fp, cell, inv, pbc, nimg = self._geom
        csr = data[D.CSR_KEY]
        col_ptr, col_perm = csr.transposed(self.num_atoms)
        K.slots_check(pos, self._pos_ref, fp, 0.5 * self.skin, self._flag)
        K.slots_count(pos, fp, cell, inv, pbc, nimg, self.r_list, self._flag, self._counts)
        K.slots_place(fp, self.slot_ptr, self._counts, self._flag, csr.row_ptr, self._overflow, self._rebuilds)
        K.slots_fill(pos, fp, cell, inv, pbc, nimg, self.r_list, self._flag, csr.row_ptr, self.pad, csr.ctr, csr.nbr,
                     data[D.EDGE_SHIFT_VEC_KEY], self._pos_ref)
        K.slots_transpose(fp, self.slot_ptr, csr.nbr, self._flag, col_ptr, col_perm, self._max_atoms)

    def _full_build(self):
        """Every frame rebuilt at the current positions into slots sized from its edge count now; then (re)capture."""
        K, pos, dev = self._kernels, self._pos, self.device
        fp, cell, inv, pbc, nimg = self._geom
        B, n = self.num_frames, self.num_atoms
        self._flag.fill_(1)
        K.slots_count(pos, fp, cell, inv, pbc, nimg, self.r_list, self._flag, self._counts)
        frame_of = self._base[D.BATCH_KEY]
        count = torch.zeros(B, dtype=torch.int64, device=dev).index_add_(0, frame_of, self._counts.long()).cpu().tolist()  # one read
        cap = [int(math.ceil(SLOT_HEADROOM * c)) + SLOT_MIN_EDGES if s > 0 else 0 for c, s in zip(count, self.sizes)]
        slot = [0]
        for c in cap:
            slot.append(slot[-1] + c)
        E = slot[-1]
        if E >= 2**31 - 1:
            raise ValueError(f"the batch's list needs {E} edges; the kernels index at most 2^31 - 2: use fewer or smaller frames")
        i32 = dict(dtype=torch.int32, device=dev)
        self.slot_ptr = torch.tensor(slot, **i32)
        self.capacity = cap
        row_ptr = torch.zeros(n + 1, **i32)
        row_ptr[n] = E
        col_ptr = torch.zeros(n + 1, **i32)
        col_ptr[n] = E
        ctr, nbr, col_perm = torch.zeros(E, **i32), torch.zeros(E, **i32), torch.zeros(E, **i32)
        shift = torch.zeros(E, 3, dtype=self.dtype, device=dev)
        csr = D.EdgeCSR(n, ctr, nbr, row_ptr, None, max(cap), self.r_list)  # max_degree: an upper bound, a row never outgrows its slot
        csr._transposed = (n, col_ptr, col_perm)
        self._overflow.zero_()
        K.slots_place(fp, self.slot_ptr, self._counts, self._flag, row_ptr, self._overflow, self._rebuilds)
        K.slots_fill(pos, fp, cell, inv, pbc, nimg, self.r_list, self._flag, row_ptr, self.pad, ctr, nbr, shift, self._pos_ref)
        K.slots_transpose(fp, self.slot_ptr, nbr, self._flag, col_ptr, col_perm, self._max_atoms)
        data = dict(self._base)
        data[D.POSITIONS_KEY] = self._pos
        data[D.CSR_KEY], data[D.EDGE_SHIFT_VEC_KEY] = csr, shift
        self._data = data
        self._graphed = None
        if self._device:
            from .graph import GraphedEnergyForces

            self._graphed = GraphedEnergyForces(self.model, data, stress=self.compute_stress, frames=True, before=self._rebuild_launches)
            self._data = self._graphed.data  # the graph's static positions are the ones the rebuild reads
            self.n_captures += 1

    def _step(self) -> D.Type:
        if self._graphed is not None:
            return self._graphed()
        self._rebuild_launches(self._data)
        return self._inner.energy_and_forces_frames(self._data, stress=self.compute_stress)

    # ---- evaluation ----------------------------------------------------------------------------
    def compute(self, pos: torch.Tensor) -> Dict[str, torch.Tensor]:
        """-> {"energy" [B,1], "forces" [N,3], "atomic_energy" [N,1]} (+ "stress", "virial" [B,3,3] with compute_stress)
        for the positions ``pos`` [N,3] of every frame, back to back in the frames' order (with a ``committee.Committee``
        as the model, also its statistics, data.COMMITTEE_KEYS).  The returned tensors are the
        graph's output buffers: the next call overwrites them.  Costs one device-to-host read (the overflow count)."""
        if not isinstance(pos, torch.Tensor) or tuple(pos.shape) != (self.num_atoms, 3):
            raise ValueError(f"pos must be [{self.num_atoms},3] (the atoms of every frame back to back), got "
                             f"{tuple(pos.shape) if isinstance(pos, torch.Tensor) else type(pos).__name__}")
        if pos.dtype != self.dtype or pos.device != self.device:
            raise ValueError(f"pos must be {self.dtype} on {self.device} (the frames' dtype and device), got {pos.dtype} on {pos.device}")
        self._data[D.POSITIONS_KEY].copy_(pos, non_blocking=True)
        out = self._step()
        if int(self._overflow[0]) != 0:
            # a frame outgrew its slot: its rows are the old ones, so nothing of this step is kept
            self.n_overflows += 1
            self._pos = self._data[D.POSITIONS_KEY]
            self._full_build()
            out = self._step()
        self.n_evaluations += 1
        res = {"energy": out[D.TOTAL_ENERGY_KEY], "forces": out[D.FORCE_KEY], "atomic_energy": out[D.PER_ATOM_ENERGY_KEY]}
        if self.compute_stress:
            res["stress"], res["virial"] = out[D.STRESS_KEY], out[D.VIRIAL_KEY]
        _committee_keys(out, res)
        return res

    # ---- state, for tests and timing -------------------------------------------------------
    @property
    def num_edges(self) -> int:
        """Edges of the batch's list, padding included (fixed between full builds)."""
        return int(self.slot_ptr[-1])

    @property
    def csr(self) -> D.EdgeCSR:
        return self._data[D.CSR_KEY]

    @property
    def shift(self) -> torch.Tensor:
        return self._data[D.EDGE_SHIFT_VEC_KEY]

    def frame_rebuilds(self) -> List[int]:
        """Builds of every frame's list so far (the first build and every full build included)."""
        return self._rebuilds.cpu().tolist()

    def real_edges(self) -> int:
        """Edges of the list that are not padding (one device-to-host read)."""
        csr, sh = self.csr, self.shift
        pad = (csr.nbr == csr.ctr) & (sh[:, 0] == torch.tensor(self.pad, dtype=sh.dtype)) & (sh[:, 1] == 0) & (sh[:, 2] == 0)
        return int(csr.nbr.shape[0] - int(pad.sum()))
