"""A committee of independently trained models evaluated on one neighbour list: the committee mean of energies, forces
(and stress) and the spread of the members' predictions (DP-GEN's model deviation), for active learning and candidate
screening.

    committee = Committee([model_a, model_b, model_c])      # AllegroModel or FusedAllegroEnergy members
    out = committee.energy_and_forces(data)                 # or energy_and_forces_frames(batch)
    out["forces"], out["force_deviation"], out["max_force_deviation"]

Each member runs its own fused pass on the same ``data`` (the same prepared CSR or ``edge_index``); then a fixed handful
of kernels forms the statistics.  ``ab2_committee_moments`` takes the members' outputs of one field and gives the mean and
the population deviation of every element's G-vector (include/allegro_b200.h); ``ab2_frame_extrema`` reduces the per-atom
force deviation to its max / min / mean over each frame.  Both are fixed-order and fp64-accumulated: a frame's statistics
are bitwise reproducible and do not depend on the rest of the batch.  The committee is a drop-in model for
``AllegroCalculator`` and ``BatchedCalculator``: one list, one rebuild and one CUDA graph serve all members.

Written (in the positions' dtype; member outputs are cast to it first):
  total_energy [B,1], atomic_energy [N,1], forces [N,3] (+ stress, virial [B,3,3])   committee means
  committee_energy [K,B]                                                            each member's total energy
  energy_std [B,1], atomic_energy_std [N,1], virial_std [B,3,3]                     deviation over the members
  force_deviation [N]       sigma_F(a) = sqrt((1/K) sum_k |F_k,a - mean_a|^2)
  max_force_deviation / min_force_deviation / mean_force_deviation [B]            over each frame's atoms
(B = 1 for ``energy_and_forces``.)  ``edge_energy`` / ``edge_features`` belong to one member and are not written.
"""
from __future__ import annotations

from typing import Dict, List

import torch

from . import _lib
from . import data as D

MAX_MEMBERS = _lib.COMMITTEE_MAX_MEMBERS
# _lib launches the statistics add after the members' passes: moments of total_energy, atomic_energy and forces (one each)
# and frame_extrema (partial + combine); with stress, moments of stress and of virial
STAT_LAUNCHES = 5
STAT_LAUNCHES_STRESS = 2


def _device_of(module: torch.nn.Module):
    for t in list(module.parameters()) + list(module.buffers()):
        return t.device
    return None


class Committee(torch.nn.Module):
    # The statistics kernels (``_lib.committee_moments`` / ``frame_extrema``).  A restatement with the same signatures may
    # stand in for them on CPU tensors (tests/committee_spec.py).
    _kernels = _lib

    def __init__(self, members):
        super().__init__()
        members = list(members)
        if not members:
            raise ValueError("a committee needs at least one member")
        if len(members) > MAX_MEMBERS:
            raise ValueError(f"a committee takes at most {MAX_MEMBERS} members, got {len(members)}")
        inners = [getattr(m, "model", m) for m in members]
        for k, inner in enumerate(inners):
            if not (hasattr(inner, "energy_and_forces") and hasattr(inner, "energy_and_forces_frames")):
                raise TypeError(f"member {k} ({type(inner).__name__}) has no fused energy_and_forces path: members are "
                                "AllegroModel or FusedAllegroEnergy")
        names = [list(inner.type_names) for inner in inners]
        for k, nm in enumerate(names):
            if nm != names[0]:
                raise ValueError(f"member {k} has type_names {nm}, member 0 has {names[0]}: a committee needs one type map")
        devs = {str(d) for d in (_device_of(m) for m in members) if d is not None}
        if len(devs) > 1:
            raise ValueError(f"the members live on different devices ({sorted(devs)})")
        self.members = torch.nn.ModuleList(members)
        self.type_names = names[0]
        self.r_max = max(float(inner.r_max) for inner in inners)
        self._own: Dict[str, tuple] = {}

    # ---- members and their caches ------------------------------------------------------------------
    def _inners(self) -> List[torch.nn.Module]:
        return [getattr(m, "model", m) for m in self.members]

    @property
    def _caches(self) -> Dict[str, tuple]:
        """Every member's per-list cache entries and the committee's own (graph.GraphedEnergyForces holds them, so that a
        later call on one member cannot free tensors a captured graph reads)."""
        out = {"committee." + k: v for k, v in self._own.items()}
        for j, inner in enumerate(self._inners()):
            for k, v in getattr(inner, "_caches", {}).items():
                out[f"{j}.{k}"] = v
        return out

    def _cached(self, slot: str, srcs, extra, build):
        """``FusedAllegroEnergy._cached``: keyed on the identity and version of the source tensors and on ``extra``."""
        hit = self._own.get(slot)
        vers = tuple(t._version for t in srcs)
        if hit is not None and len(hit[0]) == len(srcs) and all(a is b for a, b in zip(hit[0], srcs)) and hit[1] == vers and hit[2] == extra:
            return hit[3]
        val = build()
        self._own[slot] = (tuple(srcs), vers, extra, val)
        return val

    # ---- evaluation ----------------------------------------------------------------------------------
    def _check(self, data: D.Type, atomic_virial: bool, heat_current: bool):
        if atomic_virial or heat_current:
            raise NotImplementedError("a committee returns no atomic_virial / heat_current")
        csr = data.get(D.CSR_KEY)
        if csr is None:
            return
        n = data[D.POSITIONS_KEY].shape[0]
        if csr.num_atoms < n:
            raise ValueError(f"the neighbour list has rows for {csr.num_atoms} of {n} atoms: a ghost-format list gives partial "
                             "forces, whose deviations mean nothing; give every atom a row")
        if csr.radius is not None and csr.radius < self.r_max:
            raise ValueError(f"the neighbour list was built at radius {csr.radius!r}, below the committee's r_max {self.r_max!r}: "
                             "it would truncate the members with the larger cutoff")

    def energy_and_forces(self, data: D.Type, stress: bool = False, atomic_virial: bool = False, heat_current: bool = False) -> D.Type:
        """One frame: every member's ``energy_and_forces(data, stress)``, then the committee statistics (module docstring)."""
        self._check(data, atomic_virial, heat_current)
        outs = [inner.energy_and_forces(data, stress=stress) for inner in self._inners()]
        pos = data[D.POSITIONS_KEY]
        n = pos.shape[0]
        frame_ptr = self._cached("ptr", (), (n, str(pos.device)), lambda: torch.tensor([0, n], dtype=torch.int32, device=pos.device))
        return self._statistics(data, outs, frame_ptr)

    def energy_and_forces_frames(self, data: D.Type, stress: bool = False, atomic_virial: bool = False, heat_current: bool = False) -> D.Type:
        """A batch of frames (``batch.collate``): every member's ``energy_and_forces_frames(data, stress)``, then the
        committee statistics of every frame (module docstring)."""
        self._check(data, atomic_virial, heat_current)
        outs = [inner.energy_and_forces_frames(data, stress=stress) for inner in self._inners()]
        batch, num = data[D.BATCH_KEY], data.get(D.NUM_NODES_KEY)
        srcs = (batch,) + ((num,) if num is not None else ())
        frame_ptr = self._cached("frames_ptr", srcs, (batch.shape[0],), lambda: self._frame_ptr(batch, num))
        return self._statistics(data, outs, frame_ptr)

    @staticmethod
    def _frame_ptr(batch: torch.Tensor, num) -> torch.Tensor:
        """frame_ptr [B+1] int32 (the members have already checked ``batch`` against ``num_atoms``)."""
        counts = num.reshape(-1).long() if num is not None else torch.bincount(batch.reshape(-1).long())
        fp = torch.zeros(counts.shape[0] + 1, dtype=torch.int32, device=batch.device)
        fp[1:] = torch.cumsum(counts.to(batch.device), 0).to(torch.int32)
        return fp

    def _statistics(self, data: D.Type, outs: List[D.Type], frame_ptr: torch.Tensor) -> D.Type:
        Kn = self._kernels
        dt = data[D.POSITIONS_KEY].dtype

        def field(key):
            return [o[key].to(dt).contiguous() for o in outs]

        out = dict(data)
        e = field(D.TOTAL_ENERGY_KEY)
        out[D.TOTAL_ENERGY_KEY], std = Kn.committee_moments(e, 1)
        out[D.ENERGY_STD_KEY] = std.view(-1, 1)
        out[D.COMMITTEE_ENERGY_KEY] = torch.stack([x.reshape(-1) for x in e])
        out[D.PER_ATOM_ENERGY_KEY], std = Kn.committee_moments(field(D.PER_ATOM_ENERGY_KEY), 1)
        out[D.ATOMIC_ENERGY_STD_KEY] = std.view(-1, 1)
        out[D.FORCE_KEY], sigma = Kn.committee_moments(field(D.FORCE_KEY), 3)
        out[D.FORCE_DEVIATION_KEY] = sigma
        ext = Kn.frame_extrema(sigma, frame_ptr)
        out[D.MAX_FORCE_DEVIATION_KEY], out[D.MIN_FORCE_DEVIATION_KEY], out[D.MEAN_FORCE_DEVIATION_KEY] = ext[:, 0], ext[:, 1], ext[:, 2]
        if all(D.STRESS_KEY in o for o in outs):
            # stress and virial each from the members' own, so that one member gives its own bits back
            out[D.STRESS_KEY], _ = Kn.committee_moments(field(D.STRESS_KEY), 1)
            out[D.VIRIAL_KEY], std = Kn.committee_moments(field(D.VIRIAL_KEY), 1)
            out[D.VIRIAL_STD_KEY] = std.view(-1, 3, 3)
        return out
