"""Batches of frames: nequip's batched data layout for ``FusedAllegroEnergy.energy_and_forces_frames``.

    batch = collate(frames, r_max)          # list of single-frame dicts -> one batched dict
    out = model.energy_and_forces_frames(batch, stress=True)
    per_frame = split(out)                  # -> list of single-frame dicts

A batched dict holds the frames' atoms back to back: ``pos`` [N,3], ``atom_types`` [N], ``batch`` [N] (frame of every
atom, non-decreasing), ``num_atoms`` [B], ``cell`` [B,3,3] and ``pbc`` [B,3] when any frame has a cell, and one neighbour
list over global atom indices: either ``edge_index`` (+ ``edge_cell_shift``), or the prepared ``edge_csr`` +
``edge_shift_vec`` built on the device by ``data.neighbor_csr_frames``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import data as D

_PER_ATOM = (D.POSITIONS_KEY, D.ATOM_TYPE_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.VELOCITY_KEY, D.ATOMIC_VIRIAL_KEY)
_PER_EDGE = (D.EDGE_CELL_SHIFT_KEY, D.EDGE_ENERGY_KEY, D.EDGE_FEATURES_KEY)
_PER_FRAME = (D.TOTAL_ENERGY_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.CELL_KEY, D.PBC_KEY, D.HEAT_CURRENT_KEY)
_PER_FRAME_ROWS = (D.TOTAL_ENERGY_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.HEAT_CURRENT_KEY)  # kept as [1, ...] per frame


def _pbc_of(frame: D.Type) -> torch.Tensor:
    p = frame.get(D.PBC_KEY)
    if p is None:
        return torch.full((3,), D.CELL_KEY in frame, dtype=torch.bool)
    p = torch.as_tensor(p, dtype=torch.bool).reshape(-1).cpu()
    return p.expand(3).clone() if p.numel() == 1 else p


def collate(frames: Sequence[D.Type], r_max: Optional[float] = None) -> D.Type:
    """Single-frame dicts (``pos``, ``atom_types``, optional ``cell`` / ``pbc``, optional ``edge_index`` /
    ``edge_cell_shift``, optional ``velocities``, on every frame or none) -> one batched dict.  When every frame has ``edge_index`` the lists are offset and concatenated;
    when none has, the list is built on the device with ``data.neighbor_csr_frames`` (needs ``r_max``; frames of at most
    ``data.FRAMES_MAX_ATOMS`` atoms).  A mix of the two is rejected.  A frame without a cell gets a zero cell and no
    periodic axis."""
    if len(frames) == 0:
        raise ValueError("collate needs at least one frame")
    has_ei = [D.EDGE_INDEX_KEY in f for f in frames]
    if any(has_ei) and not all(has_ei):
        raise ValueError("collate: some frames carry edge_index and others do not; give every frame a neighbour list or none")
    pos = [f[D.POSITIONS_KEY] for f in frames]
    dev, dtype = pos[0].device, pos[0].dtype
    sizes = [int(p.shape[0]) for p in pos]
    B = len(frames)
    out: D.Type = {
        D.POSITIONS_KEY: torch.cat(pos, 0).to(dtype).contiguous(),
        D.ATOM_TYPE_KEY: torch.cat([f[D.ATOM_TYPE_KEY].reshape(-1) for f in frames], 0),
        D.BATCH_KEY: torch.repeat_interleave(torch.arange(B, device=dev), torch.tensor(sizes, device=dev)),
        D.NUM_NODES_KEY: torch.tensor(sizes, dtype=torch.long, device=dev),
    }
    has_vel = [D.VELOCITY_KEY in f for f in frames]
    if any(has_vel) and not all(has_vel):
        raise ValueError("collate: some frames carry velocities and others do not")
    if all(has_vel):
        out[D.VELOCITY_KEY] = torch.cat([f[D.VELOCITY_KEY].reshape(-1, 3) for f in frames], 0)
    with_cell = any(D.CELL_KEY in f for f in frames)
    pbc = torch.stack([_pbc_of(f) for f in frames]).to(dev)
    if with_cell:
        out[D.CELL_KEY] = torch.stack([f[D.CELL_KEY].reshape(3, 3).to(device=dev, dtype=dtype) if D.CELL_KEY in f
                                       else torch.zeros(3, 3, dtype=dtype, device=dev) for f in frames])
        out[D.PBC_KEY] = pbc
    if all(has_ei):
        offs = [0]
        for s in sizes[:-1]:
            offs.append(offs[-1] + s)
        out[D.EDGE_INDEX_KEY] = torch.cat([f[D.EDGE_INDEX_KEY] + o for f, o in zip(frames, offs)], 1)
        if any(D.EDGE_CELL_SHIFT_KEY in f for f in frames):
            out[D.EDGE_CELL_SHIFT_KEY] = torch.cat([f[D.EDGE_CELL_SHIFT_KEY] if D.EDGE_CELL_SHIFT_KEY in f
                                                    else torch.zeros(f[D.EDGE_INDEX_KEY].shape[1], 3, dtype=dtype, device=dev)
                                                    for f in frames], 0)
        return out
    if r_max is None:
        raise ValueError("collate: the frames carry no edge_index, so r_max is needed to build the neighbour list")
    frame_ptr = torch.zeros(B + 1, dtype=torch.int64)
    frame_ptr[1:] = torch.cumsum(torch.tensor(sizes), 0)
    csr, shift = D.neighbor_csr_frames(out[D.POSITIONS_KEY], frame_ptr, out.get(D.CELL_KEY), pbc, r_max)
    out[D.CSR_KEY], out[D.EDGE_SHIFT_VEC_KEY] = csr, shift
    return out


def _sub_csr(csr: D.EdgeCSR, a0: int, a1: int, e0: int, e1: int) -> D.EdgeCSR:
    """Rows [a0, a1) of a centre-sorted CSR (edges [e0, e1)) with the atom and edge offsets removed."""
    counts = csr.row_ptr[a0 + 1 : a1 + 1] - csr.row_ptr[a0:a1]
    row_ptr = (csr.row_ptr[a0 : a1 + 1] - e0).contiguous()
    return D.EdgeCSR(a1 - a0, (csr.ctr[e0:e1] - a0).contiguous(), (csr.nbr[e0:e1] - a0).contiguous(), row_ptr, None,
                     int(counts.max()) if a1 > a0 else 0)


def split(out: D.Type) -> List[D.Type]:
    """A batched dict (input or output of ``energy_and_forces_frames``) -> one single-frame dict per frame, with local
    atom indices.  Per-edge entries keep their order; a prepared list becomes each frame's own ``edge_csr`` /
    ``edge_shift_vec``."""
    sizes = [int(s) for s in out[D.NUM_NODES_KEY].reshape(-1).tolist()]
    B = len(sizes)
    a_off = [0]
    for s in sizes:
        a_off.append(a_off[-1] + s)
    frames: List[D.Type] = [{} for _ in range(B)]
    for b in range(B):
        a0, a1 = a_off[b], a_off[b + 1]
        for k in _PER_ATOM:
            if k in out:
                frames[b][k] = out[k][a0:a1]
        for k in _PER_FRAME:
            if k in out:
                frames[b][k] = out[k][b : b + 1] if k in _PER_FRAME_ROWS else out[k][b]
    if D.CSR_KEY in out:
        csr = out[D.CSR_KEY]
        rp = csr.row_ptr.cpu()
        for b in range(B):
            a0, a1 = a_off[b], a_off[b + 1]
            e0, e1 = int(rp[a0]), int(rp[a1])
            frames[b][D.CSR_KEY] = _sub_csr(csr, a0, a1, e0, e1)
            for k in (D.EDGE_SHIFT_VEC_KEY,) + _PER_EDGE:
                if k in out:
                    frames[b][k] = out[k][e0:e1]
    elif D.EDGE_INDEX_KEY in out:
        ei = out[D.EDGE_INDEX_KEY]
        eb = out[D.BATCH_KEY].reshape(-1)[ei[0]]
        for b in range(B):
            sel = (eb == b).nonzero().reshape(-1)
            frames[b][D.EDGE_INDEX_KEY] = ei[:, sel] - a_off[b]
            for k in _PER_EDGE:
                if k in out:
                    frames[b][k] = out[k][sel]
    return frames
