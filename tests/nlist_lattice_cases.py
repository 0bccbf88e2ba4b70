"""Geometries the general-lattice neighbour-list tests run on: non-orthogonal crystals (hcp, rhombohedral fcc, LAMMPS
boxes at the largest tilts and past them, a left-handed cell), periodic axes shorter than 3 r_max and shorter than
r_max, tilted sheets and wires, ASE's zero rows and ``cell=None``, raw coordinates 100 cells out along tilted axes, a
perfect lattice with r_max on the nearest-neighbour shell, a far-flung atom on a tilted open axis, 0 / 1 / 2 atoms,
heights of exactly 3 r_max and the c2 frame in a tilted basis.

``cases()`` -> list of LCase; positions are fp64 on the CPU, ``cell`` the [3,3] rows a user passes (or None)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

import nlist_cases

F64 = torch.float64


@dataclass
class LCase:
    name: str
    pos: torch.Tensor
    cell: Optional[torch.Tensor]
    pbc: Tuple[bool, bool, bool]
    r_max: float
    ref_centres: Optional[int] = None  # hold that many random centres to the reference (large frames)


def _rows(*r):
    return torch.tensor(r, dtype=F64)


def _gas(n, rows, seed, lo=0.0, hi=1.0):
    """n atoms uniform in the fractional box [lo, hi)^3 of ``rows``"""
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(n, 3, generator=g, dtype=F64)) @ rows


def _crystal(basis_frac, prim, reps, jitter, seed):
    """supercell reps of the primitive rows ``prim`` with fractional basis -> (pos, supercell rows)"""
    g = torch.Generator().manual_seed(seed)
    ijk = torch.stack(torch.meshgrid(*[torch.arange(k) for k in reps], indexing="ij"), -1).reshape(-1, 1, 3).to(F64)
    frac = (ijk + torch.as_tensor(basis_frac, dtype=F64).unsqueeze(0)).reshape(-1, 3)
    pos = frac @ prim
    if jitter:
        pos = pos + jitter * torch.randn(pos.shape, generator=g, dtype=F64)
    return pos, torch.diag(torch.tensor(reps, dtype=F64)) @ prim


def hcp(a=2.95, c=4.68, reps=(4, 4, 3), jitter=0.05, seed=1):
    prim = _rows([a, 0.0, 0.0], [-0.5 * a, 0.5 * math.sqrt(3.0) * a, 0.0], [0.0, 0.0, c])
    return _crystal([[0.0, 0.0, 0.0], [1 / 3, 2 / 3, 0.5]], prim, reps, jitter, seed)


def fcc_rhombohedral(a=3.6, reps=(5, 5, 5), jitter=0.05, seed=2):
    prim = 0.5 * a * _rows([0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0])
    return _crystal([[0.0, 0.0, 0.0]], prim, reps, jitter, seed)


def graphite(a=2.46, c=6.7, reps=(6, 6, 1), jitter=0.03, seed=3):
    prim = _rows([a, 0.0, 0.0], [-0.5 * a, 0.5 * math.sqrt(3.0) * a, 0.0], [0.0, 0.0, c])
    basis = [[0.0, 0.0, 0.0], [1 / 3, 2 / 3, 0.0], [0.0, 0.0, 0.5], [2 / 3, 1 / 3, 0.5]]  # AB stacking
    return _crystal(basis, prim, reps, jitter, seed)


def lammps(lx, ly, lz, xy, xz, yz):
    return _rows([lx, 0.0, 0.0], [xy, ly, 0.0], [xz, yz, lz])


def tilted_sheet(seed=4):
    """hexagonal sheet (pbc T, T, F) with a tilted, non-zero open row; atoms within 3 A of the plane"""
    rows = _rows([12.0, 0.0, 0.0], [6.0, 10.4, 0.0], [2.0, 1.0, 15.0])
    pos = _gas(120, rows, seed)
    pos[:, 2] = pos[:, 2] * 0.2 - 1.0
    return pos, rows


def tilted_wire(seed=5, zero_rows=False):
    """wire along a tilted periodic c (pbc F, F, T); atoms within a 3 A tube"""
    c = torch.tensor([2.0, 1.0, 13.0], dtype=F64)
    g = torch.Generator().manual_seed(seed)
    t = torch.rand(80, 1, generator=g, dtype=F64)
    u = torch.tensor([1.0, -2.0, 0.0], dtype=F64) / math.sqrt(5.0)
    v = torch.linalg.cross(c / c.norm(), u)
    a, b = (torch.rand(80, 2, generator=g, dtype=F64) * 6.0 - 3.0).unbind(1)
    pos = t * c + a[:, None] * u + b[:, None] * v + 10.0
    if zero_rows:
        rows = torch.stack([torch.zeros(3, dtype=F64), torch.zeros(3, dtype=F64), c])
    else:
        rows = torch.stack([torch.tensor([20.0, 3.0, 0.0], dtype=F64), torch.tensor([-1.0, 18.0, 4.0], dtype=F64), c])
    return pos, rows


def cluster(seed=6):
    """a planar flake of ~40 atoms (z extent 0) plus a few atoms above it"""
    sheet, (lx, ly) = nlist_cases._hex_sheet(2.46, 7, 4)
    sheet = sheet - torch.tensor([lx / 2, ly / 2, 0.0], dtype=F64)
    return sheet[sheet.norm(dim=-1) < 6.0].clone()


def cases(full_size: bool = True) -> List[LCase]:
    out: List[LCase] = []
    T, F = True, False
    r = 5.0
    # L1 non-orthogonal crystals
    pos, rows = hcp()
    out.append(LCase("L1-hcp-120deg", pos, rows, (T, T, T), r))
    pos, rows = fcc_rhombohedral()
    out.append(LCase("L1-fcc-rhombohedral", pos, rows, (T, T, T), r))
    rows = lammps(20.0, 18.0, 16.0, 10.0, -10.0, 5.4)  # xy = lx/2, xz = -lx/2, yz = 0.3 ly
    out.append(LCase("L1-lammps-max-tilt", _gas(300, rows, 7), rows, (T, T, T), r))
    rows = lammps(20.0, 18.0, 16.0, 60.0, 0.0, 0.0)  # "tilt large": xy = 3 lx
    out.append(LCase("L1-lammps-tilt-large", _gas(300, rows, 8), rows, (T, T, T), r))
    rows = _rows([13.0, 0.0, 0.0], [2.0, 0.0, 14.0], [1.0, 15.0, 0.0])  # det < 0
    out.append(LCase("L1-left-handed", _gas(250, rows, 9), rows, (T, T, T), r))
    # L2 short periodic axes
    pos, rows = graphite()
    out.append(LCase("L2-graphite-c6.7", pos, rows, (T, T, T), r))
    for f, n_at in ((2.2, 150), (1.0, 80), (0.4, 40)):
        rows = _rows([16.0, 0.0, 0.0], [3.0, 15.0, 0.0], [1.0, 0.5, f * r])  # height along c: f r_max
        out.append(LCase(f"L2-height-{f}r", _gas(n_at, rows, 10), rows, (T, T, T), r))
    # L3 sheets and wires with tilted rows
    pos, rows = tilted_sheet()
    out.append(LCase("L3-tilted-sheet-TTF", pos, rows, (T, T, F), r))
    rows = _rows([15.0, 0.0, 0.0], [1.0, 12.0, 2.0], [3.0, 0.0, 14.0])
    pos = _gas(120, rows, 11)
    pos = pos - (pos @ torch.linalg.inv(rows))[:, 1:2] * 0.7 * rows[1:2]  # squeeze the open b extent
    out.append(LCase("L3-tilted-slab-TFT", pos, rows, (T, F, T), r))
    pos, rows = tilted_wire()
    out.append(LCase("L3-tilted-wire-FFT", pos, rows, (F, F, T), r))
    # L4 ASE zero open rows, and no cell
    pos, rows = tilted_sheet(12)
    rows = rows.clone()
    rows[2] = 0.0
    out.append(LCase("L4-ase-sheet-zero-c", pos, rows, (T, T, F), r))
    pos, rows = tilted_wire(13, zero_rows=True)
    out.append(LCase("L4-ase-wire-zero-ab", pos, rows, (F, F, T), r))
    out.append(LCase("L4-cluster-cell-None", cluster(), None, (F, F, F), r))
    # L5 raw coordinates 100 cells out along tilted axes
    rows = lammps(20.0, 18.0, 16.0, 10.0, -10.0, 5.4)
    pos = _gas(300, rows, 14)
    ks = torch.tensor([1, -1, 7, -7, 100, -100], dtype=F64)
    g = torch.Generator().manual_seed(15)
    for i in range(0, 60, 2):
        pos[i] += ks[i // 2 % 6] * rows[int(torch.randint(0, 3, (1,), generator=g))]
    pos[1] = rows[0]  # on a face
    pos[3] = -0.5 * rows.sum(0)
    out.append(LCase("L5-raw-100-cells", pos, rows, (T, T, T), r))
    # L6 perfect fcc with r_max on the nearest-neighbour shell: every first-shell pair is a band pair
    pos, rows = fcc_rhombohedral(jitter=0.0, reps=(4, 4, 4))
    out.append(LCase("L6-fcc-rmax-at-nn", pos, rows, (T, T, T), 3.6 / math.sqrt(2.0)))
    # L7 a far-flung atom on a tilted open axis
    pos, rows = tilted_sheet(16)
    pos = torch.cat([pos, (pos[:1] + 1e4 * rows[2:3] / rows[2].norm())])
    out.append(LCase("L7-far-tilted-open", pos, rows, (T, T, F), r))
    # L8 0, 1 and 2 atoms (the single atom sees its own images along the short a row)
    rows = _rows([4.0, 0.0, 0.0], [1.0, 11.0, 0.0], [2.0, -1.0, 12.0])
    out.append(LCase("L8-empty", torch.zeros(0, 3, dtype=F64), rows, (T, T, T), r))
    out.append(LCase("L8-one", torch.tensor([[0.3, 0.2, 0.1]], dtype=F64), rows, (T, T, T), r))
    out.append(LCase("L8-two", torch.tensor([[0.3, 0.2, 0.1], [3.9, 10.0, 11.5]], dtype=F64), rows, (T, T, T), r))
    # L9 heights of exactly 3 r_max (the c axis of a LAMMPS box has height lz)
    for rr in (5.5,) + nlist_cases.R_ODD:
        rows = lammps(3.6 * rr, 3.3 * rr, 3 * rr, 0.4 * rr, -0.3 * rr, 0.2 * rr)
        out.append(LCase(f"L9-height-3rmax-r{rr}", _gas(200, rows, 17), rows, (T, T, T), rr))
    # L10 c2 at full size in a tilted basis
    if full_size:
        from allegro_b200 import systems

        pos, cell, _ = systems.make_positions("c2")
        M = torch.tensor([[1.0, 1.0, 0.0], [0.0, 1.0, 0.0], [1.0, 0.0, 1.0]], dtype=F64)  # unimodular
        out.append(LCase("L10-c2-tilted", pos, M @ cell, (T, T, T), r, ref_centres=256))
    return out
