"""Geometries the neighbour-list tests run on: where a cell list goes wrong (boxes of exactly 3 r_max, cells one ulp
either side of r_max, every periodicity, layers and molecules thinner than the cutoff, raw MD coordinates many boxes
out, density extremes, the halo's local frame, a far-flung atom) and one full-size frame.

``cases()`` -> list of Case; positions are fp64 on the CPU, ``box`` the orthorhombic lengths."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

from allegro_b200 import systems

R_ODD = (5.024670687252072, 7.222109257625241)  # (3 r) // r == 2.0 in Python floats for both


@dataclass
class Case:
    name: str
    pos: torch.Tensor
    box: Tuple[float, float, float]
    pbc: Tuple[bool, bool, bool]
    r_max: float
    n_centres: Optional[int] = None  # rows for atoms [0, n_centres) only (the halo's owned atoms)
    ref_centres: Optional[int] = None  # hold that many random centres to the reference (large frames)

    @property
    def cell(self) -> torch.Tensor:
        return torch.diag(torch.tensor(self.box, dtype=torch.float64))


def _gas(n, box, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, generator=g, dtype=torch.float64) * torch.tensor(box, dtype=torch.float64)


def _hex_sheet(a, nx, ny, z=(0.0,)):
    """rectangular supercell of a hexagonal lattice (2 atoms per rectangle of a x a*sqrt(3)), one copy per layer z"""
    b = a * math.sqrt(3.0)
    base = torch.tensor([[0.0, 0.0], [0.5 * a, 0.5 * b]], dtype=torch.float64)
    ij = torch.stack(torch.meshgrid(torch.arange(nx), torch.arange(ny), indexing="ij"), -1).reshape(-1, 2).double()
    xy = (ij * torch.tensor([a, b], dtype=torch.float64)).unsqueeze(1) + base
    xy = xy.reshape(-1, 2)
    layers = []
    for k, zz in enumerate(z):  # odd layers stacked over the hollow sites
        shift = torch.tensor([0.5 * a, a / math.sqrt(3.0)], dtype=torch.float64) * (k % 2)
        layers.append(torch.cat([xy + shift, torch.full((xy.shape[0], 1), zz, dtype=torch.float64)], 1))
    return torch.cat(layers, 0), (nx * a, ny * b)


def _raw_md(pos, box, seed):
    """atoms moved by k in {+-1, +-7, +-100} box vectors, atoms on the faces, negative coordinates"""
    g = torch.Generator().manual_seed(seed)
    p = pos.clone()
    L = torch.tensor(box, dtype=torch.float64)
    ks = torch.tensor([1, -1, 7, -7, 100, -100], dtype=torch.float64)
    for i in range(0, 60, 2):
        a = int(torch.randint(0, 3, (1,), generator=g))
        p[i, a] += ks[i // 2 % 6] * L[a]
    p[1, 0], p[3, 0], p[5, 0] = 0.0, L[0], L[0] * (1 - 2.0 ** -24)
    p[7, 1], p[9, 2] = L[1], 0.0
    p[11] -= L * 0.5  # negative coordinates inside the first image below
    return p


def cases(full_size: bool = True) -> List[Case]:
    out: List[Case] = []
    # G1 periodic box of exactly 3 r_max
    for k, r in enumerate((5.5,) + R_ODD):
        L = 3 * r
        out.append(Case(f"G1-3rmax-r{r}", _gas(200, (L, L, L), 10 + k), (L, L, L), (True, True, True), r))
    # G2 cells exactly r_max wide and one ulp either side; anisotropic 3 x 4 x 11 cells
    r = 5.0
    for f, tag in ((1.0, "exact"), (1 - 1e-12, "minus"), (1 + 1e-12, "plus")):
        for k in (4, 7):
            L = k * r * f
            p = _gas(40 * k, (L, L, L), 20 + k)
            p[:k, 0] = torch.arange(k, dtype=torch.float64) * (L / k)  # atoms on the cell faces
            out.append(Case(f"G2-k{k}-{tag}", p, (L, L, L), (True, True, True), r))
        box = (3 * r * f, 4 * r * f, 11 * r * f)
        out.append(Case(f"G2-3x4x11-{tag}", _gas(300, box, 27), box, (True, True, True), r))
    # G3 all eight periodicities on one gas
    box = (20.0, 23.0, 26.0)
    gas = _gas(300, box, 3)
    for m in range(8):
        pbc = tuple(bool(m >> a & 1) for a in range(3))
        out.append(Case(f"G3-pbc{''.join('T' if p else 'F' for p in pbc)}", gas, box, pbc, 5.0))
    # G4 thin open axes
    sheet, (lx, ly) = _hex_sheet(2.46, 7, 4)
    out.append(Case("G4-graphene-TTF", sheet, (lx, ly, 20.0), (True, True, False), 5.0))
    mos2, (lx, ly) = _hex_sheet(3.16, 6, 4, z=(0.0, 1.6, 3.2))
    out.append(Case("G4-trilayer-TTF", mos2, (lx, ly, 20.0), (True, True, False), 5.5))
    wire = _gas(60, (4.0, 4.0, 20.0), 4) + torch.tensor([3.0, 3.0, 0.0], dtype=torch.float64)
    out.append(Case("G4-wire-FFT", wire, (30.0, 30.0, 20.0), (False, False, True), 5.0))
    ang = torch.arange(12, dtype=torch.float64) * (2 * math.pi / 12)
    ring = torch.stack([2.7 * torch.cos(ang), 2.7 * torch.sin(ang), torch.zeros(12, dtype=torch.float64)], 1)
    out.append(Case("G4-ring-FFF", ring, (30.0, 30.0, 30.0), (False, False, False), 5.0))
    chain = torch.zeros(10, 3, dtype=torch.float64)
    chain[:, 0] = 1.5 * torch.arange(10, dtype=torch.float64)
    out.append(Case("G4-chain-FFF", chain, (30.0, 30.0, 30.0), (False, False, False), 5.0))
    one = torch.tensor([[1.0, 2.0, 3.0]], dtype=torch.float64)
    out.append(Case("G4-one-TTF", one, (16.0, 16.0, 16.0), (True, True, False), 5.0))
    out.append(Case("G4-one-FFF", one, (16.0, 16.0, 16.0), (False, False, False), 5.0))
    two = torch.tensor([[1.0, 2.0, 3.0], [15.0, 2.5, 3.0]], dtype=torch.float64)  # neighbours only across the x face
    out.append(Case("G4-two-TTF", two, (16.0, 16.0, 16.0), (True, True, False), 5.0))
    pair = torch.tensor([[1.0, 2.0, 3.0], [1.0, 5.0, 3.0]], dtype=torch.float64)
    out.append(Case("G4-two-FFF", pair, (16.0, 16.0, 16.0), (False, False, False), 5.0))
    out.append(Case("G4-empty-TTT", torch.zeros(0, 3, dtype=torch.float64), (16.0, 16.0, 16.0), (True, True, True), 5.0))
    out.append(Case("G4-empty-TFF", torch.zeros(0, 3, dtype=torch.float64), (16.0, 16.0, 16.0), (True, False, False), 5.0))
    # G5 raw MD coordinates
    box = (20.0, 23.0, 26.0)
    raw = _raw_md(_gas(300, box, 5), box, 6)
    out.append(Case("G5-raw-TTT", raw, box, (True, True, True), 5.0))
    out.append(Case("G5-raw-TFT", raw, box, (True, False, True), 5.0))
    # G6 density extremes
    clump = _gas(50, (4.0, 4.0, 4.0), 7) + 28.0
    out.append(Case("G6-clump-in-one-cell", clump, (60.0, 60.0, 60.0), (True, True, True), 5.0))
    out.append(Case("G6-dilute", _gas(40, (60.0, 60.0, 60.0), 8), (60.0, 60.0, 60.0), (True, True, True), 5.0))
    out.append(Case("G6-dense", _gas(1229, (16.0, 16.0, 16.0), 9), (16.0, 16.0, 16.0), (True, True, True), 5.0))
    # G7 the halo's local frame: x open, owned atoms first, ghosts on both x sides
    out.append(_halo_frame())
    # G8 a far-flung atom on every open axis
    blob = _gas(500, (12.0, 12.0, 12.0), 11)
    far = torch.cat([blob, torch.full((1, 3), 1e4, dtype=torch.float64)])
    out.append(Case("G8-far-FFF", far, (30.0, 30.0, 30.0), (False, False, False), 5.0))
    farz = torch.cat([_gas(500, (16.0, 16.0, 12.0), 12), torch.tensor([[3.0, 4.0, -1e4]], dtype=torch.float64)])
    out.append(Case("G8-far-TTF", farz, (16.0, 16.0, 30.0), (True, True, False), 5.0))
    # G9 c2 at full size
    if full_size:
        pos, cell, _ = systems.make_positions("c2")
        g = torch.Generator().manual_seed(13)
        pos = pos + 0.3 * torch.randn(pos.shape, generator=g, dtype=pos.dtype)
        L = float(cell[0, 0])
        out.append(Case("G9-c2-full", pos, (L, L, L), (True, True, True), 5.0, ref_centres=512))
    return out


def _halo_frame() -> Case:
    from allegro_b200.halo import SlabDecomposition

    pos, cell, types = systems.make_positions("c2", 5)
    g = torch.Generator().manual_seed(14)
    pos = pos + 0.2 * torch.randn(pos.shape, generator=g, dtype=pos.dtype)
    # rank 0 of 2: ghosts arrive from both neighbours (rank 1 on each side, one through the periodic wrap)
    dec = SlabDecomposition(pos, cell, types, 5.0, rank=0, world=2)
    local = dec.local_positions_from_global(pos)
    box = tuple(float(v) for v in torch.diagonal(cell))
    return Case("G7-halo-local-FTT", local, box, (False, True, True), 5.0, n_centres=dec.n_owned)

