"""AtomicDataDict keys, neighbour lists and the centre-sorted CSR edge format.

Key strings are nequip's ``AtomicDataDict`` constants (SURVEY appendix A.6; the three output
keys are confirmed by /root/reference/tests/model/test_allegro.py:233).

The on-device edge format every kernel consumes is *centre-sorted CSR*: edges ordered by
``edge_index[0]`` (the centre, allegro/nn/_allegro.py:238), ``row_ptr[N+1]`` int32,
``ctr[E]``/``nbr[E]`` int32.  With it, the per-centre environment sum of
allegro/nn/_strided/_contract.py:199-205 is a reduction over a contiguous edge range.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

POSITIONS_KEY = "pos"
EDGE_INDEX_KEY = "edge_index"
ATOM_TYPE_KEY = "atom_types"
CELL_KEY = "cell"
PBC_KEY = "pbc"
EDGE_CELL_SHIFT_KEY = "edge_cell_shift"
BATCH_KEY = "batch"
NUM_NODES_KEY = "num_atoms"
EDGE_VECTORS_KEY = "edge_vectors"
EDGE_LENGTH_KEY = "edge_lengths"
NORM_LENGTH_KEY = "normed_edge_lengths"
EDGE_TYPE_KEY = "edge_type"
EDGE_ATTRS_KEY = "edge_attrs"
EDGE_EMBEDDING_KEY = "edge_embedding"
EDGE_FEATURES_KEY = "edge_features"
EDGE_CUTOFF_KEY = "edge_cutoff"
EDGE_ENERGY_KEY = "edge_energy"
PER_ATOM_ENERGY_KEY = "atomic_energy"
TOTAL_ENERGY_KEY = "total_energy"
FORCE_KEY = "forces"
STRESS_KEY = "stress"
VIRIAL_KEY = "virial"
# prepared-frame keys (this package only): a prebuilt centre-sorted CSR (EdgeCSR) and the per-edge shift vectors
# [E,3] = edge_cell_shift @ cell in CSR order.  When present they are used instead of edge_index / edge_cell_shift,
# so the int64 COO list never has to exist (neighbor_csr below; 5x10^7 edges at the 1M-atom scale).
CSR_KEY = "edge_csr"
EDGE_SHIFT_VEC_KEY = "edge_shift_vec"
# per-atom virial and heat current (this package): velocities [N,3] in; the centroid per-atom virial [n_rows,3,3]
# (W[a] = -sum over the edges whose neighbour is a of r_z (x) dE/dr_z, not symmetric) and the potential heat current
# J = sum_a E_a v_a + W[a] v_a ([1,3] for one frame, [B,3] for a batch) out
VELOCITY_KEY = "velocities"
ATOMIC_VIRIAL_KEY = "atomic_virial"
HEAT_CURRENT_KEY = "heat_current"

Type = Dict[str, torch.Tensor]


def num_nodes(data: Type) -> int:
    return data[POSITIONS_KEY].shape[0]


# --------------------------------------------------------------------------- #
# neighbour lists
# --------------------------------------------------------------------------- #
def _brute_force(pos, cell, pbc, r_max):
    """All-pairs search over the periodic images within r_max.  Positions are first wrapped into the
    cell along the periodic axes (MD drivers hand over unwrapped coordinates; without the wrap, atoms
    that diffused by a lattice vector would lose neighbours) and the integer image offsets are folded
    back into the returned shifts, so  r = pos[j] + shift @ cell - pos[i]  holds for the RAW
    positions -- the same convention as ``_cell_list``."""
    dev = pos.device
    if cell is None or not any(pbc):
        shifts = torch.zeros(1, 3, dtype=torch.long, device=dev)
        cell_m = torch.zeros(3, 3, dtype=pos.dtype, device=dev)
        img0 = torch.zeros(pos.shape[0], 3, dtype=torch.long, device=dev)
        wrapped = pos
    else:
        cell_m = cell.view(3, 3).to(pos.dtype)
        pbc_t = torch.tensor([bool(p) for p in pbc], device=dev)
        frac = torch.linalg.solve(cell_m.T, pos.T).T  # pos = frac @ cell
        img0 = torch.where(pbc_t, torch.floor(frac), torch.zeros_like(frac)).to(torch.long)
        wrapped = pos - img0.to(pos.dtype) @ cell_m
        # number of images needed per axis: r_max / (height of the cell along that axis)
        vol = torch.det(cell_m).abs()
        cr = torch.stack([torch.linalg.cross(cell_m[1], cell_m[2]), torch.linalg.cross(cell_m[2], cell_m[0]), torch.linalg.cross(cell_m[0], cell_m[1])])
        heights = vol / cr.norm(dim=-1)
        reps = [int(math.ceil(r_max / float(h))) if p else 0 for h, p in zip(heights, pbc)]
        rng = [torch.arange(-r, r + 1, device=dev) for r in reps]
        shifts = torch.stack(torch.meshgrid(*rng, indexing="ij"), dim=-1).reshape(-1, 3)
    ei, sh = [], []
    for s in shifts:
        off = s.to(pos.dtype) @ cell_m
        d = wrapped.unsqueeze(0) + off - wrapped.unsqueeze(1)  # [i, j]
        mask = d.norm(dim=-1) < r_max
        if not bool(s.any()):
            mask.fill_diagonal_(False)
        ij = mask.nonzero()
        ei.append(ij.T)
        sh.append(s.expand(ij.shape[0], 3) - img0[ij[:, 1]] + img0[ij[:, 0]])
    return torch.cat(ei, dim=1), torch.cat(sh, dim=0)


# Narrowest cell the device search takes, as a fraction of r_max: the same bound as nl_geom in csrc/nlist.cu, so that a
# box of exactly 3 r_max (rounded either way) is one grid on both sides
CELL_WIDTH_TOL = 1 - 1e-12


def _cells_along(length: float, r_max: float) -> int:
    """Most cells of width >= r_max (to CELL_WIDTH_TOL) that fit in ``length``, at least 1.  Decided on the quotient the
    device check computes (length / n in double): ``length // r_max`` alone can be one short, (3 r) // r == 2 for many r."""
    w = r_max * CELL_WIDTH_TOL
    n = max(1, int(length // r_max))
    while length / (n + 1) >= w:
        n += 1
    while n > 1 and length / n < w:
        n -= 1
    return n


def cell_grid(pos: torch.Tensor, r_max: float, box, pbc=(True, True, True)):
    """Grid of the cell-list search (``neighbor_csr`` and ``neighbor_list(method="cell")``) for an orthorhombic box of
    lengths ``box`` -> (box [3], origin [3], ncell [3]) as Python numbers, or None when a periodic axis is shorter
    than 3 r_max.

    * Periodic axes span [0, L) with the most cells of width >= r_max; at least 3, so the 27-cell walk never visits a
      cell twice.
    * Open axes span the occupied extent [lo, hi], widened to r_max when thinner (a sheet, a wire, a molecule, one
      atom): one cell of width >= r_max is a valid grid.
    * The cell count stays at most max(27, 4 N): an atom far out on an open axis would otherwise ask for billions of
      mostly empty cells (and overflow the int32 cell id).  Open axes are coarsened first, periodic axes never below 3
      cells; wider cells are always correct, only slower.
    Every grid returned has cells >= r_max wide (to CELL_WIDTH_TOL) and passes the device check (``nl_geom`` in
    csrc/nlist.cu)."""
    r = float(r_max)
    pbc = [bool(p) for p in pbc]
    box = [float(b) for b in box]
    origin = [0.0, 0.0, 0.0]
    n = int(pos.shape[0])
    open_axes = [a for a in range(3) if not pbc[a]]
    if open_axes:
        lo, hi = (pos.amin(0).tolist(), pos.amax(0).tolist()) if n > 0 else ([0.0] * 3, [0.0] * 3)
        for a in open_axes:
            origin[a] = float(lo[a])
            box[a] = max((float(hi[a]) - float(lo[a])) * (1 + 1e-9) + 1e-6, r)
    if any(p and not box[a] > 0 for a, p in enumerate(pbc)):
        return None
    ncell = [_cells_along(b, r) for b in box]
    if any(p and ncell[a] < 3 for a, p in enumerate(pbc)):
        return None
    limit = max(27, 4 * n)
    while ncell[0] * ncell[1] * ncell[2] > limit:
        cand = [a for a in open_axes if ncell[a] > 1] or [a for a in range(3) if pbc[a] and ncell[a] > 3]
        a = max(cand, key=lambda x: ncell[x])
        ncell[a] = max(3 if pbc[a] else 1, ncell[a] // 2)
    return box, origin, ncell


def _cell_list(pos, box, r_max, pbc=(True, True, True), origin=None, ncell=None):
    """Orthorhombic box, per-axis periodicity.  Periodic axes need >= 3 cells; on a
    non-periodic axis the grid spans [origin, origin+box) and nothing wraps.  ``ncell``: the grid of ``cell_grid``
    (default: cells of edge >= r_max)."""
    dev = pos.device
    n = pos.shape[0]
    pbc_t = torch.tensor([bool(p) for p in pbc], device=dev)
    if origin is None:
        origin = torch.zeros(3, dtype=pos.dtype, device=dev)
    if ncell is None:
        ncell = torch.floor(box / r_max).to(torch.long).clamp(min=1)
    else:
        ncell = torch.tensor([int(c) for c in ncell], dtype=torch.long, device=dev)
    assert int(ncell[pbc_t].min() if bool(pbc_t.any()) else 3) >= 3, "cell list needs box >= 3 r_max on every periodic axis"
    rel = pos - origin
    img0 = torch.where(pbc_t, torch.floor(rel / box), torch.zeros_like(rel)).to(torch.long)  # image index of the raw position
    wrapped = rel - img0.to(pos.dtype) * box
    cidx3 = torch.minimum(torch.clamp((wrapped / box * ncell).to(torch.long), min=0), ncell - 1)
    nc = [int(v) for v in ncell]
    cid = (cidx3[:, 0] * nc[1] + cidx3[:, 1]) * nc[2] + cidx3[:, 2]
    order = torch.argsort(cid, stable=True)
    ncells = nc[0] * nc[1] * nc[2]
    counts = torch.bincount(cid, minlength=ncells)
    starts = torch.cumsum(counts, 0) - counts
    ei, sh = [], []
    ar = torch.arange(n, device=dev)
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                d = torch.tensor([dx, dy, dz], device=dev)
                c3 = cidx3 + d
                img = torch.div(c3, ncell, rounding_mode="floor")  # -1, 0, +1
                valid = (pbc_t | (img == 0)).all(-1)
                img = torch.where(pbc_t, img, torch.zeros_like(img))
                c3w = torch.clamp(c3 - img * ncell, min=0)
                c3w = torch.minimum(c3w, ncell - 1)
                ncid = (c3w[:, 0] * nc[1] + c3w[:, 1]) * nc[2] + c3w[:, 2]
                cnt = counts[ncid] * valid
                tot = int(cnt.sum())
                if tot == 0:
                    continue
                i_rep = torch.repeat_interleave(ar, cnt)
                offs = torch.arange(tot, device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
                j_rep = order[starts[ncid][i_rep] + offs]
                img_rep = img[i_rep]
                rij = wrapped[j_rep] + img_rep.to(pos.dtype) * box - wrapped[i_rep]
                keep = (rij.norm(dim=-1) < r_max) & ~((i_rep == j_rep) & (img_rep == 0).all(-1))
                i_k, j_k = i_rep[keep], j_rep[keep]
                # shift relative to the *raw* positions: r = pos[j] + shift*box - pos[i]
                s = img_rep[keep] - img0[j_k] + img0[i_k]
                ei.append(torch.stack([i_k, j_k]))
                sh.append(s)
    if not ei:
        return torch.zeros(2, 0, dtype=torch.long, device=dev), torch.zeros(0, 3, dtype=torch.long, device=dev)
    return torch.cat(ei, dim=1), torch.cat(sh, dim=0)


def neighbor_list(
    pos: torch.Tensor,
    r_max: float,
    cell: Optional[torch.Tensor] = None,
    pbc=(True, True, True),
    method: str = "auto",
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Full (directed) neighbour list, sorted by centre then neighbour.
    Returns edge_index [2,E] int64 (row 0 = centre) and edge_cell_shift [E,3] (pos dtype)."""
    pbc = tuple(bool(p) for p in (pbc if not isinstance(pbc, bool) else (pbc,) * 3))
    ortho = cell is not None and bool((cell.view(3, 3) - torch.diag(torch.diagonal(cell.view(3, 3)))).abs().max() == 0)
    grid = None
    if ortho and (method == "cell" or (method == "auto" and pos.shape[0] > 3000)):
        grid = cell_grid(pos, r_max, torch.diagonal(cell.view(3, 3)).tolist(), pbc)
    if method == "auto":
        method = "cell" if grid is not None else "brute"
    if method == "cell":
        if grid is None:
            raise ValueError("the cell list needs an orthorhombic box with >= 3 r_max on every periodic axis")
        box_l, origin_l, ncell = grid  # open axes: grid over the occupied extent
        box = torch.tensor(box_l, dtype=pos.dtype, device=pos.device)
        origin = torch.tensor(origin_l, dtype=pos.dtype, device=pos.device)
        ei, sh = _cell_list(pos, box, float(r_max), pbc, origin, ncell)
    else:
        ei, sh = _brute_force(pos, cell, pbc, float(r_max))
    n = pos.shape[0]
    # sort by (centre, neighbour); ties (same pair through different images) keep a deterministic order
    # via the shift.  Successive stable sorts from the least significant key (any shift magnitude --
    # raw MD positions may sit many cells away from the home cell).
    order = torch.arange(ei.shape[1], device=ei.device)
    for k in (sh[:, 2], sh[:, 1], sh[:, 0], ei[0] * n + ei[1]):
        order = order[torch.argsort(k[order], stable=True)]
    return ei[:, order].contiguous(), sh[order].to(pos.dtype).contiguous()


# --------------------------------------------------------------------------- #
# CSR edge format
# --------------------------------------------------------------------------- #
class EdgeCSR:
    """Centre-sorted edge list. ``perm`` maps sorted position -> original edge (None if the
    input was already sorted).  ``radius``: the single radius the list holds every pair within (set by the device
    searches; None when unknown or after ``prune_csr``)."""

    __slots__ = ("num_atoms", "num_edges", "ctr", "nbr", "row_ptr", "perm", "max_degree", "radius", "_transposed")

    def __init__(self, num_atoms, ctr, nbr, row_ptr, perm, max_degree, radius: Optional[float] = None):
        self.num_atoms = int(num_atoms)
        self.num_edges = int(ctr.shape[0])
        self.ctr, self.nbr, self.row_ptr, self.perm = ctr, nbr, row_ptr, perm
        self.max_degree = int(max_degree)
        self.radius = None if radius is None else float(radius)
        self._transposed = None

    def transposed(self, n_total: int):
        """Transposed CSR for the neighbour-side force reduction (ab2_force_scatter): ``col_ptr``
        [n_total+1] int32 and ``col_perm`` [E] int32 = edge ids grouped by neighbour atom, in
        ascending edge order inside a group (stable sort -> a fixed summation order).  Built once
        per neighbour list; ``n_total`` counts owned + ghost atoms."""
        if self._transposed is None or self._transposed[0] != int(n_total):
            nbr64 = self.nbr.long()
            col_perm = torch.argsort(nbr64, stable=True).to(torch.int32).contiguous()
            counts = torch.bincount(nbr64, minlength=int(n_total))
            if counts.shape[0] != int(n_total):
                raise ValueError("edge neighbour index out of range")
            col_ptr = torch.zeros(int(n_total) + 1, dtype=torch.int32, device=self.nbr.device)
            col_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
            self._transposed = (int(n_total), col_ptr, col_perm)
        return self._transposed[1], self._transposed[2]


def build_csr(edge_index: torch.Tensor, num_centres: int) -> EdgeCSR:
    """Sort edges by centre (stable) and build row_ptr.  ``num_centres`` = number of atoms that
    may be centres (owned atoms); neighbour indices may exceed it (ghost atoms,
    /root/reference/allegro/_compile.py:41-61)."""
    ctr64, nbr64 = edge_index[0], edge_index[1]
    E = ctr64.shape[0]
    if E > 0 and bool((ctr64[1:] >= ctr64[:-1]).all()):
        perm = None
    else:
        perm = torch.argsort(ctr64, stable=True)
        ctr64, nbr64 = ctr64[perm], nbr64[perm]
    counts = torch.bincount(ctr64, minlength=num_centres)
    if counts.shape[0] != num_centres:
        raise ValueError("edge centre index out of range")
    row_ptr = torch.zeros(num_centres + 1, dtype=torch.int32, device=edge_index.device)
    row_ptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
    maxdeg = int(counts.max()) if E > 0 else 0
    return EdgeCSR(num_centres, ctr64.to(torch.int32).contiguous(), nbr64.to(torch.int32).contiguous(), row_ptr, perm, maxdeg)


def to_ghost_format(data: Type) -> Type:
    """PBC (cell shifts) -> appended ghost atoms, the pair_allegro data contract
    (/root/reference/allegro/_compile.py:17-65): ghost pos = pos[j] + shift @ cell, ghost index
    = N + arange, inside-cell edges first.  Also the single-r_max halo format used for the
    multi-GPU decomposition."""
    data = dict(data)
    data.pop(BATCH_KEY, None)
    data.pop(NUM_NODES_KEY, None)
    if EDGE_CELL_SHIFT_KEY not in data:
        return data
    pos, ei = data[POSITIONS_KEY], data[EDGE_INDEX_KEY]
    shift, cell = data[EDGE_CELL_SHIFT_KEY], data[CELL_KEY].view(3, 3)
    outside = shift.abs().sum(-1) != 0
    ei_out = ei[:, outside].clone()
    pos_out = pos[ei_out[1]] + shift[outside].to(pos.dtype) @ cell.to(pos.dtype)
    typ = data[ATOM_TYPE_KEY].reshape(-1)
    typ_out = typ[ei_out[1]]
    ei_out[1] = torch.arange(pos.shape[0], pos.shape[0] + pos_out.shape[0], device=pos.device)
    data[POSITIONS_KEY] = torch.cat([pos, pos_out], 0)
    data[ATOM_TYPE_KEY] = torch.cat([typ, typ_out], 0)
    data[EDGE_INDEX_KEY] = torch.cat([ei[:, ~outside], ei_out], 1)
    data.pop(EDGE_CELL_SHIFT_KEY)
    data.pop(CELL_KEY)
    data.pop(PBC_KEY, None)
    data["num_local_atoms"] = torch.tensor(pos.shape[0])
    return data


def _lattice_metrics(h):
    """-> (det, heights [3], regular) of the rows ``h``, with the operations of nl_lattice_geom (csrc/nlist.cu) in the same
    order, so that the host and the device agree on every quotient: H_a = |det| / |h_p x h_q|; regular = finite and
    |det| > 1e-12 |h_0| |h_1| |h_2| (rows not within 1e-12 rad of a common plane)."""
    cr, norm = [], []
    for a in range(3):
        p, q = h[(a + 1) % 3], h[(a + 2) % 3]
        cr.append((p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]))
        norm.append(math.sqrt(h[a][0] * h[a][0] + h[a][1] * h[a][1] + h[a][2] * h[a][2]))
    det = h[0][0] * cr[0][0] + h[0][1] * cr[0][1] + h[0][2] * cr[0][2]
    regular = math.isfinite(det) and abs(det) > 1e-12 * norm[0] * norm[1] * norm[2]
    if not regular:
        return det, None, False
    heights = [abs(det) / math.sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) for c in cr]
    return det, heights, True


def is_regular_cell(cell: torch.Tensor) -> bool:
    """Finite rows not within 1e-12 rad of a common plane: the test the lattice search (nl_lattice_geom) and the
    calculator's stress apply."""
    return _lattice_metrics(cell.detach().reshape(3, 3).to(device="cpu", dtype=torch.float64).tolist())[2]


def _lattice_metrics_batched(h: torch.Tensor):
    """``_lattice_metrics`` of every frame of h [B,3,3] (fp64, CPU), the same operations in the same order, so bitwise
    the same -> (regular [B] bool, heights [B,3], NaN where not regular).  numpy, whose square root is correctly rounded
    (torch's vectorised CPU square root is not always)."""
    h = h.numpy()
    cr, sq = [], []
    with np.errstate(all="ignore"):
        for a in range(3):
            p, q, r = h[:, (a + 1) % 3], h[:, (a + 2) % 3], h[:, a]
            cr.append((p[:, 1] * q[:, 2] - p[:, 2] * q[:, 1], p[:, 2] * q[:, 0] - p[:, 0] * q[:, 2], p[:, 0] * q[:, 1] - p[:, 1] * q[:, 0]))
            sq.append(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2])
        det = h[:, 0, 0] * cr[0][0] + h[:, 0, 1] * cr[0][1] + h[:, 0, 2] * cr[0][2]
        regular = np.isfinite(det) & (np.abs(det) > 1e-12 * np.sqrt(sq[0]) * np.sqrt(sq[1]) * np.sqrt(sq[2]))
        heights = np.stack([np.abs(det) / np.sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) for c in cr], 1)
    heights[~regular] = np.nan
    return torch.from_numpy(regular), torch.from_numpy(heights)


def regular_cells(cell: torch.Tensor) -> torch.Tensor:
    """``is_regular_cell`` of every frame of a batch: cell [B,3,3] -> bool [B] on the CPU."""
    return _lattice_metrics_batched(cell.detach().reshape(-1, 3, 3).to(device="cpu", dtype=torch.float64))[0]


def _unit(v):
    n = math.sqrt(sum(x * x for x in v))
    return [x / n for x in v] if n > 0 and math.isfinite(n) else None


def _cross(p, q):
    return [p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]]


def _complete_open_rows(h, pbc):
    """Rows with every open axis replaced: the unit normal of the two periodic rows (one open axis), an orthonormal
    completion of the one periodic row (two), the identity (three).  None when the periodic rows are degenerate."""
    per = [a for a in range(3) if pbc[a]]
    opn = [a for a in range(3) if not pbc[a]]
    h = [list(r) for r in h]
    if len(per) == 2:
        u = _unit(_cross(h[per[0]], h[per[1]]))
        if u is None:
            return None
        h[opn[0]] = u
    elif len(per) == 1:
        v = _unit(h[per[0]])
        if v is None:
            return None
        e = [0.0, 0.0, 0.0]
        e[min(range(3), key=lambda x: abs(v[x]))] = 1.0  # the axis least aligned with v
        d = sum(e[x] * v[x] for x in range(3))
        u1 = _unit([e[x] - d * v[x] for x in range(3)])
        h[opn[0]], h[opn[1]] = u1, _cross(v, u1)
    elif len(per) == 0:
        h = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]
    return h


def _reach_along(height: float, n: int, r_max: float) -> int:
    """Fewest bins k with (height / n) * k >= r_max (to CELL_WIDTH_TOL), on the quotient nl_lattice_geom computes."""
    w = r_max * CELL_WIDTH_TOL
    k = max(1, math.ceil(w / (height / n)))
    while height / n * k < w:
        k += 1
    while k > 1 and height / n * (k - 1) >= w:
        k -= 1
    return k


def lattice_grid(pos: torch.Tensor, r_max: float, cell: Optional[torch.Tensor], pbc=(True, True, True)):
    """Grid of the general-lattice cell list (``neighbor_csr`` for the frames ``cell_grid`` does not take) -> (rows [3][3],
    origin [3], ncell [3], reach [3]) as Python numbers, or None.

    * Atoms are binned in fractional coordinates f = pos . rows^-1 - origin; bins are parallelepipeds of thickness
      t_a = H_a / ncell_a (H_a the height of the rows along a) and a centre walks reach_a = ceil(r_max / t_a) bins
      either side (to CELL_WIDTH_TOL).  Periodic axes keep the cell's rows and take the most bins with t_a >= r_max:
      one bin and reach > 1 when the cell is thinner than r_max.
    * Open-axis rows that are zero (ASE's 2-D and 1-D cells), or that leave the cell singular, and all rows of a frame
      with ``cell=None`` and no periodic axis, are replaced: by the unit normal of the periodic rows (one open axis) or an
      orthonormal completion (more).  Shifts along open axes are 0, so a replaced row never reaches an output.
    * An open axis spans the occupied fractional extent, widened to r_max: its row is scaled so that the atoms lie in
      [0, 1) from ``origin``.
    * The bin count stays at most max(27, 4 N): open axes are coarsened first, then periodic ones, down to 1 bin.
    None when a periodic axis has no cell (``cell=None``), the periodic rows are singular or not finite, or the walk
    would visit 2^31 - 1 or more bins per centre.  Every grid returned passes the device check (nl_lattice_geom)."""
    r = float(r_max)
    pbc = [bool(p) for p in pbc]
    n = int(pos.shape[0])
    if cell is None:
        if any(pbc):
            return None
        h = [[0.0] * 3 for _ in range(3)]
    else:
        h = cell.detach().reshape(3, 3).to(device="cpu", dtype=torch.float64).tolist()
    open_axes = [a for a in range(3) if not pbc[a]]
    if not all(math.isfinite(v) for a in range(3) if pbc[a] for v in h[a]):
        return None
    if open_axes and (any(not any(h[a]) for a in open_axes) or not all(math.isfinite(v) for row in h for v in row)
                      or not _lattice_metrics(h)[2]):
        h = _complete_open_rows(h, pbc)
        if h is None:
            return None
    det, heights, regular = _lattice_metrics(h)
    if not regular:
        return None
    origin = [0.0, 0.0, 0.0]
    if open_axes:
        # fractional extent of the atoms along the open axes (hinv column a = (h_p x h_q) / det)
        cols = [_cross(h[(a + 1) % 3], h[(a + 2) % 3]) for a in open_axes]
        hinv = torch.tensor(cols, dtype=torch.float64, device=pos.device).T / det
        if n > 0:
            f = pos.detach().to(torch.float64) @ hinv
            lo, hi = f.amin(0).tolist(), f.amax(0).tolist()
        else:
            lo, hi = [0.0] * len(open_axes), [0.0] * len(open_axes)
        for k, a in enumerate(open_axes):
            # in length units across the axis; half the margin goes below the lowest atom
            span = max((hi[k] - lo[k]) * heights[a] * (1 + 1e-9) + 1e-6, r)
            s = span / heights[a]
            h[a] = [v * s for v in h[a]]
            origin[a] = (lo[k] - 0.5e-9 * (hi[k] - lo[k]) - 0.5e-6 / heights[a]) / s
        det, heights, regular = _lattice_metrics(h)
        if not regular:
            return None
    ncell = [_cells_along(heights[a], r) for a in range(3)]
    limit = max(27, 4 * n)
    while ncell[0] * ncell[1] * ncell[2] > limit:
        cand = [a for a in open_axes if ncell[a] > 1] or [a for a in range(3) if ncell[a] > 1]
        a = max(cand, key=lambda x: ncell[x])
        ncell[a] = max(1, ncell[a] // 2)
    reach = [_reach_along(heights[a], ncell[a], r) for a in range(3)]
    if math.prod(2 * k + 1 for k in reach) >= 2**31 - 1 or math.prod(ncell) >= 2**31 - 1:
        return None
    return h, origin, ncell, reach


def csr_supported(pos: torch.Tensor, r_max: float, cell: Optional[torch.Tensor], pbc=(True, True, True)) -> bool:
    """Can ``neighbor_csr`` (CUDA cell list) take this frame?  CUDA positions and any cell ``lattice_grid`` accepts:
    orthorhombic or triclinic, periodic axes of any height, open axes of any extent (zero rows included), or no cell
    at all when no axis is periodic.  Frames ``cell_grid`` accepts (an orthorhombic box with >= 3 r_max on every
    periodic axis) take the orthorhombic grid, every other frame the general-lattice one."""
    return _csr_grid(pos, r_max, cell, pbc) is not None


def search_grid(pos, r_max, cell, pbc):
    """The grid ``neighbor_csr`` searches this frame on (for positions on any device) -> ("ortho", ``cell_grid``),
    ("lattice", ``lattice_grid``) or None."""
    if cell is not None:
        c = cell.view(3, 3)
        if bool((c - torch.diag(torch.diagonal(c))).abs().max() == 0):
            grid = cell_grid(pos, r_max, torch.diagonal(c).tolist(), pbc)
            if grid is not None:
                return "ortho", grid
    grid = lattice_grid(pos, r_max, cell, pbc)
    return None if grid is None else ("lattice", grid)


def _csr_grid(pos, r_max, cell, pbc):
    if not pos.is_cuda:
        return None
    return search_grid(pos, r_max, cell, pbc)


def _csr_of(row_ptr: torch.Tensor, nbr: torch.Tensor, radius: Optional[float]) -> EdgeCSR:
    """EdgeCSR of device rows (``ctr`` and ``max_degree`` rebuilt from row_ptr)."""
    nc = row_ptr.shape[0] - 1
    counts = (row_ptr[1:] - row_ptr[:-1])
    ctr = torch.repeat_interleave(torch.arange(nc, device=row_ptr.device, dtype=torch.int32), counts.long())
    maxdeg = int(counts.max()) if nc > 0 else 0
    return EdgeCSR(nc, ctr.contiguous(), nbr, row_ptr, None, maxdeg, radius)


def neighbor_csr(pos: torch.Tensor, r_max: float, cell: Optional[torch.Tensor], pbc=(True, True, True), n_centres: Optional[int] = None,
                 types: Optional[torch.Tensor] = None, cutoffs: Optional[torch.Tensor] = None):
    """Neighbour search on the device straight into the kernels' format -> (EdgeCSR, shift_vec [E,3] in the positions'
    dtype).  Centres are atoms [0, n_centres) (owned atoms first).  An orthorhombic box with >= 3 r_max per periodic
    axis takes ab2_nl_bin / count / fill (SURVEY 8 row f2); any other cell, and ``cell=None`` for a frame without
    periodic axes, takes ab2_nl_lattice_bin / count / fill.  r = pos[nbr] + shift - pos[ctr] holds for the raw positions.

    ``cutoffs`` [T,T] (with ``types`` [n], one per atom): the list searched at ``r_max`` is then pruned to the per-type-pair
    radii (``prune_csr``; every refusal of ``prune_csr`` is raised before the search)."""
    from . import _lib

    pbc = tuple(bool(p) for p in (pbc if not isinstance(pbc, bool) else (pbc,) * 3))
    route = _csr_grid(pos, r_max, cell, pbc)
    if route is None:
        raise ValueError("neighbor_csr needs CUDA positions and a finite non-singular cell on the periodic axes (or cell=None "
                         "with no periodic axis)")
    n = pos.shape[0]
    prune = _prune_args(types, cutoffs, n, r_max, pos.device)
    kind, grid = route
    nc = n if n_centres is None else int(n_centres)
    if kind == "ortho":
        box, origin, ncell = grid
        row_ptr, nbr, shift = _lib.neighbor_csr(pos, r_max, box, ncell, pbc, origin, nc)
    else:
        rows, origin, ncell, reach = grid
        row_ptr, nbr, shift = _lib.neighbor_csr_lattice(pos, r_max, rows, origin, ncell, reach, pbc, nc)
    if prune is not None:
        return _prune(pos, row_ptr, nbr, shift, *prune)
    return _csr_of(row_ptr, nbr, r_max), shift


def _prune_args(types: Optional[torch.Tensor], cutoffs: Optional[torch.Tensor], n: int, r_list: Optional[float], device):
    """Checks of ``prune_csr``, all made with ONE device-to-host read -> (types [n] int32, cut2 [T*T] fp64) on ``device``, or
    None when neither ``types`` nor ``cutoffs`` is given."""
    if cutoffs is None and types is None:
        return None
    if cutoffs is None or types is None:
        raise ValueError("pruning needs both the per-atom types and the [T, T] cutoff table")
    if r_list is None:
        raise ValueError("prune_csr: the radius the list was built with is unknown; pass r_list")
    c = torch.as_tensor(cutoffs)
    if c.dim() != 2 or c.shape[0] != c.shape[1] or c.shape[0] < 1:
        raise ValueError(f"the cutoff table must be [T, T] with T >= 1, got shape {tuple(c.shape)}")
    T = int(c.shape[0])
    t = torch.as_tensor(types).reshape(-1)
    if t.shape[0] != n:
        raise ValueError(f"types has {t.shape[0]} entries for {n} atoms: one type per atom (neighbours included)")
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise ValueError(f"types must be integers, got {t.dtype}")
    c64 = c.detach().to(torch.float64).reshape(-1)
    # one read: the table and the type range
    ext = torch.stack([t.min(), t.max()]).to(device=c64.device, dtype=torch.float64) if n else c64.new_zeros(0)
    host = torch.cat([c64, ext]).cpu()
    tab, trange = host[: T * T], host[T * T:].tolist()
    if not bool(torch.isfinite(tab).all()) or not bool((tab > 0).all()):
        raise ValueError(f"every cutoff must be finite and > 0, got {tab.view(T, T).tolist()}")
    if float(tab.max()) > float(r_list):
        raise ValueError(f"a cutoff ({float(tab.max())!r}) exceeds the radius the list was built with ({float(r_list)!r}): pairs "
                         "between them are not in the list")
    if trange and (trange[0] < 0 or trange[1] >= T):
        raise ValueError(f"types must lie in [0, {T}), got [{int(trange[0])}, {int(trange[1])}]")
    cut2 = (tab * tab).view(T, T).to(device)
    return t.to(device=device, dtype=torch.int32).contiguous(), cut2


def _prune(pos, row_ptr, nbr, shift, types_i32, cut2):
    from . import _lib

    row_ptr, nbr, shift = _lib.nl_prune(pos, row_ptr, nbr, shift, types_i32, cut2)
    return _csr_of(row_ptr, nbr, None), shift


def prune_csr(csr: EdgeCSR, shift_vec: torch.Tensor, pos: torch.Tensor, types: torch.Tensor, cutoffs: torch.Tensor,
              r_list: Optional[float] = None) -> Tuple[EdgeCSR, torch.Tensor]:
    """Drop the edges at or beyond their own pair's radius (ab2_nl_prune_count / fill) -> (EdgeCSR, shift_vec).

    Edge z (centre i, neighbour j, shift s) is kept iff d2 < cutoffs[t_i, t_j]^2, d2 = sum_x (pos[j] + s - pos[i])_x^2 in
    fp64 with the operations of include/allegro_b200.h.  ``cutoffs`` [T,T] is directed (row = centre type), indexed as the
    model's ``rmax_table``; ``types`` [n] holds one type per atom of ``pos`` (neighbours included).  Each row of the result
    is an ordered subsequence of the input row, with nbr and shift copied bitwise; ``ctr`` and ``max_degree`` are rebuilt,
    ``perm`` is dropped (per-edge outputs of a pruned list are in its own order).  ``r_list``: the radius the list was
    built with (default ``csr.radius``).  Raises ValueError before any launch when the table is not [T,T], an entry is
    not finite or <= 0 or exceeds ``r_list``, or ``types`` has the wrong length or values outside [0, T).  The checks cost
    one device-to-host read."""
    n = pos.shape[0]
    if csr.row_ptr.shape[0] != csr.num_atoms + 1 or csr.num_atoms > n:
        raise ValueError(f"the list has {csr.num_atoms} centres for {n} atoms")
    prune = _prune_args(types, cutoffs, n, csr.radius if r_list is None else r_list, pos.device)
    return _prune(pos, csr.row_ptr, csr.nbr, shift_vec, *prune)


# Largest frame neighbor_csr_frames takes: its search is all-pairs per frame, O(N_b^2 * images).  Larger frames belong to
# neighbor_csr (cell list) or neighbor_list.
FRAMES_MAX_ATOMS = 4096
# Most images per pair, prod_a (2 n_a + 1), neighbor_csr_frames searches: a cell 0.01 r_max high on every axis needs
# 201^3 = 8.1e6.  Such frames belong to neighbor_csr, whose cell list visits bins instead of images.
FRAMES_MAX_IMAGES = 1 << 20


def _frames_pbc(pbc, B: int, device) -> torch.Tensor:
    if pbc is None:
        return torch.zeros(B, 3, dtype=torch.bool, device=device)
    if isinstance(pbc, bool):
        pbc = (pbc,) * 3
    t = torch.as_tensor(pbc, dtype=torch.bool, device=device)
    if t.dim() == 1:
        t = t.expand(B, 3)
    if tuple(t.shape) != (B, 3):
        raise ValueError(f"pbc has shape {tuple(t.shape)}, expected (3,) or ({B}, 3)")
    return t


def frames_geometry(cell: Optional[torch.Tensor], pbc: torch.Tensor, r_max: float, dtype=torch.float64):
    """Geometry of every frame of a batch for ab2_nl_frames_* -> (rows [B,3,3] fp64, nimg [B,3] int64), both on the CPU.

    ``cell`` [B,3,3] or None, ``pbc`` [B,3] booleans, ``dtype`` the positions' dtype: the rows are those the search sees,
    the cell rounded to ``dtype``.
    * A frame with no periodic axis gets zero rows and no images: a molecule, its cell is not used.
    * Open-axis rows that are zero (ASE's 2-D and 1-D cells), not finite, or that leave the cell singular are replaced as
      ``lattice_grid`` replaces them (``_complete_open_rows``).  Shifts along open axes are 0, so a replaced row never
      reaches an output.
    * A periodic axis a searches nimg_a = ceil(r_max / H_a) images on each side, H_a the height of the rows along a,
      computed in fp64 with the operations of ``_lattice_metrics``.
    Raises ValueError, before any search, for a periodic frame without a cell, a non-finite periodic row, rows that
    ``is_regular_cell`` rejects (a zero periodic row, rows within 1e-12 rad of a common plane), or more than
    FRAMES_MAX_IMAGES images per pair.  Applied to its own rows it returns them unchanged, with the same counts:
    ``_lib.nl_frames`` takes the kernels' image counts from it."""
    pbc = pbc.to(device="cpu", dtype=torch.bool).numpy()
    B = pbc.shape[0]
    periodic = pbc.any(axis=1)
    if cell is None:
        if periodic.any():
            raise ValueError("periodic frames need a cell")
        return torch.zeros(B, 3, 3, dtype=torch.float64), torch.zeros(B, 3, dtype=torch.int64)
    if cell.numel() != 9 * B:
        raise ValueError(f"cell has {cell.numel()} entries for {B} frames")
    h = cell.detach().reshape(B, 3, 3).to(device="cpu", dtype=dtype).to(torch.float64).numpy().copy()
    h[~periodic] = 0.0
    finite = np.isfinite(h).all(axis=2)
    bad = (pbc & ~finite).any(axis=1)
    if bad.any():
        raise ValueError(f"frame {int(np.flatnonzero(bad)[0])} has a periodic cell row that is not finite")
    regular, heights = _lattice_metrics_batched(torch.from_numpy(np.where(finite[:, :, None], h, 0.0)))
    regular = regular.numpy()
    zero_open = ((h == 0).all(axis=2) & ~pbc).any(axis=1)
    fix = periodic & (~pbc).any(axis=1) & (zero_open | ~finite.all(axis=1) | ~regular)
    if fix.any():
        for b in np.flatnonzero(fix).tolist():
            rows = _complete_open_rows(h[b].tolist(), pbc[b].tolist())
            if rows is not None:
                h[b] = torch.tensor(rows, dtype=torch.float64).to(dtype).to(torch.float64).numpy()
        regular, heights = _lattice_metrics_batched(torch.from_numpy(h))
        regular = regular.numpy()
    bad = periodic & ~regular
    if bad.any():
        raise ValueError(f"frame {int(np.flatnonzero(bad)[0])} has a singular or near-coplanar periodic cell "
                         "(rows within 1e-12 rad of a common plane)")
    with np.errstate(invalid="ignore"):
        nimg = np.where(pbc, np.ceil(float(r_max) / heights.numpy()), 0.0)
    images = (2 * nimg + 1).prod(axis=1)
    bad = ~(images <= FRAMES_MAX_IMAGES)
    if bad.any():
        b = int(np.flatnonzero(bad)[0])
        raise ValueError(f"frame {b} needs {float(images[b]):.3g} periodic images per pair (cell heights "
                         f"{heights[b].tolist()} for r_max {r_max}); neighbor_csr_frames searches at most {FRAMES_MAX_IMAGES}: "
                         "use neighbor_csr")
    return torch.from_numpy(h), torch.from_numpy(nimg.astype(np.int64))


def neighbor_csr_frames(pos: torch.Tensor, frame_ptr, cell: Optional[torch.Tensor], pbc, r_max: float, types: Optional[torch.Tensor] = None,
                        cutoffs: Optional[torch.Tensor] = None):
    """Neighbour lists of a batch of small frames in one pass on the device (ab2_nl_frames_count / fill), straight into the
    kernels' format -> (EdgeCSR over all atoms of the batch, shift_vec [E,3] in the positions' dtype).

    ``frame_ptr`` [B+1]: the atoms of frame b are [frame_ptr[b], frame_ptr[b+1]).  ``cell`` [B,3,3] (or None: no frame is
    periodic), ``pbc`` [B,3] or (3,) booleans.  Any regular cell: triclinic, left-handed, narrower than r_max, mixed
    periodicity, ASE's zero rows on open axes; a frame with no periodic axis is a molecule (its cell is not used).  Rows
    are those of ``neighbor_list(frame, method="brute")`` in the same order (by neighbour, then by image), with the frame's
    atom offset added;  r = pos[nbr] + shift - pos[ctr]  holds for the raw positions.  Refused with ValueError before any
    search (``frames_geometry``): frames above FRAMES_MAX_ATOMS atoms (the search is all-pairs per frame), periodic frames
    with a non-finite, singular or near-coplanar cell, and frames needing more than FRAMES_MAX_IMAGES images per pair.
    ``cutoffs`` [T,T] with ``types`` [n]: the list is pruned to per-type-pair radii, as in ``neighbor_csr``."""
    from . import _lib

    dev = pos.device
    fp = torch.as_tensor(frame_ptr).reshape(-1).to(device="cpu", dtype=torch.int64)
    B = fp.shape[0] - 1
    n = pos.shape[0]
    if B < 1 or int(fp[0]) != 0 or int(fp[-1]) != n or bool((fp[1:] < fp[:-1]).any()):
        raise ValueError(f"frame_ptr must rise from 0 to the number of atoms ({n})")
    big = int((fp[1:] - fp[:-1]).max())
    if big > FRAMES_MAX_ATOMS:
        raise ValueError(f"neighbor_csr_frames takes frames of at most {FRAMES_MAX_ATOMS} atoms (got {big}); "
                         "use neighbor_csr or neighbor_list for large frames")
    pbc_t = _frames_pbc(pbc, B, "cpu")
    rows, _ = frames_geometry(cell, pbc_t, r_max, pos.dtype)  # refuses before any device work; _lib.nl_frames derives nimg
    prune = _prune_args(types, cutoffs, n, r_max, dev)
    rows = rows.to(dev)
    periodic = pbc_t.any(dim=1).view(B, 1, 1).to(dev)
    eye = torch.eye(3, dtype=torch.float64, device=dev).expand(B, 3, 3)
    inv = torch.where(periodic, torch.linalg.inv(torch.where(periodic, rows, eye)), torch.zeros_like(rows))
    row_ptr, nbr, shift = _lib.nl_frames(pos.contiguous(), fp.to(device=dev, dtype=torch.int32), rows.to(pos.dtype).contiguous(),
                                         inv.to(pos.dtype).contiguous(), pbc_t.to(device=dev, dtype=torch.int32), float(r_max))
    if prune is not None:
        return _prune(pos, row_ptr, nbr, shift, *prune)
    return _csr_of(row_ptr, nbr, r_max), shift
