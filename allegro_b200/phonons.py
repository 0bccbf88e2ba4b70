"""Harmonic force constants by finite displacements, as phonopy forms them, from local displacement clusters.

    fc = force_constants(model, pos, cell, atom_types, pbc=True, atoms=None, displacement=0.01, max_edges=None)
    fc.blocks[k][alpha][beta] = -(F+_{col[k],beta} - F-_{col[k],beta}) / (2h)  ~  d2E / dr_{atoms[a],alpha} dr_{col[k],beta}

Displacing atom j by +-h along alpha moves only the edges of the rows in C_j = {j} u {k : an edge of row k has neighbour
j}, each by s h e_alpha ([nbr = j] - [ctr = j]) (an edge from j to its own image does not move), and Allegro's energy is
a sum of per-centre terms that see only their own row.  So F(r + h e) - F(r - h e) is exactly the difference of the forces
of those rows alone: each displacement costs |C_j| rows instead of the whole frame (DESIGN.md section 4.9).  The list is
built at r_max + h, so every pair that comes within r_max under a displacement is in it, and the edges beyond r_max add
exact zeros.

The plan (C_j, the non-zero columns of each row, the batched jobs) and the fold of per-edge gradients into blocks are the
ab2_fc_* kernels (csrc/fc.cu); each chunk of jobs runs through the same per-edge pipeline as ``energy_and_forces``
(nn._pipeline.edge_energy_grad).  A displaced atom's blocks do not depend on the chunking or on the other displaced atoms:
bitwise for fp32 models, to rounding for fp64 models (their tensor-product adjoint adds with atomics).

    fc3 = third_order_force_constants(model, pos, cell, atom_types, pbc=True, atoms=None, displacement=0.03, max_edges=None)

gives phono3py's third-order constants the same way: a pair of displacements (j, alpha), (k, beta) changes the mixed
difference only through the rows of C_j n C_k, so each unit (j, k, alpha, beta) evaluates those rows alone, in four jobs
(ab2_fc3_* kernels, DESIGN.md section 4.10).

    hv = hessian_vector_product(model, pos, cell, atom_types, v, pbc=True)
    fc = analytic_force_constants(model, pos, cell, atom_types, pbc=True, atoms=None, max_edges=None)

are exact second derivatives instead: forward-mode differentiation of the fused force path (nn._hessian, DESIGN.md
section 4.11).  ``hessian_vector_product`` gives d2E/dr2 . v for the whole frame (no dense Hessian: Lanczos lowest modes,
dimer searches, Hessian-free normal modes of large cells); ``analytic_force_constants`` gives the blocks of
``force_constants`` with no step, no step error and Phi(j,i)_{alpha beta} = Phi(i,j)_{beta alpha} to rounding, each unit
(j, alpha) one job on the undisplaced rows of C_j with the edge tangent e_alpha ([nbr = j] - [ctr = j]).
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib
from . import data as D

# the kernels index edges with int32 (AB2 lists): one chunk holds at most this many edges
MAX_CHUNK_EDGES = (1 << 31) - 2


class ForceConstants:
    """Block-sparse force constants: row a (displaced atom ``atoms[a]``) holds the blocks ``blocks[row_ptr[a]:row_ptr[a+1]]``
    of the atoms ``col[row_ptr[a]:row_ptr[a+1]]`` (ascending).  Blocks are fp64 in the model's energy unit per length^2;
    the first index is the displaced atom (phonopy's convention)."""

    def __init__(self, atoms: torch.Tensor, row_ptr: torch.Tensor, col: torch.Tensor, blocks: torch.Tensor, num_atoms: int):
        self.atoms, self.row_ptr, self.col, self.blocks = atoms, row_ptr, col, blocks
        self.num_atoms = int(num_atoms)

    def dense(self) -> torch.Tensor:
        """[A,N,3,3] fp64: phonopy's force-constant array (its compact form when ``atoms`` lists the primitive atoms)."""
        A = self.atoms.shape[0]
        out = torch.zeros(A, self.num_atoms, 3, 3, dtype=torch.float64, device=self.blocks.device)
        rows = torch.repeat_interleave(torch.arange(A, device=self.blocks.device), self.row_ptr[1:] - self.row_ptr[:-1])
        out[rows, self.col] = self.blocks
        return out


def _fused(model, name: str):
    from .committee import Committee
    from .model.allegro_models import FusedAllegroEnergy

    inner = getattr(model, "model", model)
    if isinstance(inner, Committee) or not isinstance(inner, FusedAllegroEnergy):
        raise TypeError(f"{name} takes an AllegroModel or a FusedAllegroEnergy, got {type(model).__name__}")
    return inner


def _pbc3(pbc):
    return tuple(bool(p) for p in (pbc if not isinstance(pbc, bool) else (pbc,) * 3))


def _atoms(atoms, n: int) -> torch.Tensor:
    """-> the displaced atoms as a CPU int64 tensor, checked."""
    if atoms is None:
        return torch.arange(n, dtype=torch.int64)
    a = torch.as_tensor(atoms).detach().cpu()
    if a.dim() != 1 or a.dtype.is_floating_point or a.dtype.is_complex or a.dtype == torch.bool:
        raise ValueError(f"atoms must be a 1-D integer tensor, got {a.dtype} of shape {tuple(a.shape)}")
    a = a.to(torch.int64)
    if a.numel() and (int(a.min()) < 0 or int(a.max()) >= n):
        raise ValueError(f"atoms must lie in [0, {n})")
    if torch.unique(a).numel() != a.numel():
        raise ValueError("atoms must not repeat")
    return a


def edge_bytes(core) -> int:
    """Device bytes the per-edge pipeline allocates per edge of a chunk, counted from the model's widths (activations,
    their gradients, the batched list and edge vectors), with 50 % headroom for the per-centre tensors and the allocator."""
    es = torch.empty(0, dtype=core.dtype).element_size()
    ac = torch.empty(0, dtype=core.acc).element_size()
    hid = max([core.readout.dims[1]] + [ly["mlp"].dims[1] for ly in core.layers] + [core.S])
    tp = sum(ly["d_out"] * core.U for ly in core.layers)
    act = 2 * core.S * (core.L + 1) + 3 * core.nw * (core.L + 1) + 2 * tp + 4 * hid * (core.L + 2) + core.S_in
    return int(1.5 * (es * act + ac * (2 * core.D + 9) + 12))


def _default_max_edges(core, device) -> int:
    free, _ = torch.cuda.mem_get_info(device)
    return int(max(1, min(MAX_CHUNK_EDGES, free // 2 // edge_bytes(core))))


def force_constants(model, pos: torch.Tensor, cell: Optional[torch.Tensor], atom_types: torch.Tensor, pbc=True, atoms=None,
                    displacement: float = 0.01, max_edges: Optional[int] = None) -> ForceConstants:
    """Force constants of the displaced ``atoms`` (default: every atom) by central differences with step ``displacement``,
    equal to the full-frame finite difference up to rounding.  ``model``: an ``AllegroModel`` or ``FusedAllegroEnergy`` on a
    CUDA device (TypeError otherwise, a committee included).  ``pos`` [N,3] fp32 / fp64 and ``atom_types`` [N] on the
    device; ``cell`` [3,3] (needed, and regular, on every periodic axis) or None.  Displacements run in chunks of at most
    ``max_edges`` batched edges (default: half the free device memory over ``edge_bytes``)."""
    inner, h, pbc, atoms_h = _checked("force_constants", model, pos, cell, atom_types, pbc, atoms, displacement, max_edges)
    n = pos.shape[0]
    core = inner.core()
    dev = pos.device
    pos = pos.detach().contiguous()
    types_i32 = atom_types.to(torch.int32).contiguous()
    if cell is not None:
        cell = cell.detach().reshape(3, 3).to(device=dev, dtype=pos.dtype)
    from .calculator import prune_table

    cutoffs = prune_table(inner, h)
    prune = {} if cutoffs is None else dict(types=types_i32, cutoffs=cutoffs)
    csr, shift = D.neighbor_csr(pos, inner.r_max + h, cell, pbc, **prune)
    A = atoms_h.shape[0]
    atoms_d = atoms_h.to(dev)
    # the plan: C_j and its edge offsets, then the non-zero columns of every row
    cptr, cen, coff, ea = _lib.fc_centres(atoms_d, csr, n)
    fptr, col = _lib.fc_columns(cptr, cen, csr, n)
    blocks = torch.empty(col.shape[0], 3, 3, dtype=torch.float64, device=dev)
    # units u = 3 a + alpha, each two jobs (+h, -h) of m_a centres and E_a edges
    Cp = _lib._prefix((cptr[1:] - cptr[:-1]).repeat_interleave(3))
    Ep = _lib._prefix(ea.repeat_interleave(3))
    Cp_h, Ep_h = Cp.cpu(), Ep.cpu()
    cap = int(max_edges) if max_edges is not None else _default_max_edges(core, dev)
    unit_edges = 2 * (Ep_h[1:] - Ep_h[:-1])
    if unit_edges.numel() and int(unit_edges.max()) > cap:
        raise ValueError(f"max_edges = {cap} is below the {int(unit_edges.max())} edges of one displacement pair")
    hp = float(torch.tensor(h, dtype=pos.dtype))  # the step as the positions hold it
    gscale, pair = _energy_terms(inner, core, atom_types, dev)
    from .nn._pipeline import edge_energy_grad

    U = 3 * A
    u0 = 0
    while u0 < U:
        # the largest run of units whose jobs fit in cap edges
        u1 = int(torch.searchsorted(Ep_h, Ep_h[u0] + cap // 2, right=True)) - 1
        u1 = max(u0 + 1, min(u1, U))
        while u1 > u0 + 1 and int(2 * (Cp_h[u1] - Cp_h[u0])) + n > MAX_CHUNK_EDGES:  # batched centres and atoms index int32 too
            u1 = u0 + (u1 - u0) // 2
        Cb, Eb = int(2 * (Cp_h[u1] - Cp_h[u0])), int(2 * (Ep_h[u1] - Ep_h[u0]))
        if Eb == 0:
            # every cluster of the chunk is an isolated atom: zero gradients (energy_forces' E == 0 path)
            gvec = torch.zeros(0, 3, dtype=core.acc, device=dev)
        else:
            row_ptr_b, cen_b, ctr_b, nbr_b, vec_b = _lib.fc_gather(pos, shift, hp, core.acc, atoms_d, cptr, cen, coff, ea, csr, Cp, Ep,
                                                                   u0, u1, Cb, Eb)
            csr_b = D.EdgeCSR(Cb, ctr_b, nbr_b, row_ptr_b, None, csr.max_degree)
            types_b = torch.cat([types_i32[cen_b.long()], types_i32])
            _, _, _, gvec, _ = edge_energy_grad(core, inner._upstream, csr_b, vec_b, types_b, gscale[cen_b.long()], pair)
        _lib.fc_fold(gvec, hp, cptr, cen, coff, ea, csr, n, fptr, col, Ep, u0, u1, blocks)
        u0 = u1
    return ForceConstants(atoms_d, fptr, col.long(), blocks, n)


def _checked(name, model, pos, cell, atom_types, pbc, atoms, displacement, max_edges, max_atoms: int = _lib.FC_MAX_ATOMS):
    """The refusals shared by force_constants, third_order_force_constants and the analytic entry points (``displacement``
    None: no step), before any kernel runs -> (the fused model, the step h or None, pbc as three bools, the displaced
    atoms as a CPU int64 tensor)."""
    inner = _fused(model, name)
    if not torch.is_tensor(pos) or not pos.is_cuda or not torch.is_tensor(atom_types) or not atom_types.is_cuda:
        raise RuntimeError("allegro_b200: inputs must be CUDA tensors (no CPU fallback on the hot path)")
    h = None
    if displacement is not None:
        h = float(displacement)
        if not math.isfinite(h) or h <= 0.0:
            raise ValueError(f"displacement must be finite and > 0, got {displacement!r}")
    if pos.dim() != 2 or pos.shape[1] != 3 or pos.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"pos must be fp32 or fp64 [N,3], got {pos.dtype} of shape {tuple(pos.shape)}")
    n = pos.shape[0]
    if atom_types.dim() != 1 or atom_types.shape[0] != n or atom_types.dtype.is_floating_point or atom_types.dtype == torch.bool:
        raise ValueError(f"atom_types must be [N] = [{n}] integers, got {atom_types.dtype} of shape {tuple(atom_types.shape)}")
    if n < 1 or n > max_atoms:
        raise ValueError(f"{name} takes frames of 1 .. {max_atoms} atoms, got {n}")
    pbc = _pbc3(pbc)
    if any(pbc) and (cell is None or not D.is_regular_cell(cell)):
        raise ValueError("a periodic axis needs a regular cell (data.is_regular_cell)")
    atoms_h = _atoms(atoms, n)
    if max_edges is not None and not (1 <= int(max_edges) <= MAX_CHUNK_EDGES):
        raise ValueError(f"max_edges must lie in [1, {MAX_CHUNK_EDGES}], got {max_edges!r}")
    return inner, h, pbc, atoms_h


def _energy_terms(inner, core, atom_types, dev):
    """(per-centre energy scales in the accumulate dtype, the pair-potential term or None) as energy_forces takes them."""
    ss = inner.per_type_energy_scale_shift
    gscale = ss.scales[atom_types.long()].to(core.acc)
    pair = None
    if inner.pair_potential is not None:
        pair = (inner.pair_potential, inner.edge_norm.rmax_table.to(device=dev, dtype=core.acc))
    return gscale, pair


class ThirdOrderForceConstants:
    """Block-sparse third-order force constants.  Row a (displaced atom j = ``atoms[a]``) holds the pairs
    ``pair_ptr[a]:pair_ptr[a+1]`` with second atoms k = ``pair_col[p]`` (ascending); pair p holds the blocks
    ``blocks[row_ptr[p]:row_ptr[p+1]]`` of the atoms i = ``col[...]`` (ascending), blocks[t][alpha][beta][gamma] =
    Phi_{alpha beta gamma}(j, k, i) in fp64, the model's energy unit per length^3 (phono3py's index order)."""

    def __init__(self, atoms, pair_ptr, pair_col, row_ptr, col, blocks, num_atoms: int):
        self.atoms, self.pair_ptr, self.pair_col = atoms, pair_ptr, pair_col
        self.row_ptr, self.col, self.blocks = row_ptr, col, blocks
        self.num_atoms = int(num_atoms)

    def dense(self) -> torch.Tensor:
        """[A,N,N,3,3,3] fp64: phono3py's fc3 (its compact form when ``atoms`` lists the primitive atoms)."""
        A, N = self.atoms.shape[0], self.num_atoms
        dev = self.blocks.device
        out = torch.zeros(A, N, N, 3, 3, 3, dtype=torch.float64, device=dev)
        P = self.pair_col.shape[0]
        rows = torch.repeat_interleave(torch.arange(A, device=dev), self.pair_ptr[1:] - self.pair_ptr[:-1])
        of_t = torch.repeat_interleave(torch.arange(P, device=dev), self.row_ptr[1:] - self.row_ptr[:-1])
        out[rows[of_t], self.pair_col[of_t], self.col] = self.blocks
        return out


def third_order_force_constants(model, pos: torch.Tensor, cell: Optional[torch.Tensor], atom_types: torch.Tensor, pbc=True,
                                atoms=None, displacement: float = 0.03, max_edges: Optional[int] = None) -> ThirdOrderForceConstants:
    """Third-order force constants of the displaced ``atoms`` (default: every atom) by mixed central differences with step
    ``displacement`` (phono3py's default distance), equal to the full-frame mixed difference up to rounding:

        Phi_{alpha beta gamma}(j, k, i) = -(F++ - F+- - F-+ + F--)_{i,gamma} / (4 h^2)

    where F^{s1 s2} are the forces with atom j moved by s1 h e_alpha and atom k by s2 h e_beta.  The second atoms k of j
    are its harmonic columns (the atoms with C_j n C_k non-empty); each unit (j, k, alpha, beta) evaluates only the rows of
    C_j n C_k, in four jobs.  Arguments and refusals as ``force_constants``; a unit whose four jobs exceed ``max_edges``
    raises ValueError once the plan is known."""
    name = "third_order_force_constants"
    inner, h, pbc, atoms_h = _checked(name, model, pos, cell, atom_types, pbc, atoms, displacement, max_edges)
    n = pos.shape[0]
    core = inner.core()
    dev = pos.device
    pos = pos.detach().contiguous()
    types_i32 = atom_types.to(torch.int32).contiguous()
    if cell is not None:
        cell = cell.detach().reshape(3, 3).to(device=dev, dtype=pos.dtype)
    from .calculator import prune_table

    # two displacements can shorten a pair by 2h
    cutoffs = prune_table(inner, 2 * h)
    prune = {} if cutoffs is None else dict(types=types_i32, cutoffs=cutoffs)
    csr, shift = D.neighbor_csr(pos, inner.r_max + 2 * h, cell, pbc, **prune)
    atoms_d = atoms_h.to(dev)
    # the plan: the pairs of each displaced atom (its harmonic columns), C_j n C_k of each pair, and the pair's columns
    cptr, cen, _, _ = _lib.fc_centres(atoms_d, csr, n)
    pair_ptr, pair_col = _lib.fc_columns(cptr, cen, csr, n)
    Kptr, Ken, _, _ = _lib.fc_centres(torch.arange(n, dtype=torch.int64, device=dev), csr, n)
    pj = atoms_d.to(torch.int32).repeat_interleave(pair_ptr[1:] - pair_ptr[:-1])
    iptr, icen, ioff, pe = _lib.fc3_pairs(pj, pair_col, Kptr, Ken, csr)
    rptr, col = _lib.fc_columns(iptr, icen, csr, n)
    blocks = torch.empty(col.shape[0], 3, 3, 3, dtype=torch.float64, device=dev)
    # units u = 9 p + 3 alpha + beta, each four jobs of m_p centres and E_p edges
    P = pj.shape[0]
    Pe = _lib._prefix(pe)
    ip_h, Pe_h = iptr.cpu(), Pe.cpu()
    cap = int(max_edges) if max_edges is not None else _default_max_edges(core, dev)
    if P and 4 * int(pe.max()) > cap:
        raise ValueError(f"max_edges = {cap} is below the {4 * int(pe.max())} edges of one pair's four displacements")

    def start(pref, u):  # centres or edges of one job summed over the units before u
        p, r = divmod(u, 9)
        return 9 * int(pref[p]) + (r * int(pref[p + 1] - pref[p]) if p < P else 0)

    hp = float(torch.tensor(h, dtype=pos.dtype))  # the step as the positions hold it
    gscale, pair = _energy_terms(inner, core, atom_types, dev)
    from .nn._pipeline import edge_energy_grad

    U = 9 * P
    E9 = 9 * Pe_h
    u0 = 0
    while u0 < U:
        # the largest run of units whose jobs fit in cap edges
        target = start(Pe_h, u0) + cap // 4
        ph = int(torch.searchsorted(E9, target, right=True)) - 1
        if ph >= P:
            u1 = U
        else:
            e = int(Pe_h[ph + 1] - Pe_h[ph])
            u1 = 9 * ph + (8 if e == 0 else min(8, (target - int(E9[ph])) // e))
        u1 = max(u0 + 1, min(u1, U))
        while u1 > u0 + 1 and 4 * (start(ip_h, u1) - start(ip_h, u0)) + n > MAX_CHUNK_EDGES:  # batched centres and atoms index int32 too
            u1 = u0 + (u1 - u0) // 2
        Cb, Eb = 4 * (start(ip_h, u1) - start(ip_h, u0)), 4 * (start(Pe_h, u1) - start(Pe_h, u0))
        if Eb == 0:
            # every cluster of the chunk is an isolated atom: zero gradients
            gvec = torch.zeros(0, 3, dtype=core.acc, device=dev)
        else:
            row_ptr_b, cen_b, ctr_b, nbr_b, vec_b = _lib.fc3_gather(pos, shift, hp, core.acc, pj, pair_col, iptr, icen, ioff, Pe, csr,
                                                                    u0, u1, Cb, Eb)
            csr_b = D.EdgeCSR(Cb, ctr_b, nbr_b, row_ptr_b, None, csr.max_degree)
            types_b = torch.cat([types_i32[cen_b.long()], types_i32])
            _, _, _, gvec, _ = edge_energy_grad(core, inner._upstream, csr_b, vec_b, types_b, gscale[cen_b.long()], pair)
        _lib.fc3_fold(gvec, hp, iptr, icen, ioff, Pe, csr, n, rptr, col, u0, u1, blocks)
        u0 = u1
    return ThirdOrderForceConstants(atoms_d, pair_ptr, pair_col.long(), rptr, col.long(), blocks, n)


def _frame_list(inner, pos, cell, pbc, types_i32):
    """The device list at r_max (pruned to the per-edge-type cutoffs where the model has them) -> (csr, shift)."""
    from .calculator import prune_table

    cutoffs = prune_table(inner, 0.0)
    prune = {} if cutoffs is None else dict(types=types_i32, cutoffs=cutoffs)
    return D.neighbor_csr(pos, inner.r_max, cell, pbc, **prune)


def hessian_vector_product(model, pos: torch.Tensor, cell: Optional[torch.Tensor], atom_types: torch.Tensor, v: torch.Tensor,
                           pbc=True) -> torch.Tensor:
    """d2E/dr2 . v [N,3] for the whole frame, exact to rounding (forward mode over the fused force path, no step), in the
    model's accumulate dtype.  ``v`` [N,3] floating on the device; the edge tangents are v[nbr] - v[ctr], so an edge from an
    atom to its own image does not move.  Arguments and refusals as ``force_constants`` (without its atom limit); a ``v``
    that is not a floating [N,3] device tensor raises ValueError.  A frame without edges gives zeros."""
    name = "hessian_vector_product"
    inner, _, pbc, _ = _checked(name, model, pos, cell, atom_types, pbc, None, None, None, max_atoms=(1 << 31) - 1)
    n = pos.shape[0]
    if (not torch.is_tensor(v) or not v.is_cuda or v.device != pos.device or not v.dtype.is_floating_point or v.dim() != 2
            or tuple(v.shape) != (n, 3)):
        desc = f"{v.dtype} of shape {tuple(v.shape)} on {v.device}" if torch.is_tensor(v) else type(v).__name__
        raise ValueError(f"v must be a floating [N,3] = [{n},3] tensor on {pos.device}, got {desc}")
    core = inner.core()
    dev = pos.device
    pos = pos.detach().contiguous()
    types_i32 = atom_types.to(torch.int32).contiguous()
    if cell is not None:
        cell = cell.detach().reshape(3, 3).to(device=dev, dtype=pos.dtype)
    csr, shift = _frame_list(inner, pos, cell, pbc, types_i32)
    if csr.num_edges == 0:
        return torch.zeros(n, 3, dtype=core.acc, device=dev)
    vec = _lib.edge_vec(pos, csr.ctr, csr.nbr, shift, core.acc)
    vdot = _lib.edge_vec(v.detach().to(core.acc).contiguous(), csr.ctr, csr.nbr, None, core.acc)
    gscale, pair = _energy_terms(inner, core, atom_types, dev)
    from .nn._hessian import edge_energy_grad_tangent

    _, gvec_dot = edge_energy_grad_tangent(core, inner._upstream, csr, vec, vdot, types_i32, gscale, pair)
    return -_lib.force_scatter(gvec_dot, csr, n)


def analytic_force_constants(model, pos: torch.Tensor, cell: Optional[torch.Tensor], atom_types: torch.Tensor, pbc=True, atoms=None,
                             max_edges: Optional[int] = None) -> ForceConstants:
    """The force constants of ``force_constants`` (same ``ForceConstants`` layout, phonopy's convention) as exact second
    derivatives: each unit (displaced atom j, axis alpha) is one tangent job on the undisplaced rows of C_j, folded
    without a step.  The plan is that of ``force_constants`` on a list built at r_max exactly.  Arguments and refusals as
    ``force_constants`` without ``displacement``; chunks of at most ``max_edges`` batched edges (default: half the free
    device memory over ``nn._hessian.hvp_edge_bytes``).  A displaced atom's blocks do not depend on the chunking or on the
    other displaced atoms: bitwise for fp32 models, to rounding for fp64 models."""
    name = "analytic_force_constants"
    inner, _, pbc, atoms_h = _checked(name, model, pos, cell, atom_types, pbc, atoms, None, max_edges)
    n = pos.shape[0]
    core = inner.core()
    dev = pos.device
    pos = pos.detach().contiguous()
    types_i32 = atom_types.to(torch.int32).contiguous()
    if cell is not None:
        cell = cell.detach().reshape(3, 3).to(device=dev, dtype=pos.dtype)
    csr, shift = _frame_list(inner, pos, cell, pbc, types_i32)
    A = atoms_h.shape[0]
    atoms_d = atoms_h.to(dev)
    cptr, cen, coff, ea = _lib.fc_centres(atoms_d, csr, n)
    fptr, col = _lib.fc_columns(cptr, cen, csr, n)
    blocks = torch.empty(col.shape[0], 3, 3, dtype=torch.float64, device=dev)
    # units u = 3 a + alpha, each ONE job of m_a centres and E_a edges
    Cp = _lib._prefix((cptr[1:] - cptr[:-1]).repeat_interleave(3))
    Ep = _lib._prefix(ea.repeat_interleave(3))
    Cp_h, Ep_h = Cp.cpu(), Ep.cpu()
    from .nn._hessian import edge_energy_grad_tangent, hvp_edge_bytes

    if max_edges is not None:
        cap = int(max_edges)
    else:
        free, _ = torch.cuda.mem_get_info(dev)
        cap = int(max(1, min(MAX_CHUNK_EDGES, free // 2 // hvp_edge_bytes(core))))
    unit_edges = Ep_h[1:] - Ep_h[:-1]
    if unit_edges.numel() and int(unit_edges.max()) > cap:
        raise ValueError(f"max_edges = {cap} is below the {int(unit_edges.max())} edges of one displaced atom's cluster")
    gscale, pair = _energy_terms(inner, core, atom_types, dev)
    U = 3 * A
    u0 = 0
    while u0 < U:
        # the largest run of units whose jobs fit in cap edges
        u1 = int(torch.searchsorted(Ep_h, Ep_h[u0] + cap, right=True)) - 1
        u1 = max(u0 + 1, min(u1, U))
        while u1 > u0 + 1 and int(Cp_h[u1] - Cp_h[u0]) + n > MAX_CHUNK_EDGES:  # batched centres and atoms index int32 too
            u1 = u0 + (u1 - u0) // 2
        Cb, Eb = int(Cp_h[u1] - Cp_h[u0]), int(Ep_h[u1] - Ep_h[u0])
        if Eb == 0:
            # every cluster of the chunk is an isolated atom: zero blocks
            gvec_dot = torch.zeros(0, 3, dtype=core.acc, device=dev)
        else:
            row_ptr_b, cen_b, ctr_b, nbr_b, vec_b, vdot_b = _lib.fc_gather_tangent(pos, shift, core.acc, atoms_d, cptr, cen, coff, ea, csr, Cp, Ep,
                                                                                   u0, u1, Cb, Eb)
            csr_b = D.EdgeCSR(Cb, ctr_b, nbr_b, row_ptr_b, None, csr.max_degree)
            types_b = torch.cat([types_i32[cen_b.long()], types_i32])
            _, gvec_dot = edge_energy_grad_tangent(core, inner._upstream, csr_b, vec_b, vdot_b, types_b, gscale[cen_b.long()], pair)
        _lib.fc_fold_tangent(gvec_dot, cptr, cen, coff, ea, csr, n, fptr, col, Ep, u0, u1, blocks)
        u0 = u1
    return ForceConstants(atoms_d, fptr, col.long(), blocks, n)
