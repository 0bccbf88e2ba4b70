"""fp64 CPU references for the force-constant tests: synthetic ragged lists, the oracle on the displacement clusters of
tests/fc_spec.py, central differences of the oracle's full-frame forces, and the oracle's Hessian rows by double autograd."""
from __future__ import annotations

import torch

import fc_spec
from allegro_b200 import data as D


def synthetic_list(seed: int, n: int, max_deg: int = 6, isolated: int = 2, dtype=torch.float64):
    """A ragged centre-sorted list over n atoms: random (asymmetric) rows, edges from an atom to its own images (nbr =
    ctr with a non-zero shift) and ``isolated`` atoms that are nobody's neighbour and have empty rows.
    -> (pos [n,3], row_ptr [n+1], ctr [E], nbr [E] int64, shift [E,3])."""
    g = torch.Generator().manual_seed(seed)
    iso = set(torch.randperm(n, generator=g)[:isolated].tolist()) if n > isolated else set()
    live = [i for i in range(n) if i not in iso]
    ctr, nbr = [], []
    for k in range(n):
        if k in iso or not live:
            continue
        deg = int(torch.randint(0, max_deg + 1, (1,), generator=g))
        for _ in range(deg):
            ctr.append(k)
            nbr.append(live[int(torch.randint(0, len(live), (1,), generator=g))])
    ctr_t, nbr_t = torch.tensor(ctr, dtype=torch.int64), torch.tensor(nbr, dtype=torch.int64)
    row_ptr = fc_spec.prefix(torch.bincount(ctr_t, minlength=n))
    pos = torch.randn(n, 3, generator=g, dtype=torch.float64).to(dtype) * 3
    shift = torch.randn(ctr_t.shape[0], 3, generator=g, dtype=torch.float64).to(dtype)
    shift[ctr_t != nbr_t] *= 0.0
    shift[ctr_t == nbr_t] += 4.0  # a self edge is to an image
    return pos, row_ptr, ctr_t, nbr_t, shift


def frame_list(pos, cell, pbc, r_list):
    """CPU list of a frame at r_list -> (row_ptr, ctr, nbr int64, shift_vec [E,3] fp64)."""
    ei, sh = D.neighbor_list(pos, r_list, cell, pbc)
    csr = D.build_csr(ei, pos.shape[0])
    if csr.perm is not None:
        sh = sh[csr.perm]
    sv = sh.double() @ cell.double() if cell is not None else torch.zeros(ei.shape[1], 3, dtype=torch.float64)
    return csr.row_ptr.long(), csr.ctr.long(), csr.nbr.long(), sv


def _gvec(oracle, types_b, ctr_b, nbr_b, vec_b, Cb):
    """d (sum of the batched centres' atomic energies) / d vec from the oracle with the edge vectors as the leaf."""
    m = getattr(oracle, "model", oracle)
    vec = vec_b.double().detach().requires_grad_(True)
    inp = {D.POSITIONS_KEY: torch.zeros(types_b.shape[0], 3, dtype=torch.float64), D.ATOM_TYPE_KEY: types_b, D.EDGE_INDEX_KEY: torch.stack([ctr_b, nbr_b]),
           "edge_vectors": vec, "edge_lengths": vec.norm(dim=-1)}
    with torch.enable_grad():
        e = m(inp)[D.PER_ATOM_ENERGY_KEY].reshape(-1)[:Cb]
        return torch.autograd.grad(e.sum(), vec)[0] if vec.shape[0] else torch.zeros_like(vec)


def cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, shift, atoms, h):
    """Dense force-constant rows [A,N,3,3] from the oracle evaluated on the displacement clusters alone (fc_spec plan,
    gather and fold, one unit at a time)."""
    n = pos.shape[0]
    cptr, cen, coff, ea = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    fptr, col = fc_spec.columns(cptr, cen, row_ptr, nbr, n)
    out = torch.zeros(atoms.shape[0], n, 3, 3, dtype=torch.float64)
    for u in range(3 * atoms.shape[0]):
        rp, cb, cz, nz, vb = fc_spec.gather(pos, shift, h, torch.float64, atoms, cptr, cen, coff, ea, row_ptr, nbr, u, u + 1)
        Cb = cb.shape[0]
        g = _gvec(oracle, torch.cat([types[cb], types]), cz, nz, vb, Cb)
        for (p, alpha), v in fc_spec.fold(g, h, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, u, u + 1).items():
            a = u // 3
            out[a, int(col[p]), alpha] = v
    return out


def full_forces(oracle, pos, cell, types, ctr, nbr, shift):
    """Oracle forces of the whole frame on a fixed list (the list at r_max + h holds every pair a displacement brings
    within r_max)."""
    vec0 = shift
    m = getattr(oracle, "model", oracle)
    p = pos.double().detach().requires_grad_(True)
    with torch.enable_grad():
        vec = p[nbr] - p[ctr] + vec0
        inp = {D.POSITIONS_KEY: p, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: torch.stack([ctr, nbr]), "edge_vectors": vec, "edge_lengths": vec.norm(dim=-1)}
        e = m(inp)[D.TOTAL_ENERGY_KEY].sum()
        return -torch.autograd.grad(e, p)[0]


def full_fd_blocks(oracle, pos, cell, types, ctr, nbr, shift, atoms, h):
    """-(F(r + h e) - F(r - h e)) / (2h) of the whole frame -> [A,N,3,3]."""
    n = pos.shape[0]
    out = torch.zeros(atoms.shape[0], n, 3, 3, dtype=torch.float64)
    for a, j in enumerate(atoms.tolist()):
        for alpha in range(3):
            fs = []
            for s in (1.0, -1.0):
                q = pos.double().clone()
                q[j, alpha] += s * h
                fs.append(full_forces(oracle, q, cell, types, ctr, nbr, shift))
            out[a, :, alpha, :] = -(fs[0] - fs[1]) / (2 * h)
    return out


def hessian_rows(oracle, pos, types, ctr, nbr, shift, atoms):
    """Rows d2E / dr_{j,alpha} dr of the oracle by double autograd (3 Hessian-vector products per atom) -> [A,N,3,3]."""
    m = getattr(oracle, "model", oracle)
    n = pos.shape[0]
    p = pos.double().detach().requires_grad_(True)
    out = torch.zeros(atoms.shape[0], n, 3, 3, dtype=torch.float64)
    with torch.enable_grad():
        vec = p[nbr] - p[ctr] + shift
        inp = {D.POSITIONS_KEY: p, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: torch.stack([ctr, nbr]), "edge_vectors": vec, "edge_lengths": vec.norm(dim=-1)}
        e = m(inp)[D.TOTAL_ENERGY_KEY].sum()
        (g,) = torch.autograd.grad(e, p, create_graph=True)
        for a, j in enumerate(atoms.tolist()):
            for alpha in range(3):
                (hv,) = torch.autograd.grad(g[j, alpha], p, retain_graph=True)
                out[a, :, alpha, :] = hv
    return out


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)
