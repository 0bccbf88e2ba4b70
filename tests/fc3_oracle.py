"""fp64 CPU references for the third-order force-constant tests: the oracle on the pair clusters of tests/fc3_spec.py,
mixed central differences of the oracle's full-frame forces, and the oracle's third derivatives by triple autograd.
Every function takes the pairs (pj, pk) to evaluate and returns [P,N,3,3,3]: [p, i, alpha, beta, gamma]."""
from __future__ import annotations

import torch

import fc3_spec
import fc_spec
from fc_oracle import _gvec, full_forces
from allegro_b200 import data as D


def cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, shift, pj, pk, h):
    """The blocks of the pairs from the oracle evaluated on C_j n C_k alone (fc3_spec plan, gather and fold, one unit at a
    time)."""
    n = pos.shape[0]
    iptr, icen, ioff, pe = fc3_spec.intersections(pj, pk, row_ptr, ctr, nbr, n)
    rptr, col = fc_spec.columns(iptr, icen, row_ptr, nbr, n)
    out = torch.zeros(pj.shape[0], n, 3, 3, 3, dtype=torch.float64)
    for u in range(9 * pj.shape[0]):
        rp, cb, cz, nz, vb = fc3_spec.gather(pos, shift, h, torch.float64, pj, pk, iptr, icen, ioff, pe, row_ptr, nbr, u, u + 1)
        g = _gvec(oracle, torch.cat([types[cb], types]), cz, nz, vb, cb.shape[0])
        for (t, alpha, beta), v in fc3_spec.fold(g, h, iptr, icen, ioff, pe, row_ptr, ctr, nbr, rptr, col, u, u + 1).items():
            out[u // 9, int(col[t]), alpha, beta] = v
    return out


def full_fd_blocks(oracle, pos, types, ctr, nbr, shift, pj, pk, h):
    """-(F++ - F+- - F-+ + F--) / (4h^2) of the whole frame on a fixed list."""
    out = torch.zeros(pj.shape[0], pos.shape[0], 3, 3, 3, dtype=torch.float64)
    for p, (j, k) in enumerate(zip(pj.tolist(), pk.tolist())):
        for alpha in range(3):
            for beta in range(3):
                fs = []
                for s1, s2 in fc3_spec.SIGNS:
                    q = pos.double().clone()
                    q[j, alpha] += s1 * h
                    q[k, beta] += s2 * h
                    fs.append(full_forces(oracle, q, None, types, ctr, nbr, shift))
                out[p, :, alpha, beta] = -((fs[0] + fs[3]) - (fs[1] + fs[2])) / (4 * h * h)
    return out


def third_derivatives(oracle, pos, types, ctr, nbr, shift, pj, pk):
    """d3E / dr_{j,alpha} dr_{k,beta} dr_{i,gamma} of the oracle by triple autograd (a gradient of each Hessian-vector
    product taken with create_graph)."""
    m = getattr(oracle, "model", oracle)
    n = pos.shape[0]
    p = pos.double().detach().requires_grad_(True)
    out = torch.zeros(pj.shape[0], n, 3, 3, 3, dtype=torch.float64)
    with torch.enable_grad():
        vec = p[nbr] - p[ctr] + shift
        inp = {D.POSITIONS_KEY: p, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: torch.stack([ctr, nbr]), "edge_vectors": vec, "edge_lengths": vec.norm(dim=-1)}
        e = m(inp)[D.TOTAL_ENERGY_KEY].sum()
        (g,) = torch.autograd.grad(e, p, create_graph=True)
        for j in sorted(set(pj.tolist())):
            for alpha in range(3):
                (hv,) = torch.autograd.grad(g[j, alpha], p, retain_graph=True, create_graph=True)
                for q, k in enumerate(pk.tolist()):
                    if int(pj[q]) != j:
                        continue
                    for beta in range(3):
                        (tv,) = torch.autograd.grad(hv[k, beta], p, retain_graph=True)
                        out[q, :, alpha, beta] = tv
    return out

