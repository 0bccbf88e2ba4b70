"""Plain-torch restatement of the third-order force-constant kernels (csrc/fc.cu, include/allegro_b200.h ab2_fc3_*), on
the CPU.

Lists as in tests/fc_spec.py.  Pairs p = (pj[p], pk[p]) of displaced atoms; units u = 9 p + 3 alpha + beta, each four jobs
sigma = 0..3 with (s1, s2) = (+,+), (+,-), (-,+), (-,-)."""
from __future__ import annotations

import torch

import fc_spec

SIGNS = ((1.0, 1.0), (1.0, -1.0), (-1.0, 1.0), (-1.0, -1.0))


def pairs(atoms, row_ptr, ctr, nbr, n):
    """-> (pair_ptr [A+1], pair_col): the second atoms of each displaced atom are its harmonic columns."""
    cptr, cen, _, _ = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    return fc_spec.columns(cptr, cen, row_ptr, nbr, n)


def intersections(pj, pk, row_ptr, ctr, nbr, n):
    """-> (iptr [P+1], icen, ioff, pe): C_j n C_k ascending, each centre's row offset inside the pair's cluster, and the
    cluster's edge count, from the centre sets of every atom."""
    Kptr, Ken, _, _ = fc_spec.centres(torch.arange(n), row_ptr, ctr, nbr, n)
    deg = (row_ptr[1:] - row_ptr[:-1]).long()
    cens, offs, pes = [], [], []
    for j, k in zip(pj.tolist(), pk.tolist()):
        cj = set(Ken[Kptr[j]:Kptr[j + 1]].tolist())
        c = torch.tensor(sorted(cj & set(Ken[Kptr[k]:Kptr[k + 1]].tolist())), dtype=torch.int64)
        d = deg[c]
        cens.append(c)
        offs.append(torch.cumsum(d, 0) - d)
        pes.append(int(d.sum()))
    iptr = fc_spec.prefix(torch.tensor([c.numel() for c in cens], dtype=torch.int64))
    cat = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64)  # noqa: E731
    return iptr, cat(cens), cat(offs), torch.tensor(pes, dtype=torch.int64)


def unit_prefix(iptr, pe):
    """(Cp, Ep) [9P+1]: exclusive prefix sums of one job's centres and edges over units."""
    return fc_spec.prefix((iptr[1:] - iptr[:-1]).repeat_interleave(9)), fc_spec.prefix(pe.repeat_interleave(9))


def gather(pos, shift, h, acc_dtype, pj, pk, iptr, icen, ioff, pe, row_ptr, nbr, u0, u1):
    """-> (row_ptr_b, cen_b, ctr_b, nbr_b, vec_b) of the units [u0, u1).  vec in the positions' dtype: (pos[n] - pos[c])
    + shift, then + delta, delta_x = [x = alpha] s1 h ([n = j] - [c = j]) + [x = beta] s2 h ([n = k] - [c = k]) (exact),
    rounded once to acc_dtype.  ``h`` is the step as the positions hold it."""
    Cp, Ep = unit_prefix(iptr, pe)
    Cb = int(4 * (Cp[u1] - Cp[u0]))
    rp, cb_, cz, nz, vz = [], [], [], [], []
    for u in range(u0, u1):
        p, alpha, beta = u // 9, (u // 3) % 3, u % 3
        j, k = int(pj[p]), int(pk[p])
        ks = icen[iptr[p]:iptr[p + 1]].long()
        for sigma, (s1, s2) in enumerate(SIGNS):
            q0 = int(4 * (Cp[u] - Cp[u0])) + sigma * ks.numel()
            e0 = int(4 * (Ep[u] - Ep[u0])) + sigma * int(pe[p])
            for c, kc in enumerate(ks.tolist()):
                z = torch.arange(int(row_ptr[kc]), int(row_ptr[kc + 1]))
                rp.append(e0 + int(ioff[iptr[p] + c]))
                cb_.append(kc)
                jn = nbr[z].long()
                cz.append(torch.full((z.numel(),), q0 + c, dtype=torch.int64))
                nz.append(Cb + jn)
                d = pos[jn] - pos[kc]
                if shift is not None:
                    d = d + shift[z]
                dj = ((jn == j).to(torch.int64) - int(kc == j)).to(pos.dtype)
                dk = ((jn == k).to(torch.int64) - int(kc == k)).to(pos.dtype)
                t1 = torch.tensor(s1 * h, dtype=pos.dtype)
                t2 = torch.tensor(s2 * h, dtype=pos.dtype)
                zero = torch.zeros_like(dj)
                delta = torch.stack([(dj * t1 if x == alpha else zero) + (dk * t2 if x == beta else zero) for x in range(3)], 1)
                vz.append(d + delta)
    Eb = int(4 * (Ep[u1] - Ep[u0]))
    row_ptr_b = torch.tensor(rp + [Eb], dtype=torch.int64)
    vec = torch.cat(vz) if vz else torch.zeros(0, 3, dtype=pos.dtype)
    cat = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64)  # noqa: E731
    return row_ptr_b, torch.tensor(cb_, dtype=torch.int64), cat(cz), cat(nz), vec.to(acc_dtype)


def fold(gvec, h, iptr, icen, ioff, pe, row_ptr, ctr, nbr, rptr, col, u0, u1):
    """-> {(t, alpha, beta): [3] fp64} for the units [u0, u1): -((F++ + F--) - (F+- + F-+)) * (1 / (4h^2)) of atom col[t],
    F_i = sum of gvec over the job's edges centred on i - sum over its edges with neighbour i."""
    Cp, Ep = unit_prefix(iptr, pe)
    g = gvec.double()
    out = {}
    for u in range(u0, u1):
        p, alpha, beta = u // 9, (u // 3) % 3, u % 3
        ks = icen[iptr[p]:iptr[p + 1]].long()
        Ez = int(pe[p])
        e0 = int(4 * (Ep[u] - Ep[u0]))
        zs = torch.cat([torch.arange(int(row_ptr[k]), int(row_ptr[k + 1])) for k in ks.tolist()]) if ks.numel() else torch.zeros(0, dtype=torch.int64)
        gj = [g[e0 + s * Ez:e0 + (s + 1) * Ez] for s in range(4)]
        dg = (gj[0] + gj[3]) - (gj[1] + gj[2])
        for t in range(int(rptr[p]), int(rptr[p + 1])):
            i = int(col[t])
            f = dg[ctr[zs].long() == i].sum(0) - dg[nbr[zs].long() == i].sum(0)
            out[(t, alpha, beta)] = -f * (1.0 / (4.0 * h * h))
    return out
