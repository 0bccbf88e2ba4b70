"""Plain-torch restatement of the force-constant kernels (csrc/fc.cu, include/allegro_b200.h ab2_fc_*), on the CPU.

Lists are centre-sorted CSR (row_ptr [n+1], ctr / nbr [E]) with a row per atom; shifts [E,3] in the positions' dtype or
None.  Units u = 3 a + alpha, each two jobs (s = +1, then s = -1)."""
from __future__ import annotations

import torch


def prefix(counts: torch.Tensor) -> torch.Tensor:
    return torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(counts.to(torch.int64), 0)])


def centres(atoms, row_ptr, ctr, nbr, n):
    """-> (cptr [A+1], cen, coff, ea): C_j = sorted unique {j} u {ctr[z] : nbr[z] = j}; coff = the row's edge offset inside
    the cluster, ea = the cluster's edge count."""
    deg = (row_ptr[1:] - row_ptr[:-1]).long()
    cens, offs, eas = [], [], []
    for j in atoms.tolist():
        c = torch.unique(torch.cat([torch.tensor([j]), ctr[nbr == j].long()]))
        d = deg[c]
        cens.append(c)
        offs.append(torch.cumsum(d, 0) - d)
        eas.append(int(d.sum()))
    cptr = prefix(torch.tensor([c.numel() for c in cens], dtype=torch.int64))
    cat = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64)  # noqa: E731
    return cptr, cat(cens), cat(offs), torch.tensor(eas, dtype=torch.int64)


def columns(cptr, cen, row_ptr, nbr, n):
    """-> (fptr [A+1], col): per displaced atom the sorted unique centres of C_j and neighbours of their rows."""
    cols = []
    for a in range(cptr.shape[0] - 1):
        ks = cen[cptr[a]:cptr[a + 1]].long()
        parts = [ks] + [nbr[row_ptr[k]:row_ptr[k + 1]].long() for k in ks.tolist()]
        cols.append(torch.unique(torch.cat(parts)))
    fptr = prefix(torch.tensor([c.numel() for c in cols], dtype=torch.int64))
    return fptr, (torch.cat(cols) if cols else torch.zeros(0, dtype=torch.int64))


def unit_prefix(cptr, ea):
    """(Cp, Ep) [3A+1]: exclusive prefix sums of centres and edges over units."""
    return prefix((cptr[1:] - cptr[:-1]).repeat_interleave(3)), prefix(ea.repeat_interleave(3))


def gather(pos, shift, h, acc_dtype, atoms, cptr, cen, coff, ea, row_ptr, nbr, u0, u1):
    """-> (row_ptr_b, cen_b, ctr_b, nbr_b, vec_b) of the units [u0, u1).  vec in the positions' dtype: (pos[n] - pos[c])
    + shift, then + s h on axis alpha when [n = j] - [c = j] = +-1, rounded once to acc_dtype.  ``h`` is the step as the
    positions hold it."""
    Cp, Ep = unit_prefix(cptr, ea)
    Cb = int(2 * (Cp[u1] - Cp[u0]))
    rp, cb_, cz, nz, vz = [], [], [], [], []
    for u in range(u0, u1):
        a, alpha = u // 3, u % 3
        j = int(atoms[a])
        ks = cen[cptr[a]:cptr[a + 1]].long()
        for sigma, s in ((0, 1.0), (1, -1.0)):
            q0 = int(2 * (Cp[u] - Cp[u0])) + sigma * ks.numel()
            e0 = int(2 * (Ep[u] - Ep[u0])) + sigma * int(ea[a])
            for c, k in enumerate(ks.tolist()):
                z = torch.arange(int(row_ptr[k]), int(row_ptr[k + 1]))
                rp.append(e0 + int(coff[cptr[a] + c]))
                cb_.append(k)
                jn = nbr[z].long()
                cz.append(torch.full((z.numel(),), q0 + c, dtype=torch.int64))
                nz.append(Cb + jn)
                d = pos[jn] - pos[k]
                if shift is not None:
                    d = d + shift[z]
                dl = (jn == j).to(torch.int64) - int(k == j)
                step = torch.tensor(s * h, dtype=pos.dtype)
                d[:, alpha] = torch.where(dl > 0, d[:, alpha] + step, torch.where(dl < 0, d[:, alpha] - step, d[:, alpha]))
                vz.append(d)
    Eb = int(2 * (Ep[u1] - Ep[u0]))
    row_ptr_b = torch.tensor(rp + [Eb], dtype=torch.int64)
    vec = torch.cat(vz) if vz else torch.zeros(0, 3, dtype=pos.dtype)
    cat = lambda xs: torch.cat(xs) if xs else torch.zeros(0, dtype=torch.int64)  # noqa: E731
    return row_ptr_b, torch.tensor(cb_, dtype=torch.int64), cat(cz), cat(nz), vec.to(acc_dtype)


def fold(gvec, h, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, u0, u1):
    """-> {(p, alpha): [3] fp64} for the units [u0, u1): -(F+ - F-) * (1 / (2h)) of atom col[p], F_i = sum of gvec over the
    job's edges centred on i - sum over its edges with neighbour i."""
    Cp, Ep = unit_prefix(cptr, ea)
    g = gvec.double()
    out = {}
    for u in range(u0, u1):
        a, alpha = u // 3, u % 3
        ks = cen[cptr[a]:cptr[a + 1]].long()
        Ea = int(ea[a])
        ep = int(2 * (Ep[u] - Ep[u0]))
        # original edge id and cluster offset of every edge of the cluster
        zs = torch.cat([torch.arange(int(row_ptr[k]), int(row_ptr[k + 1])) for k in ks.tolist()]) if ks.numel() else torch.zeros(0, dtype=torch.int64)
        dg = g[ep:ep + Ea] - g[ep + Ea:ep + 2 * Ea]
        for p in range(int(fptr[a]), int(fptr[a + 1])):
            i = int(col[p])
            f = dg[ctr[zs].long() == i].sum(0) - dg[nbr[zs].long() == i].sum(0)
            out[(p, alpha)] = -f * (1.0 / (2.0 * h))
    return out
