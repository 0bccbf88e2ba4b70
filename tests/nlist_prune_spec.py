"""Torch restatement of ab2_nl_prune_count / fill (include/allegro_b200.h), the signature of ``_lib.nl_prune``, and the
helpers the pruning tests share.  The restatement runs on the device of its inputs with the same fp64 operations in the
same order as the kernel (no contraction: torch launches each elementwise operation on its own), so the GPU test holds the
kernel to it bit for bit."""
from __future__ import annotations

import numpy as np
import torch


def nl_prune(pos, row_ptr, nbr, shift, types, cut2):
    nc, E = row_ptr.shape[0] - 1, nbr.shape[0]
    if nc == 0 or E == 0:
        return row_ptr.clone(), nbr.clone(), shift.clone()
    dev = pos.device
    counts = (row_ptr[1:] - row_ptr[:-1]).long()
    ctr = torch.repeat_interleave(torch.arange(nc, device=dev), counts)
    j = nbr.long()
    p, s = pos.double(), shift.double()
    d = (p[j] + s) - p[ctr]
    d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
    d2 = d2 + d[:, 2] * d[:, 2]
    t = types.long()
    T = cut2.shape[0]
    keep = d2 < cut2.reshape(-1)[t[ctr] * T + t[j]]
    out_ptr = torch.zeros(nc + 1, dtype=torch.int32, device=dev)
    out_ptr[1:] = torch.cumsum(torch.bincount(ctr[keep], minlength=nc), 0).to(torch.int32)
    return out_ptr, nbr[keep].contiguous(), shift[keep].contiguous()


def random_table(T: int, r_max: float, seed: int) -> torch.Tensor:
    """A directed [T,T] fp64 table with entries in [0.4, 1.0] r_max, some exactly r_max (the diagonal's first entry and
    one off-diagonal entry), asymmetric whenever T > 1."""
    g = torch.Generator().manual_seed(seed)
    tab = r_max * (0.4 + 0.6 * torch.rand(T, T, generator=g, dtype=torch.float64))
    tab[0, 0] = r_max
    if T > 1:
        tab[T - 1, 0] = r_max
    return tab


def random_types(n: int, T: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, T, (n,), generator=g)


def is_ordered_subsequence(row_ptr, nbr, shift, row_ptr_p, nbr_p, shift_p) -> bool:
    """Every pruned row is an ordered subsequence of the unpruned row, (nbr, shift) compared bitwise."""
    rp, rpp = row_ptr.cpu().tolist(), row_ptr_p.cpu().tolist()
    a = torch.cat([nbr.cpu().double().view(-1, 1), shift.cpu().double()], 1).numpy()
    b = torch.cat([nbr_p.cpu().double().view(-1, 1), shift_p.cpu().double()], 1).numpy()
    for i in range(len(rp) - 1):
        k = rp[i]
        for z in range(rpp[i], rpp[i + 1]):
            while k < rp[i + 1] and not np.array_equal(a[k], b[z]):
                k += 1
            if k == rp[i + 1]:
                return False
            k += 1
    return True


def compare_pruned(got_rows, ref_rows, ref_dist, types, table, band: float, n: int):
    """Kept (i, j, s0, s1, s2) rows against the fp64 reference pairs (every pair within r_max + band): a pair more than
    ``band`` inside its own cutoff table[t_i, t_j] must be kept once, a pair more than ``band`` beyond it must not be kept.
    -> (pairs inside the band of their own cutoff, of which kept)."""
    from nlist_oracle import keys

    got_rows, ref_rows = np.asarray(got_rows, dtype=np.int64).reshape(-1, 5), np.asarray(ref_rows, dtype=np.int64).reshape(-1, 5)
    t = np.asarray(types, dtype=np.int64)
    tab = np.asarray(table, dtype=np.float64)
    cut = tab[t[ref_rows[:, 0]], t[ref_rows[:, 1]]] if ref_rows.size else np.zeros(0)
    g = keys(got_rows, n)
    ug, cnt = np.unique(g, return_counts=True)
    assert (cnt == 1).all(), "duplicate rows"
    rk = keys(ref_rows, n)
    ref_dist = np.asarray(ref_dist)
    must = rk[ref_dist < cut - band]
    may = rk[ref_dist < cut + band]
    missing = must[~np.isin(must, ug)]
    assert missing.size == 0, f"{missing.size} pairs inside their own cutoff were dropped"
    extra = ug[~np.isin(ug, may)]
    assert extra.size == 0, f"{extra.size} kept pairs are beyond their own cutoff (or not pairs at all)"
    in_band = rk[np.abs(ref_dist - cut) <= band]
    return int(in_band.size), int(np.isin(in_band, ug).sum())
