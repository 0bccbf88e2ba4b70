"""fp64 pair search in plain numpy for any non-singular cell rows and per-axis periodicity: the reference the
general-lattice neighbour list is held to.

It shares no code with ``allegro_b200``: fractional coordinates are solved for (pos = frac . rows), periodic axes are
wrapped with img0 = floor(frac), and every image n with |n_a| <= ceil((r_max + reach) / H_a) on each periodic axis
(H_a = |det| / |row_p x row_q|, the height of the cell along a) is tried against every atom.  Pairs come out as
(i, j, s0, s1, s2) with s = n - img0[j] + img0[i], so that  r = pos[j] + s . rows - pos[i]  holds for the RAW positions,
together with that distance in fp64.  Keys, the comparison and the band are those of nlist_oracle.
"""
from __future__ import annotations

import math

import numpy as np

from nlist_oracle import band_for as _band_for
from nlist_oracle import compare, keys  # noqa: F401  (re-exported for the lattice tests)


def complete(rows, pbc):
    """Rows with the open axes replaced by an orthonormal basis of the complement of the periodic rows (numpy SVD)
    when the given rows are singular: zero rows of ASE's 2-D / 1-D cells, or no cell at all (None)."""
    pbc = [bool(p) for p in pbc]
    h = np.zeros((3, 3)) if rows is None else np.array(rows, dtype=np.float64).reshape(3, 3)
    if abs(np.linalg.det(h)) > 1e-9 * np.prod(np.linalg.norm(h, axis=1)):
        return h
    per = [a for a in range(3) if pbc[a]]
    opn = [a for a in range(3) if not pbc[a]]
    if per:
        _, _, vt = np.linalg.svd(h[per], full_matrices=True)
        comp = vt[len(per):]
    else:
        comp = np.eye(3)
    h = h.copy()
    for k, a in enumerate(opn):
        h[a] = comp[k]
    assert abs(np.linalg.det(h)) > 0, "periodic rows are singular"
    return h


def heights(rows):
    h = np.asarray(rows, dtype=np.float64).reshape(3, 3)
    vol = abs(np.linalg.det(h))
    return np.array([vol / np.linalg.norm(np.cross(h[(a + 1) % 3], h[(a + 2) % 3])) for a in range(3)])


def band_for(pos, rows, r_max, fp32: bool) -> float:
    return _band_for(pos, np.linalg.norm(np.asarray(rows, dtype=np.float64).reshape(3, 3), axis=1), r_max, fp32)


def pairs(pos, rows, pbc, r_max: float, centres=None, reach: float = 0.0):
    """-> (rows [P,5] int64 = (i, j, s0, s1, s2), dist [P] fp64) of every pair with |pos[j] + s . rows - pos[i]| <
    r_max + reach.  ``rows`` non-singular [3,3] (lattice vectors as rows), ``pos`` the exact values the search saw."""
    pos = np.asarray(pos, dtype=np.float64).reshape(-1, 3)
    h = np.asarray(rows, dtype=np.float64).reshape(3, 3)
    pbc = np.asarray([bool(p) for p in pbc])
    n = pos.shape[0]
    centres = np.arange(n) if centres is None else np.asarray(centres, dtype=np.int64)
    if n == 0 or centres.size == 0:
        return np.zeros((0, 5), dtype=np.int64), np.zeros(0)
    cut = float(r_max) + float(reach)
    frac = np.linalg.solve(h.T, pos.T).T
    img0 = np.where(pbc, np.floor(frac), 0.0).astype(np.int64)
    wrapped = pos - img0 @ h
    H = heights(h)
    reps = [int(math.ceil(cut / H[a])) if pbc[a] else 0 for a in range(3)]
    imgs = np.stack(np.meshgrid(*[np.arange(-r, r + 1) for r in reps], indexing="ij"), -1).reshape(-1, 3)
    off = imgs @ h  # [M,3]
    out_rows, dists = [], []
    chunk = max(1, 4_000_000 // (n * imgs.shape[0]))
    for c0 in range(0, centres.size, chunk):
        ci = centres[c0 : c0 + chunk]
        d = wrapped[None, :, None, :] + off[None, None, :, :] - wrapped[ci, None, None, :]
        r = np.sqrt((d * d).sum(-1))
        sel = np.nonzero(r < cut + 1e-6 * cut)
        i, j, m = ci[sel[0]], sel[1], sel[2]
        s = imgs[m] - img0[j] + img0[i]
        v = pos[j] + s @ h - pos[i]
        dist = np.sqrt((v * v).sum(-1))
        keep = (dist < cut) & ~((i == j) & (s == 0).all(-1))
        out_rows.append(np.concatenate([i[keep, None], j[keep, None], s[keep]], 1))
        dists.append(dist[keep])
    return np.concatenate(out_rows, 0).astype(np.int64), np.concatenate(dists, 0)


def images_of(shift, rows):
    """Integer image coefficients of shift vectors [E,3] in the basis ``rows`` -> (coefficients [E,3] int64, largest
    deviation of coefficients . rows from the shifts)."""
    h = np.asarray(rows, dtype=np.float64).reshape(3, 3)
    shift = np.asarray(shift, dtype=np.float64).reshape(-1, 3)
    c = np.rint(np.linalg.solve(h.T, shift.T).T).astype(np.int64)
    dev = np.abs(c @ h - shift).max() if shift.size else 0.0
    return c, float(dev)
