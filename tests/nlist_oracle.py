"""fp64 pair search in plain numpy: the reference every neighbour list of the package is held to.

It shares no code with ``allegro_b200.data``: positions are wrapped with img0 = floor((pos - origin) / L) on the periodic
axes of an orthorhombic box, every image offset n in [-ceil(r/L), ceil(r/L)] of each periodic axis is tried against every
atom, and pairs come out as (i, j, s) with s = n - img0[j] + img0[i], so that  r = pos[j] + s * L - pos[i]  holds for
the RAW positions (the package's convention), together with that distance in fp64.

Pairs whose distance is within ``band`` of r_max may be present or absent (an fp32 search cannot decide them); every
other pair must match exactly.  ``band`` is 1e-10 (fp64 positions) or 1e-6 (fp32 positions) of the largest length in
the problem: r_max, max |pos| or max L.
"""
from __future__ import annotations

import math

import numpy as np

_S_OFF = 1 << 8  # shift components are packed in 9 bits each (|s| < 256), the pair in 36 (n < 2^18)


def band_for(pos, box, r_max, fp32: bool) -> float:
    pos = np.asarray(pos, dtype=np.float64)
    scale = max(float(r_max), float(np.abs(pos).max()) if pos.size else 0.0, float(np.max(np.asarray(box, dtype=np.float64))))
    return (1e-6 if fp32 else 1e-10) * scale


def pairs(pos, box, pbc, r_max: float, centres=None, reach: float = 0.0):
    """-> (rows [P,5] int64 = (i, j, s0, s1, s2), dist [P] fp64) of every pair with |pos[j] + s*L - pos[i]| < r_max + reach.
    ``pos`` are the exact values the search saw (fp32-rounded when it ran in fp32), ``box`` the orthorhombic lengths,
    ``centres`` an optional subset of centre indices."""
    pos = np.asarray(pos, dtype=np.float64).reshape(-1, 3)
    box = np.asarray(box, dtype=np.float64).reshape(3)
    pbc = np.asarray([bool(p) for p in pbc])
    n = pos.shape[0]
    centres = np.arange(n) if centres is None else np.asarray(centres, dtype=np.int64)
    cut = float(r_max) + float(reach)
    img0 = np.zeros((n, 3), dtype=np.int64)
    L = np.where(pbc, box, 1.0)
    img0[:, pbc] = np.floor(pos[:, pbc] / L[pbc]).astype(np.int64)
    wrapped = pos - img0 * np.where(pbc, box, 0.0)
    reps = [int(math.ceil(cut / box[a])) if pbc[a] else 0 for a in range(3)]
    imgs = np.stack(np.meshgrid(*[np.arange(-r, r + 1) for r in reps], indexing="ij"), -1).reshape(-1, 3)
    off = imgs * np.where(pbc, box, 0.0)  # [M,3]
    rows, dists = [], []
    if n == 0 or centres.size == 0:
        return np.zeros((0, 5), dtype=np.int64), np.zeros(0)
    chunk = max(1, 4_000_000 // (n * imgs.shape[0]))
    for c0 in range(0, centres.size, chunk):
        ci = centres[c0 : c0 + chunk]
        # [C, N, M] distances between wrapped centre i and image n of wrapped atom j: only used to select candidates
        d = wrapped[None, :, None, :] + off[None, None, :, :] - wrapped[ci, None, None, :]
        r = np.sqrt((d * d).sum(-1))
        sel = np.nonzero(r < cut + 1e-6 * cut)
        i, j, m = ci[sel[0]], sel[1], sel[2]
        s = imgs[m] - img0[j] + img0[i]
        # the distance the consumers see: raw positions plus the shift
        v = pos[j] + s * np.where(pbc, box, 0.0) - pos[i]
        dist = np.sqrt((v * v).sum(-1))
        keep = (dist < cut) & ~((i == j) & (s == 0).all(-1))
        rows.append(np.concatenate([i[keep, None], j[keep, None], s[keep]], 1))
        dists.append(dist[keep])
    return np.concatenate(rows, 0).astype(np.int64), np.concatenate(dists, 0)


def keys(rows, n: int) -> np.ndarray:
    """(i, j, s) rows -> one int64 per row (|s| < 256, n < 2^18)."""
    rows = np.asarray(rows, dtype=np.int64).reshape(-1, 5)
    assert n < (1 << 18) and (np.abs(rows[:, 2:]) < _S_OFF).all()
    k = rows[:, 0] * n + rows[:, 1]
    for a in (2, 3, 4):
        k = k * (2 * _S_OFF) + rows[:, a] + _S_OFF
    return k


def compare(got_rows, ref_rows, ref_dist, r_max: float, band: float, n: int):
    """Hold a search's rows to the reference's (built with reach >= band).  Raises AssertionError on a missing pair, a
    pair the reference does not have (wrong image, self pair at image 0, a pair beyond r_max + band) or a duplicate row.
    -> (pairs inside the band, of which present)."""
    g = keys(got_rows, n)
    ug, cnt = np.unique(g, return_counts=True)
    assert (cnt == 1).all(), f"{int((cnt > 1).sum())} duplicate rows, e.g. {np.asarray(got_rows)[np.isin(g, ug[cnt > 1])][:3].tolist()}"
    rk = keys(ref_rows, n)
    ref_dist = np.asarray(ref_dist)
    must = rk[ref_dist < r_max - band]
    may = rk[ref_dist < r_max + band]
    missing = must[~np.isin(must, ug)]
    assert missing.size == 0, f"{missing.size} pairs missing, e.g. {_unkey(missing[:3], n)}"
    extra = ug[~np.isin(ug, may)]
    assert extra.size == 0, f"{extra.size} pairs the reference does not have, e.g. {_unkey(extra[:3], n)}"
    in_band = rk[np.abs(ref_dist - r_max) <= band]
    return int(in_band.size), int(np.isin(in_band, ug).sum())


def _unkey(k, n):
    out = []
    for v in np.asarray(k).tolist():
        s = []
        for _ in range(3):
            s.append(v % (2 * _S_OFF) - _S_OFF)
            v //= 2 * _S_OFF
        out.append((v // n, v % n, s[2], s[1], s[0]))
    return out
