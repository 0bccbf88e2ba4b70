"""Neighbour lists on the CPU against the fp64 pair search of nlist_oracle: the reference's own self-test, the torch
searches (``neighbor_list`` brute / cell, the fall-backs of the MD driver for triclinic and small cells) over the
geometry matrix of nlist_cases, and the cell grid every cell-list search is built on (``data.cell_grid``) against
the predicates the device check (nl_geom, csrc/nlist.cu) enforces."""
import math

import numpy as np
import pytest
import torch

import nlist_cases
import nlist_oracle as O
from allegro_b200 import data as D

CASES = nlist_cases.cases()
IDS = [c.name for c in CASES]


def _rows(ei, sh):
    return np.concatenate([ei.T.cpu().numpy(), torch.round(sh.double()).long().cpu().numpy()], 1).astype(np.int64)


def _ref_box(case, dtype):
    """lengths the search wraps with: the box rounded to the positions' dtype"""
    return [float(torch.tensor(b, dtype=torch.float64).to(dtype)) for b in case.box]


# --------------------------------------------------------------------------- #
# the reference itself
# --------------------------------------------------------------------------- #
def test_oracle_dimer_across_a_periodic_face():
    # 3-cell box (L = 15, r_max 5): 0.5 and 14.0 on x are 1.5 apart through the x face, 13.5 apart inside the box
    pos = np.array([[0.5, 7.5, 7.5], [14.0, 7.5, 7.5]])
    rows, dist = O.pairs(pos, (15.0, 15.0, 15.0), (True, True, True), 5.0)
    got = sorted(map(tuple, rows.tolist()))
    assert got == [(0, 1, -1, 0, 0), (1, 0, 1, 0, 0)]
    assert np.allclose(dist, 1.5, rtol=0, atol=1e-14)
    # raw coordinates: atom 1 two boxes out, atom 0 one box below -> the shifts carry the images back
    pos2 = pos + np.array([[-15.0, 0, 0], [30.0, 0, 0]])
    rows, dist = O.pairs(pos2, (15.0, 15.0, 15.0), (True, True, True), 5.0)
    assert sorted(map(tuple, rows.tolist())) == [(0, 1, -4, 0, 0), (1, 0, 4, 0, 0)]
    v = pos2[1] + np.array([-4 * 15.0, 0, 0]) - pos2[0]
    assert abs(np.linalg.norm(v) - 1.5) < 1e-13 and np.allclose(dist, 1.5, atol=1e-13)
    # open x: no pair at all
    rows, _ = O.pairs(pos, (15.0, 15.0, 15.0), (False, True, True), 5.0)
    assert rows.shape[0] == 0


def test_oracle_comparison_rejects_planted_defects():
    case = next(c for c in CASES if c.name == "G3-pbcTTT")
    pos, n = case.pos.numpy(), case.pos.shape[0]
    band = O.band_for(pos, case.box, case.r_max, fp32=False)
    ref, dist = O.pairs(pos, case.box, case.pbc, case.r_max, reach=band)
    assert O.compare(ref, ref, dist, case.r_max, band, n)[0] == 0
    inside = np.nonzero(dist < case.r_max - band)[0]
    k = int(inside[len(inside) // 2])
    defects = {
        "dropped pair": np.delete(ref, k, 0),
        "wrong image": np.concatenate([np.delete(ref, k, 0), ref[k : k + 1] + np.array([[0, 0, 1, 0, 0]])]),
        "duplicate row": np.concatenate([ref, ref[k : k + 1]]),
        "self pair at image 0": np.concatenate([ref, np.array([[5, 5, 0, 0, 0]])]),
    }
    for what, rows in defects.items():
        with pytest.raises(AssertionError):
            O.compare(rows, ref, dist, case.r_max, band, n)
        # and the order of rows does not matter to an accepted list
    O.compare(ref[::-1], ref, dist, case.r_max, band, n)


def test_oracle_band_pairs_may_go_either_way():
    pos = np.array([[1.0, 1.0, 1.0], [6.0, 1.0, 1.0]])  # exactly r_max apart
    band = 1e-9
    ref, dist = O.pairs(pos, (20.0, 20.0, 20.0), (False, False, False), 5.0, reach=band)
    assert ref.shape[0] == 2
    assert O.compare(ref, ref, dist, 5.0, band, 2) == (2, 2)
    assert O.compare(ref[:0], ref, dist, 5.0, band, 2) == (2, 0)


# --------------------------------------------------------------------------- #
# the torch searches
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("method", ["brute", "cell"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_neighbor_list_matches_reference(case, method, dtype):
    if method == "brute" and case.ref_centres is not None:
        pytest.skip("all-pairs over the full frame: the cell list covers the full-size frame")
    pos = case.pos.to(dtype)
    ei, sh = D.neighbor_list(pos, case.r_max, case.cell, case.pbc, method=method)
    got = _rows(ei, sh)
    n = pos.shape[0]
    box = _ref_box(case, dtype)
    band = O.band_for(pos.double().numpy(), box, case.r_max, fp32=dtype == torch.float32)
    centres = None
    if case.ref_centres is not None:
        centres = np.sort(np.random.default_rng(0).choice(n, case.ref_centres, replace=False))
        got = got[np.isin(got[:, 0], centres)]
    ref, dist = O.pairs(pos.double().numpy(), box, case.pbc, case.r_max, centres=centres, reach=band)
    O.compare(got, ref, dist, case.r_max, band, n)


def test_neighbor_list_auto_takes_the_cell_list_at_three_cutoffs():
    """More than 3000 atoms in a periodic box of exactly 3 r_max for an r_max where (3 r) // r == 2: the automatic
    choice picks the cell list, which has to take the grid of 3 cells."""
    r = nlist_cases.R_ODD[0]
    L = 3 * r
    assert L // r == 2.0
    g = torch.Generator().manual_seed(2)
    pos = torch.rand(3001, 3, generator=g, dtype=torch.float64) * L
    ei, sh = D.neighbor_list(pos, r, torch.eye(3, dtype=torch.float64) * L, (True, True, True))
    got = _rows(ei, sh)
    centres = np.arange(0, 3001, 47)
    band = O.band_for(pos.numpy(), (L,) * 3, r, fp32=False)
    ref, dist = O.pairs(pos.numpy(), (L,) * 3, (True, True, True), r, centres=centres, reach=band)
    O.compare(got[np.isin(got[:, 0], centres)], ref, dist, r, band, 3001)


# --------------------------------------------------------------------------- #
# the cell grid
# --------------------------------------------------------------------------- #
def _check_grid(grid, pos, r_max, pbc):
    box, origin, ncell = grid
    n = pos.shape[0]
    for a in range(3):
        assert ncell[a] >= 1 and isinstance(ncell[a], int)
        assert box[a] / ncell[a] >= r_max * (1 - 1e-12), (a, box[a], ncell[a])  # nl_geom: cells >= r_max wide
        if pbc[a]:
            assert ncell[a] >= 3 and origin[a] == 0.0
        elif n:
            # open axis: every atom inside [origin, origin + box)
            assert float(pos[:, a].min()) >= origin[a] and float(pos[:, a].max()) < origin[a] + box[a]
    total = int(np.prod(np.array(ncell, dtype=np.int64)))
    assert total <= max(27, 4 * n) and total < 2**31 - 1


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_cell_grid_predicates(case, dtype):
    pos = case.pos.to(dtype)
    grid = D.cell_grid(pos, case.r_max, case.box, case.pbc)
    assert grid is not None  # every periodic axis of the matrix is >= 3 r_max long
    _check_grid(grid, pos, case.r_max, case.pbc)
    assert not D.csr_supported(pos, case.r_max, case.cell, case.pbc)  # CPU positions never take the device search


@pytest.mark.parametrize("r_max", [5.5, *nlist_cases.R_ODD, 3.0, 4.1, 6.3])
def test_cell_grid_at_three_cutoffs(r_max):
    L = 3 * r_max
    box, _, ncell = D.cell_grid(torch.zeros(1, 3, dtype=torch.float64), r_max, (L, L, L), (True, True, True))
    assert ncell == [3, 3, 3] and box == [L, L, L]
    assert L / 3 >= r_max * (1 - 1e-12)  # what nl_geom tests


def test_cell_grid_rejects_short_periodic_axes_only():
    pos = torch.zeros(4, 3, dtype=torch.float64)
    r = 5.0
    L = 3 * r * (1 - 1e-9)
    assert D.cell_grid(pos, r, (L, 20.0, 20.0), (True, True, True)) is None
    assert D.cell_grid(pos, r, (0.0, 20.0, 20.0), (True, True, True)) is None
    # an open axis takes any box length: the grid spans the atoms
    grid = D.cell_grid(pos, r, (L, 20.0, 20.0), (False, True, True))
    assert grid is not None and grid[2][0] == 1
    _check_grid(grid, pos, r, (False, True, True))


def test_cell_grid_bounds_the_cell_count():
    """A far-flung atom on open axes: 2000 cells per axis at r_max 5 without the bound (8e9 cells, past int32)."""
    g = torch.Generator().manual_seed(3)
    pos = torch.cat([torch.rand(500, 3, generator=g, dtype=torch.float64) * 12, torch.full((1, 3), 1e4, dtype=torch.float64)])
    grid = D.cell_grid(pos, 5.0, (30.0, 30.0, 30.0), (False, False, False))
    _check_grid(grid, pos, 5.0, (False, False, False))
    assert math.prod(math.floor(b / 5.0) for b in grid[0]) > 2**31  # what the unbounded grid would have been
    # periodic axes are coarsened last and never below 3 cells
    grid = D.cell_grid(torch.zeros(0, 3, dtype=torch.float64), 5.0, (100.0, 100.0, 100.0), (True, True, True))
    assert grid[2] == [3, 3, 3]
    grid = D.cell_grid(torch.zeros(2, 3, dtype=torch.float64), 5.0, (100.0, 100.0, 100.0), (True, True, False))
    assert grid[2][2] == 1 and min(grid[2][:2]) >= 3
    _check_grid(grid, torch.zeros(2, 3), 5.0, (True, True, False))
