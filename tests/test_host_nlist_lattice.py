"""The general-lattice pair search of nlist_lattice_oracle against hand-worked and orthorhombic results, and the grid
of the device lattice search (``data.lattice_grid``) against the predicates its device check (nl_lattice_geom,
csrc/nlist.cu) enforces, on every geometry of nlist_lattice_cases."""
import math

import numpy as np
import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
import nlist_oracle as O
from allegro_b200 import data as D

CASES = nlist_lattice_cases.cases()
IDS = [c.name for c in CASES]


# --------------------------------------------------------------------------- #
# the reference itself
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", ["G3-pbcTTT", "G3-pbcTFT", "G3-pbcFFF", "G5-raw-TTT", "G4-two-TTF", "G6-dense"])
def test_oracle_equals_the_orthorhombic_oracle_on_diagonal_cells(name):
    case = next(c for c in nlist_cases.cases(full_size=False) if c.name == name)
    pos = case.pos.numpy()
    a, da = LO.pairs(pos, np.diag(case.box), case.pbc, case.r_max)
    b, db = O.pairs(pos, case.box, case.pbc, case.r_max)
    n = pos.shape[0]
    ka, kb = O.keys(a, n), O.keys(b, n)
    assert np.array_equal(np.sort(ka), np.sort(kb))
    assert np.allclose(da[np.argsort(ka)], db[np.argsort(kb)], rtol=0, atol=1e-12)


def test_oracle_triclinic_dimer():
    # rows a = (10,0,0), b = (8,6,0), c = (0,0,10); atom 1 = atom 0 + b - (0,2,0): 2.0 apart through the -b image,
    # sqrt(80) apart inside the cell
    rows = np.array([[10.0, 0, 0], [8.0, 6.0, 0], [0, 0, 10.0]])
    pos = np.array([[3.0, 1.0, 5.0], [11.0, 5.0, 5.0]])
    got, dist = LO.pairs(pos, rows, (True, True, True), 3.0)
    assert sorted(map(tuple, got.tolist())) == [(0, 1, 0, -1, 0), (1, 0, 0, 1, 0)]
    assert np.allclose(dist, 2.0, rtol=0, atol=1e-13)
    got, dist = LO.pairs(pos, rows, (True, True, True), 9.0)
    assert (0, 1, 0, 0, 0) in set(map(tuple, got.tolist()))
    assert abs(dist[(got[:, :2] == [0, 1]).all(1) & (got[:, 2:] == 0).all(1)][0] - math.sqrt(80.0)) < 1e-13
    # b open, r_max 9: the pair inside the cell (sqrt(80)) and through -a ((-2, 4, 0): sqrt(20)); no b image
    got, dist = LO.pairs(pos, rows, (True, False, True), 9.0)
    assert sorted(map(tuple, got.tolist())) == [(0, 1, -1, 0, 0), (0, 1, 0, 0, 0), (1, 0, 0, 0, 0), (1, 0, 1, 0, 0)]
    assert np.allclose(np.sort(dist), np.sqrt([20.0, 20.0, 80.0, 80.0]), rtol=0, atol=1e-13)
    # raw coordinates: atom 1 moved by 3a - 2b: the shift carries the image back
    pos2 = pos + np.array([[0, 0, 0], 3 * rows[0] - 2 * rows[1]])
    got, dist = LO.pairs(pos2, rows, (True, True, True), 3.0)
    assert sorted(map(tuple, got.tolist())) == [(0, 1, -3, 1, 0), (1, 0, 3, -1, 0)]
    assert np.allclose(dist, 2.0, atol=1e-12)


@pytest.mark.parametrize("M", [[[1, 1, 0], [0, 1, 0], [0, 0, 1]], [[0, 1, 0], [1, 0, 0], [1, 1, 1]], [[2, 1, 0], [1, 1, 0], [0, -1, 1]]],
                         ids=["shear", "det-1", "mixed"])
def test_oracle_pairs_map_under_a_unimodular_basis_change(M):
    case = next(c for c in CASES if c.name == "L1-lammps-max-tilt")
    M = np.array(M, dtype=np.float64)
    assert abs(abs(np.linalg.det(M)) - 1) < 1e-12
    h = case.cell.numpy()
    pos = case.pos.numpy()
    n = pos.shape[0]
    a, da = LO.pairs(pos, h, case.pbc, case.r_max)
    b, db = LO.pairs(pos, M @ h, case.pbc, case.r_max)
    mapped = a.copy()
    mapped[:, 2:] = np.rint(a[:, 2:] @ np.linalg.inv(M)).astype(np.int64)  # s' = s M^-1
    km, kb = O.keys(mapped, n), O.keys(b, n)
    assert np.array_equal(np.sort(km), np.sort(kb))
    assert np.allclose(np.sort(da), np.sort(db), rtol=0, atol=1e-10)


def test_oracle_comparison_rejects_planted_defects():
    case = next(c for c in CASES if c.name == "L1-hcp-120deg")
    pos, n = case.pos.numpy(), case.pos.shape[0]
    rows = case.cell.numpy()
    band = LO.band_for(pos, rows, case.r_max, fp32=False)
    ref, dist = LO.pairs(pos, rows, case.pbc, case.r_max, reach=band)
    assert LO.compare(ref, ref, dist, case.r_max, band, n)[0] == 0
    inside = np.nonzero(dist < case.r_max - band)[0]
    k = int(inside[len(inside) // 2])
    defects = {
        "dropped pair": np.delete(ref, k, 0),
        "wrong image": np.concatenate([np.delete(ref, k, 0), ref[k : k + 1] + np.array([[0, 0, 0, 1, 0]])]),
        "duplicate row": np.concatenate([ref, ref[k : k + 1]]),
        "self pair at image 0": np.concatenate([ref, np.array([[5, 5, 0, 0, 0]])]),
    }
    for what, bad in defects.items():
        with pytest.raises(AssertionError):
            LO.compare(bad, ref, dist, case.r_max, band, n)
    LO.compare(ref[::-1], ref, dist, case.r_max, band, n)


def test_oracle_completes_zero_rows():
    h = LO.complete([[3.0, 0, 0], [1.0, 4.0, 0], [0, 0, 0]], (True, True, False))
    assert np.allclose(h[2], [0, 0, 1]) or np.allclose(h[2], [0, 0, -1])
    assert np.allclose(LO.complete(None, (False, False, False)) @ LO.complete(None, (False, False, False)).T, np.eye(3))


# --------------------------------------------------------------------------- #
# the lattice grid
# --------------------------------------------------------------------------- #
def _metrics(rows):
    det, heights, regular = D._lattice_metrics(rows)
    assert regular
    return det, heights


def check_lattice_grid(grid, pos, r_max, pbc, cell):
    rows, origin, ncell, reach = grid
    n = pos.shape[0]
    det, heights = _metrics(rows)
    for a in range(3):
        assert isinstance(ncell[a], int) and isinstance(reach[a], int) and ncell[a] >= 1 and reach[a] >= 1
        assert heights[a] / ncell[a] * reach[a] >= r_max * (1 - 1e-12), (a, heights[a], ncell[a], reach[a])  # t_a k_a >= r_max
        if reach[a] > 1:
            assert heights[a] / ncell[a] * (reach[a] - 1) < r_max * (1 - 1e-12)  # the fewest bins that reach
        if pbc[a]:
            assert origin[a] == 0.0
            assert np.allclose(rows[a], cell.reshape(3, 3)[a].tolist(), rtol=0, atol=0)  # periodic rows are the cell's
    total = math.prod(ncell)
    assert total <= max(27, 4 * n) and total < 2**31 - 1
    assert math.prod(2 * k + 1 for k in reach) < 2**31 - 1
    open_axes = [a for a in range(3) if not pbc[a]]
    if n and open_axes:
        f = pos.double().numpy() @ np.linalg.inv(np.array(rows)) - np.array(origin)
        for a in open_axes:  # open-axis atoms inside the grid
            assert f[:, a].min() >= 0.0 and f[:, a].max() < 1.0, (a, f[:, a].min(), f[:, a].max())


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_lattice_grid_predicates(case, dtype):
    pos = case.pos.to(dtype)
    grid = D.lattice_grid(pos, case.r_max, case.cell, case.pbc)
    assert grid is not None
    check_lattice_grid(grid, pos, case.r_max, case.pbc, case.cell)
    assert not D.csr_supported(pos, case.r_max, case.cell, case.pbc)  # CPU positions never take the device search
    assert D.search_grid(pos, case.r_max, case.cell, case.pbc)[0] == "lattice"


def test_lattice_grid_stencils_on_short_axes():
    for f, k in ((2.2, 1), (1.0, 1), (0.4, 3)):
        case = next(c for c in CASES if c.name == f"L2-height-{f}r")
        _, _, ncell, reach = D.lattice_grid(case.pos, case.r_max, case.cell, case.pbc)
        assert reach[2] == k and ncell[2] == (2 if f == 2.2 else 1)
    case = next(c for c in CASES if c.name == "L2-graphite-c6.7")
    assert D.lattice_grid(case.pos, case.r_max, case.cell, case.pbc)[2][2] == 1
    for case in (c for c in CASES if c.name.startswith("L9-")):
        _, _, ncell, reach = D.lattice_grid(case.pos, case.r_max, case.cell, case.pbc)
        assert ncell[2] == 3 and reach[2] == 1


@pytest.mark.parametrize("case", nlist_cases.cases(full_size=False), ids=lambda c: c.name)
def test_frames_cell_grid_accepts_keep_the_orthorhombic_grid(case):
    route = D.search_grid(case.pos, case.r_max, case.cell, case.pbc)
    assert route[0] == "ortho" and route[1] == D.cell_grid(case.pos, case.r_max, case.box, case.pbc)
    # the lattice grid exists for them too (the lattice kernels are checked against the orthorhombic ones on the GPU)
    check_lattice_grid(D.lattice_grid(case.pos, case.r_max, case.cell, case.pbc), case.pos, case.r_max, case.pbc, case.cell)


def test_lattice_grid_refuses_what_it_cannot_bin():
    pos = torch.zeros(3, 3, dtype=torch.float64)
    assert D.lattice_grid(pos, 5.0, None, (True, False, False)) is None  # a periodic axis needs a row
    sing = torch.tensor([[10.0, 0, 0], [20.0, 0, 0], [0, 0, 10.0]], dtype=torch.float64)
    assert D.lattice_grid(pos, 5.0, sing, (True, True, True)) is None
    zero_periodic = torch.tensor([[10.0, 0, 0], [0, 0, 0], [0, 0, 10.0]], dtype=torch.float64)
    assert D.lattice_grid(pos, 5.0, zero_periodic, (True, True, True)) is None
    nan = torch.tensor([[10.0, 0, 0], [0, float("nan"), 0], [0, 0, 10.0]], dtype=torch.float64)
    assert D.lattice_grid(pos, 5.0, nan, (True, True, True)) is None
    # a singular cell is fine when the offending rows are open
    assert D.lattice_grid(pos, 5.0, sing, (True, False, True)) is not None
    # a far-flung atom: the bin count stays bounded, open axes coarsened first
    far = torch.cat([torch.rand(100, 3, dtype=torch.float64) * 10, torch.full((1, 3), 1e5, dtype=torch.float64)])
    grid = D.lattice_grid(far, 5.0, None, (False, False, False))
    check_lattice_grid(grid, far, 5.0, (False, False, False), None)
