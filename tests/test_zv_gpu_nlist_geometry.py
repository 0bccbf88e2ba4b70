"""The device cell list (ab2_nl_bin / count / fill through ``data.neighbor_csr``) against the fp64 pair search of
nlist_oracle over the geometry matrix of nlist_cases, in fp64 and fp32, and the MD calculator on the geometries that
take it: a sheet with an open axis thinner than the cutoff, an open cluster, a box of exactly 3 (r_max + skin) and
atoms drifting several boxes out.  Every other test builds its edges with the package's own helpers: a wrong list
would go unnoticed there."""
import numpy as np
import pytest
import torch

import nlist_cases
import nlist_oracle as O
from allegro_b200 import data as D

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = nlist_cases.cases()
IDS = [c.name for c in CASES]


def _ref_box(case, dtype):
    return [float(torch.tensor(b, dtype=torch.float64).to(dtype)) for b in case.box]


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_neighbor_csr_matches_reference(case, dtype):
    pos = case.pos.to(dtype)
    posd, celld = pos.to(DEV), case.cell.to(DEV)
    n, r = pos.shape[0], case.r_max
    assert D.csr_supported(posd, r, celld, case.pbc) == (D.cell_grid(pos, r, case.box, case.pbc) is not None)
    assert D.csr_supported(posd, r, celld, case.pbc)
    csr, sv = D.neighbor_csr(posd, r, celld, case.pbc, n_centres=case.n_centres)
    nc = n if case.n_centres is None else case.n_centres
    # determinism: a second search gives the same bits
    csr2, sv2 = D.neighbor_csr(posd, r, celld, case.pbc, n_centres=case.n_centres)
    assert torch.equal(csr.row_ptr, csr2.row_ptr) and torch.equal(csr.nbr, csr2.nbr) and torch.equal(sv, sv2)

    # row layout: row_ptr rises from 0 to E, rows are centre-sorted, neighbours are atoms
    row_ptr, nbr, ctr = csr.row_ptr.cpu().long(), csr.nbr.cpu().long(), csr.ctr.cpu().long()
    E = nbr.shape[0]
    assert row_ptr.shape[0] == nc + 1 and int(row_ptr[0]) == 0 and int(row_ptr[-1]) == E == sv.shape[0] == csr.num_edges
    assert bool((row_ptr[1:] >= row_ptr[:-1]).all())
    assert torch.equal(ctr, torch.repeat_interleave(torch.arange(nc), row_ptr[1:] - row_ptr[:-1]))
    assert E == 0 or (int(nbr.min()) >= 0 and int(nbr.max()) < n)
    assert sv.dtype == dtype and csr.max_degree == (int((row_ptr[1:] - row_ptr[:-1]).max()) if nc else 0)

    # shifts: integer multiples of the (dtype-rounded) box on periodic axes, exactly 0 on open ones
    box = _ref_box(case, dtype)
    svc = sv.cpu()
    img = torch.zeros(E, 3, dtype=torch.long)
    for a in range(3):
        if case.pbc[a]:
            La = torch.tensor(box[a], dtype=dtype)
            img[:, a] = torch.round(svc[:, a].double() / box[a]).long()
            assert torch.equal(img[:, a].to(dtype) * La, svc[:, a]), a
        else:
            assert bool((svc[:, a] == 0).all()), a

    band = O.band_for(pos.double().numpy(), box, r, fp32=dtype == torch.float32)
    # lengths recomputed in fp64 from the outputs
    p64 = pos.double()
    if E:
        d = (p64[nbr] + svc.double() - p64[ctr]).norm(dim=-1)
        assert float(d.max()) < r + band

    got = np.concatenate([ctr.numpy()[:, None], nbr.numpy()[:, None], img.numpy()], 1)
    centres = np.arange(nc)
    if case.ref_centres is not None:
        centres = np.sort(np.random.default_rng(0).choice(nc, case.ref_centres, replace=False))
    ref, dist = O.pairs(p64.numpy(), box, case.pbc, r, centres=centres, reach=band)
    n_band, n_band_got = O.compare(got[np.isin(got[:, 0], centres)], ref, dist, r, band, n)
    print(f"\n[nlist] {case.name} {str(dtype)[6:]}: E={E} band={band:.3e} pairs in band {n_band} (listed {n_band_got})")

    # symmetry on full lists: (i, j, s) <=> (j, i, -s) outside the band
    if case.n_centres is None and E:
        k = O.keys(got, n)
        rev = O.keys(np.concatenate([got[:, 1:2], got[:, 0:1], -got[:, 2:]], 1), n)
        lone = ~np.isin(rev, k)
        if lone.any():
            d_lone = d.numpy()[lone]
            assert bool((np.abs(d_lone - r) <= band).all()), got[lone][:3].tolist()


def test_nl_bin_refuses_a_grid_past_int32():
    """ab2_nl_bin checks the cell count in int64 before any launch: 2000^3 cells would overflow the int32 cell id."""
    import ctypes as C

    from allegro_b200 import _lib

    pos = torch.zeros(4, 3, dtype=torch.float64, device=DEV)
    cell_id = torch.empty(4, dtype=torch.int32, device=DEV)
    box, org = (C.c_double * 3)(1e4, 1e4, 1e4), (C.c_double * 3)(0.0, 0.0, 0.0)
    pbc, nc = (C.c_int32 * 3)(0, 0, 0), (C.c_int32 * 3)(2000, 2000, 2000)
    rc = _lib.load().ab2_nl_bin(_lib.DTYPE_ENUM[torch.float64], 4, pos.data_ptr(), box, org, pbc, nc, 5.0, cell_id.data_ptr(), None)
    assert rc != 0
    nc_ok = (C.c_int32 * 3)(1, 1, 1)
    assert _lib.load().ab2_nl_bin(_lib.DTYPE_ENUM[torch.float64], 4, pos.data_ptr(), box, org, pbc, nc_ok, 5.0, cell_id.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert bool((cell_id == 0).all())


# --------------------------------------------------------------------------- #
# the MD calculator on those geometries
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def models():
    from test_gpu_model import _pair

    oracle, model64, _ = _pair("c2", 3, "float64")
    _, model32, _ = _pair("c2", 3, "float32")
    return oracle, {"float64": model64, "float32": model32}


def _exact(oracle, pos, cell, types, pbc, r_max):
    rows, _ = O.pairs(pos.numpy(), torch.diagonal(cell).tolist(), pbc, r_max)
    ei = torch.from_numpy(rows[:, :2].T.copy())
    sh = torch.from_numpy(rows[:, 2:].copy()).to(pos.dtype)
    return oracle({D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh})


def _walk_geometry(kind, r_list):
    """-> (pos, cell, pbc, step(pos, t, gen) -> next positions)"""
    g = torch.Generator().manual_seed(21)
    if kind == "sheet":
        pos, (lx, ly) = nlist_cases._hex_sheet(2.46, 7, 4)
        pos[:, :2] += 0.05 * torch.randn(pos[:, :2].shape, generator=g, dtype=torch.float64)  # z extent stays 0 at the first step
        cell = torch.diag(torch.tensor([lx, ly, 20.0], dtype=torch.float64))
        return pos, cell, (True, True, False), lambda p, t, gen: p + 0.05 * torch.randn(p.shape, generator=gen, dtype=p.dtype)
    if kind == "cluster":
        # planar flake: z extent 0 at the first step, x / y extents about 2 cutoffs
        sheet, (lx, ly) = nlist_cases._hex_sheet(2.46, 7, 4)
        sheet = sheet - torch.tensor([lx / 2, ly / 2, 0.0], dtype=torch.float64)
        pos = sheet[sheet.norm(dim=-1) < 6.0].clone()
        pos[:, :2] += 0.05 * torch.randn(pos[:, :2].shape, generator=g, dtype=torch.float64)
        cell = torch.eye(3, dtype=torch.float64) * 30.0
        return pos, cell, (False, False, False), lambda p, t, gen: p + 0.05 * torch.randn(p.shape, generator=gen, dtype=p.dtype)
    if kind == "three-cutoffs":
        L = 3 * r_list
        ij = torch.stack(torch.meshgrid(*[torch.arange(6)] * 3, indexing="ij"), -1).reshape(-1, 3).double()
        pos = (ij + 0.5) * (L / 6) + 0.1 * torch.randn(ij.shape, generator=g, dtype=torch.float64)
        cell = torch.eye(3, dtype=torch.float64) * L
        return pos, cell, (True, True, True), lambda p, t, gen: p + 0.05 * torch.randn(p.shape, generator=gen, dtype=p.dtype)
    if kind == "drift":
        from allegro_b200 import systems

        pos, cell, _ = systems.make_positions("c2", 5)
        L = torch.diagonal(cell)
        jump = torch.tensor([1.37, -2.11, 0.6], dtype=torch.float64) * L  # across faces, several boxes out
        return pos, cell, (True, True, True), lambda p, t, gen: p + jump + 0.05 * torch.randn(p.shape, generator=gen, dtype=p.dtype)
    raise ValueError(kind)


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind,dtype", [("sheet", "float64"), ("cluster", "float64"), ("three-cutoffs", "float64"),
                                        ("drift", "float64"), ("sheet", "float32")])
def test_calculator_walk(models, kind, dtype, use_graph):
    from allegro_b200.calculator import AllegroCalculator

    if dtype == "float32" and not use_graph:
        pytest.skip("one fp32 run: graph replay")
    oracle, by_dtype = models
    r_max = 5.0
    skin = 0.3 if kind == "three-cutoffs" else 0.5
    pos, cell, pbc, step = _walk_geometry(kind, r_max + skin)
    calc = AllegroCalculator(by_dtype[dtype], r_max, skin=skin, pbc=pbc, use_graph=use_graph)
    if kind == "three-cutoffs":
        rs = calc.r_max + calc.skin  # the cutoff of the calculator's list, as it computes it
        assert float(cell[0, 0]) == 3 * rs and (3 * rs) // rs == 2.0  # floor division alone puts one cell short
    tol = 1e-9 if dtype == "float64" else 1e-4
    types = torch.zeros(pos.shape[0], dtype=torch.long)
    gen = torch.Generator().manual_seed(5)
    p = pos.clone()
    for t in range(5):
        out = calc.compute(p.to(DEV), cell.to(DEV), types.to(DEV))
        assert D.CSR_KEY in calc._data, "the frame did not take the device cell list"
        ref = _exact(oracle, p, cell, types, pbc, r_max)
        f, e = out["forces"].double().cpu(), out["atomic_energy"].double().cpu()
        fr, er = ref[D.FORCE_KEY], ref[D.PER_ATOM_ENERGY_KEY]
        assert float((f - fr).abs().max() / fr.abs().max()) < tol, (t, "forces")
        assert float((e - er).abs().max() / er.abs().max()) < tol, (t, "atomic energies")
        assert abs(float(out["energy"].double().cpu().sum()) - float(ref[D.TOTAL_ENERGY_KEY].sum())) < tol * float(er.abs().sum())
        p = step(p, t, gen)
    assert calc.n_evaluations == 5
    if kind == "drift":
        assert calc.n_rebuilds >= 2
