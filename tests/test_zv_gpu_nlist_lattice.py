"""The general-lattice device cell list (ab2_nl_lattice_bin / count / fill through ``data.neighbor_csr``) against the
fp64 pair search of nlist_lattice_oracle over the geometry matrix of nlist_lattice_cases, in fp64 and fp32; the route
each frame takes; the lattice kernels against the orthorhombic ones; the model's invariance under a change of cell
basis; and the MD calculator on crystals, short axes, wires, zero-row sheets, clusters without a cell and a tilted
drift."""
import ctypes as C

import numpy as np
import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
import nlist_oracle as O
from allegro_b200 import _lib
from allegro_b200 import data as D

pytestmark = pytest.mark.gpu
DEV = "cuda"

CASES = nlist_lattice_cases.cases()
IDS = [c.name for c in CASES]


def _oracle_rows(case):
    return LO.complete(None if case.cell is None else case.cell.numpy(), case.pbc)


def _check_csr(csr, sv, pos, n_centres, dtype):
    n, nc = pos.shape[0], n_centres
    row_ptr, nbr, ctr = csr.row_ptr.cpu().long(), csr.nbr.cpu().long(), csr.ctr.cpu().long()
    E = nbr.shape[0]
    assert row_ptr.shape[0] == nc + 1 and int(row_ptr[0]) == 0 and int(row_ptr[-1]) == E == sv.shape[0] == csr.num_edges
    assert bool((row_ptr[1:] >= row_ptr[:-1]).all())
    assert torch.equal(ctr, torch.repeat_interleave(torch.arange(nc), row_ptr[1:] - row_ptr[:-1]))
    assert E == 0 or (int(nbr.min()) >= 0 and int(nbr.max()) < n)
    assert sv.dtype == dtype and csr.max_degree == (int((row_ptr[1:] - row_ptr[:-1]).max()) if nc else 0)
    return ctr, nbr


def _image_rows(ctr, nbr, sv, rows, pbc, dtype):
    """(i, j, s) rows from the shift vectors: integer combinations of the cell rows, 0 along open axes"""
    img, dev = LO.images_of(sv.double().cpu().numpy(), rows)
    scale = max(1.0, float(np.abs(sv.double().cpu().numpy()).max()) if sv.numel() else 1.0)
    assert dev <= (1e-6 if dtype == torch.float32 else 1e-13) * scale, dev  # shift = s . rows, rounded once
    for a in range(3):
        if not pbc[a]:
            assert (img[:, a] == 0).all(), a
    return np.concatenate([ctr.numpy()[:, None], nbr.numpy()[:, None], img], 1)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_neighbor_csr_lattice_matches_reference(case, dtype):
    pos = case.pos.to(dtype)
    posd = pos.to(DEV)
    celld = None if case.cell is None else case.cell.to(DEV)
    n, r = pos.shape[0], case.r_max
    assert D.csr_supported(posd, r, celld, case.pbc)
    csr, sv = D.neighbor_csr(posd, r, celld, case.pbc)
    csr2, sv2 = D.neighbor_csr(posd, r, celld, case.pbc)
    assert torch.equal(csr.row_ptr, csr2.row_ptr) and torch.equal(csr.nbr, csr2.nbr) and torch.equal(sv, sv2)
    ctr, nbr = _check_csr(csr, sv, pos, n, dtype)
    rows = _oracle_rows(case)
    got = _image_rows(ctr, nbr, sv, rows, case.pbc, dtype)
    p64 = pos.double()
    band = LO.band_for(p64.numpy(), rows, r, fp32=dtype == torch.float32)
    E = nbr.shape[0]
    if E:
        d = (p64[nbr] + sv.cpu().double() - p64[ctr]).norm(dim=-1)
        assert float(d.max()) < r + band
    centres = np.arange(n)
    if case.ref_centres is not None:
        centres = np.sort(np.random.default_rng(0).choice(n, case.ref_centres, replace=False))
    ref, dist = LO.pairs(p64.numpy(), rows, case.pbc, r, centres=centres, reach=band)
    n_band, n_band_got = LO.compare(got[np.isin(got[:, 0], centres)], ref, dist, r, band, n)
    print(f"\n[nlist-lattice] {case.name} {str(dtype)[6:]}: E={E} band={band:.3e} pairs in band {n_band} (listed {n_band_got})")
    if E:
        k = O.keys(got, n)
        rev = O.keys(np.concatenate([got[:, 1:2], got[:, 0:1], -got[:, 2:]], 1), n)
        lone = ~np.isin(rev, k)
        if lone.any():
            assert bool((np.abs(d.numpy()[lone] - r) <= band).all()), got[lone][:3].tolist()


class _Spy:
    """load() stand-in that records which ab2_* entry points a search calls"""

    def __init__(self, lib):
        self.lib, self.called = lib, []

    def __getattr__(self, name):
        if name.startswith("ab2_nl"):
            self.called.append(name)
        return getattr(self.lib, name)


def _route(monkeypatch, pos, r, cell, pbc):
    spy = _Spy(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda: spy)
    D.neighbor_csr(pos, r, cell, pbc)
    monkeypatch.undo()
    return set(spy.called)


def test_routes(monkeypatch):
    for case in nlist_cases.cases(full_size=False):
        if case.n_centres is not None or case.pos.shape[0] == 0:
            continue
        called = _route(monkeypatch, case.pos.to(DEV), case.r_max, case.cell.to(DEV), case.pbc)
        assert called and all(c.startswith("ab2_nl_") and "lattice" not in c for c in called), (case.name, called)
    for case in CASES:
        if case.pos.shape[0] == 0:
            continue
        called = _route(monkeypatch, case.pos.to(DEV), case.r_max, None if case.cell is None else case.cell.to(DEV), case.pbc)
        assert called and all(c.startswith("ab2_nl_lattice_") for c in called), (case.name, called)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("case", [c for c in nlist_cases.cases() if c.n_centres is None], ids=lambda c: c.name)
def test_lattice_kernels_match_the_orthorhombic_ones(case, dtype):
    pos = case.pos.to(dtype).to(DEV)
    n, r = pos.shape[0], case.r_max
    a_csr, a_sv = D.neighbor_csr(pos, r, case.cell.to(DEV), case.pbc)  # orthorhombic route
    rows, origin, ncell, reach = D.lattice_grid(pos, r, case.cell, case.pbc)
    row_ptr, nbr, sv = _lib.neighbor_csr_lattice(pos, r, rows, origin, ncell, reach, case.pbc, n)
    ctr = torch.repeat_interleave(torch.arange(n, device=DEV), (row_ptr[1:] - row_ptr[:-1]).long())
    box = np.diag(case.box)
    rows_a = _image_rows(a_csr.ctr.cpu().long(), a_csr.nbr.cpu().long(), a_sv, box, case.pbc, dtype)
    rows_b = _image_rows(ctr.cpu(), nbr.cpu().long(), sv, box, case.pbc, dtype)
    ka, kb = O.keys(rows_a, n), O.keys(rows_b, n)
    assert np.unique(kb).size == kb.size
    diff = np.setxor1d(ka, kb)
    print(f"\n[nlist-lattice vs ortho] {case.name} {str(dtype)[6:]}: E={kb.size} differing rows {diff.size}")
    if diff.size:  # only pairs on the cutoff may differ (different rounding of the two distance tests)
        p64 = case.pos.to(dtype).double().numpy()
        both = np.concatenate([rows_a, rows_b])
        centres = np.unique(both[np.isin(O.keys(both, n), diff), 0])
        band = O.band_for(p64, case.box, r, fp32=dtype == torch.float32)
        ref, dist = O.pairs(p64, _ref_box(case.box, dtype), case.pbc, r, centres=centres, reach=band)
        rk = O.keys(ref, n)
        assert np.isin(diff, rk).all() and (np.abs(dist[np.isin(rk, diff)] - r) <= band).all()


def _ref_box(box, dtype):
    return [float(torch.tensor(b, dtype=torch.float64).to(dtype)) for b in box]


def test_lattice_abi_refuses_before_launching():
    lib = _lib.load()
    pos = torch.zeros(4, 3, dtype=torch.float64, device=DEV)
    cell_id = torch.full((4,), -7, dtype=torch.int32, device=DEV)
    org = (C.c_double * 3)(0.0, 0.0, 0.0)
    pbc = (C.c_int32 * 3)(1, 1, 1)

    def call(rows, nc, reach, r=5.0):
        return lib.ab2_nl_lattice_bin(_lib.AB2_F64, 4, pos.data_ptr(), (C.c_double * 9)(*rows), org, pbc, (C.c_int32 * 3)(*nc),
                                      (C.c_int32 * 3)(*reach), r, cell_id.data_ptr(), None)

    good = [10.0, 0, 0, 0, 10.0, 0, 0, 0, 10.0]
    assert call([10.0, 0, 0, 20.0, 0, 0, 0, 0, 10.0], [1, 1, 1], [1, 1, 1]) != 0  # singular
    assert call([10.0, 0, 0, 0, float("inf"), 0, 0, 0, 10.0], [1, 1, 1], [1, 1, 1]) != 0  # not finite
    assert call(good, [0, 1, 1], [1, 1, 1]) != 0  # no bins
    assert call(good, [2, 1, 1], [1, 1, 1], r=5.5) != 0  # bins 5 thick cannot reach r_max 5.5 in one step
    big = [1e6, 0, 0, 0, 1e6, 0, 0, 0, 1e6]
    assert call(big, [2000, 2000, 2000], [1, 1, 1]) != 0  # 8e9 bins: past int32
    assert call(good, [1, 1, 1], [1000, 1000, 1000]) != 0  # 8e9 bins visited per centre
    torch.cuda.synchronize()
    assert bool((cell_id == -7).all())  # nothing was launched
    assert call(good, [2, 1, 1], [2, 1, 1], r=5.5) == 0 and call(good, [2, 1, 1], [1, 1, 1], r=5.0) == 0
    assert call(good, [1, 1, 1], [1, 1, 1]) == 0
    torch.cuda.synchronize()
    assert bool((cell_id == 0).all())


# --------------------------------------------------------------------------- #
# the model on those lists
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def models():
    from test_gpu_model import _pair

    oracle, model64, _ = _pair("c2", 3, "float64")
    _, model32, _ = _pair("c2", 3, "float32")
    return oracle, {"float64": model64, "float32": model32}


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_energy_forces_virial_do_not_depend_on_the_cell_basis(models, dtype):
    from allegro_b200 import systems

    _, by_dtype = models
    model = by_dtype[dtype]
    inner = getattr(model, "model", model)
    pos, cell, types = systems.make_positions("c2", 5)
    pos = pos.to(getattr(torch, dtype)).to(DEV)
    types = types.to(DEV)
    outs = []
    for M in ([[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[1, 1, 0], [0, 1, 0], [1, 0, 1]], [[0, 1, 0], [1, 0, 0], [0, 1, 1]]):
        M = torch.tensor(M, dtype=torch.float64)
        h = (M @ cell).to(DEV)
        csr, sv = D.neighbor_csr(pos, 5.0, h, (True, True, True))
        d = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: types, D.CELL_KEY: h, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
        o = inner.energy_and_forces(d, stress=True)
        outs.append([o[k].double().cpu() for k in (D.TOTAL_ENERGY_KEY, D.FORCE_KEY, D.VIRIAL_KEY)])
    # energy, forces, virial.  The three lists hold the same edges with the same shift vectors (fp64 agrees to 1e-14) in a
    # different order within each row; in fp32 the force sums then differ by their own rounding, which for this model
    # is the 1e-5 level of its fp32-vs-fp64 force error, so the fp32 forces are held to 1e-4
    tols = (1e-10, 1e-10, 1e-10) if dtype == "float64" else (1e-5, 1e-4, 1e-5)
    for k, o in enumerate(outs[1:]):
        devs = [float((a - b).abs().max() / b.abs().max()) for a, b in zip(outs[0], o)]
        print(f"\n[basis] {dtype} basis {k + 1}: energy / forces / virial relative deviation {devs}")
        assert all(d < t for d, t in zip(devs, tols)), devs


def _exact(oracle, pos, case_cell, types, pbc, r_max):
    rows = LO.complete(None if case_cell is None else case_cell.numpy(), pbc)
    ref_rows, _ = LO.pairs(pos.numpy(), rows, pbc, r_max)
    ei = torch.from_numpy(ref_rows[:, :2].T.copy())
    sh = torch.from_numpy(ref_rows[:, 2:].copy()).to(pos.dtype)
    return oracle({D.POSITIONS_KEY: pos, D.CELL_KEY: torch.from_numpy(rows), D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei,
                   D.EDGE_CELL_SHIFT_KEY: sh})


def _walk_geometry(kind):
    """-> (pos, cell or None, pbc, step(pos, gen) -> next positions)"""
    jiggle = lambda p, gen: p + 0.05 * torch.randn(p.shape, generator=gen, dtype=p.dtype)  # noqa: E731
    if kind == "hcp":
        pos, rows = nlist_lattice_cases.hcp()
        return pos, rows, (True, True, True), jiggle
    if kind == "graphite":
        pos, rows = nlist_lattice_cases.graphite()
        return pos, rows, (True, True, True), jiggle
    if kind == "tilted-wire":
        pos, rows = nlist_lattice_cases.tilted_wire()
        return pos, rows, (False, False, True), jiggle
    if kind == "ase-sheet":
        pos, rows = nlist_lattice_cases.tilted_sheet(12)
        rows = rows.clone()
        rows[2] = 0.0
        return pos, rows, (True, True, False), jiggle
    if kind == "cluster":
        return nlist_lattice_cases.cluster(), None, (False, False, False), jiggle
    if kind == "tilted-drift":
        pos, rows = nlist_lattice_cases.hcp()
        jump = torch.tensor([1.37, -2.11, 0.6], dtype=torch.float64) @ rows  # several cells out along tilted axes
        return pos, rows, (True, True, True), lambda p, gen: jiggle(p + jump, gen)
    raise ValueError(kind)


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind,dtype", [("hcp", "float64"), ("graphite", "float64"), ("tilted-wire", "float64"),
                                        ("ase-sheet", "float64"), ("cluster", "float64"), ("tilted-drift", "float64"),
                                        ("hcp", "float32")])
def test_calculator_walk_lattice(models, kind, dtype, use_graph):
    from allegro_b200.calculator import AllegroCalculator

    if dtype == "float32" and not use_graph:
        pytest.skip("one fp32 run: graph replay")
    oracle, by_dtype = models
    r_max = 5.0
    pos, cell, pbc, step = _walk_geometry(kind)
    calc = AllegroCalculator(by_dtype[dtype], r_max, skin=0.5, pbc=pbc, use_graph=use_graph)
    tol = 1e-9 if dtype == "float64" else 1e-4
    types = torch.zeros(pos.shape[0], dtype=torch.long)
    gen = torch.Generator().manual_seed(5)
    # positions in the model's dtype: the fp32 run takes the fp32 lattice search; the reference sees the same rounded values
    p = pos.to(getattr(torch, dtype))
    for t in range(5):
        out = calc.compute(p.to(DEV), None if cell is None else cell.to(DEV), types.to(DEV))
        assert D.CSR_KEY in calc._data, "the frame did not take the device cell list"
        assert calc._data[D.EDGE_SHIFT_VEC_KEY].dtype == p.dtype
        ref = _exact(oracle, p.double(), cell, types, pbc, r_max)
        f, e = out["forces"].double().cpu(), out["atomic_energy"].double().cpu()
        fr, er = ref[D.FORCE_KEY], ref[D.PER_ATOM_ENERGY_KEY]
        assert float((f - fr).abs().max() / fr.abs().max()) < tol, (t, "forces")
        assert float((e - er).abs().max() / er.abs().max()) < tol, (t, "atomic energies")
        assert abs(float(out["energy"].double().cpu().sum()) - float(ref[D.TOTAL_ENERGY_KEY].sum())) < tol * float(er.abs().sum())
        p = step(p, gen).to(p.dtype)
    assert calc.n_evaluations == 5
    if kind == "tilted-drift":
        assert calc.n_rebuilds >= 2


def test_calculator_stress_needs_a_volume(models):
    from allegro_b200.calculator import AllegroCalculator

    _, by_dtype = models
    pos, rows = nlist_lattice_cases.tilted_sheet(12)
    rows = rows.clone()
    rows[2] = 0.0
    calc = AllegroCalculator(by_dtype["float64"], 5.0, skin=0.5, pbc=(True, True, False), compute_stress=True)
    types = torch.zeros(pos.shape[0], dtype=torch.long, device=DEV)
    with pytest.raises(ValueError):
        calc.compute(pos.to(DEV), rows.to(DEV), types)
    # rows within 1e-12 rad of a common plane count as singular too
    rows[2] = rows[0] + torch.tensor([0.0, 0.0, 1e-14], dtype=torch.float64)
    assert not D.is_regular_cell(rows)
    with pytest.raises(ValueError):
        calc.compute(pos.to(DEV), rows.to(DEV), types)
