"""The batched-frames device neighbour list (ab2_nl_frames_count / fill through ``data.neighbor_csr_frames``) against the
fp64 pair search of nlist_lattice_oracle, on every geometry of nlist_cases and nlist_lattice_cases small enough for it, in
fp64 and fp32: each frame alone, all of them in one batch between empty and one-atom frames, against the device cell
list (``data.neighbor_csr``); and the model on a batch of crystals, short axes, sheets, wires, a cluster without a cell,
one atom and an empty frame against the fp64 oracle, with and without stress."""
import numpy as np
import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
import nlist_oracle as O
from allegro_b200 import data as D
from allegro_b200.batch import collate, split
from nlist_lattice_cases import LCase
from test_zv_gpu_nlist_lattice import _check_csr, _exact, _image_rows

pytestmark = pytest.mark.gpu
DEV = "cuda"
T, F = True, False
DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]


def _cases():
    """every case as a user would pass it; the halo's local frame (rows for owned atoms only) has no frames equivalent"""
    out = [LCase(c.name, c.pos, c.cell, c.pbc, c.r_max) for c in nlist_cases.cases(full_size=False) if c.n_centres is None]
    out += nlist_lattice_cases.cases(full_size=False)
    return [c for c in out if c.pos.shape[0] <= D.FRAMES_MAX_ATOMS]


CASES = _cases()
IDS = [c.name for c in CASES]


def _search(frames, dtype, r_max):
    """one batch of ``frames`` -> (EdgeCSR, shift_vec, frame_ptr); zero cells for frames without one, as collate does"""
    pos = torch.cat([f.pos.to(dtype) for f in frames]).to(DEV)
    fp = torch.tensor([0] + [f.pos.shape[0] for f in frames]).cumsum(0)
    pbc = torch.tensor([f.pbc for f in frames], device=DEV)
    if all(f.cell is None for f in frames):
        cell = None
    else:
        cell = torch.stack([torch.zeros(3, 3, dtype=torch.float64) if f.cell is None else f.cell for f in frames]).to(DEV, dtype)
    csr, sv = D.neighbor_csr_frames(pos, fp, cell, pbc, r_max)
    return csr, sv, fp


def _rows(case, dtype):
    """the oracle's rows: the cell the search saw (rounded to the positions' dtype), zero or missing rows completed"""
    return LO.complete(None if case.cell is None else case.cell.to(dtype).double().numpy(), case.pbc)


def _listed(case, dtype):
    """(i, j, s) rows of the frame alone, in list order"""
    csr, sv, _ = _search([case], dtype, case.r_max)
    ctr, nbr = _check_csr(csr, sv, case.pos, case.pos.shape[0], dtype)
    return _image_rows(ctr, nbr, sv, _rows(case, dtype), case.pbc, dtype), csr, sv


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_neighbor_csr_frames_matches_reference(case, dtype):
    n, r = case.pos.shape[0], case.r_max
    got, csr, sv = _listed(case, dtype)
    csr2, sv2, _ = _search([case], dtype, r)
    assert torch.equal(csr.row_ptr, csr2.row_ptr) and torch.equal(csr.nbr, csr2.nbr) and torch.equal(sv, sv2)
    E = got.shape[0]
    k = O.keys(got, n)
    assert (np.diff(k) > 0).all(), "rows are not ordered by centre, neighbour, then image"
    rows = _rows(case, dtype)
    p64 = case.pos.to(dtype).double()
    band = LO.band_for(p64.numpy(), rows, r, fp32=dtype == torch.float32)
    if E:
        ctr, nbr = torch.from_numpy(got[:, 0]), torch.from_numpy(got[:, 1])
        d = (p64[nbr] + sv.cpu().double() - p64[ctr]).norm(dim=-1)
        assert float(d.max()) < r + band
    ref, dist = LO.pairs(p64.numpy(), rows, case.pbc, r, reach=band)
    n_band, n_band_got = LO.compare(got, ref, dist, r, band, n)
    print(f"\n[nlist-frames] {case.name} {str(dtype)[6:]}: E={E} band={band:.3e} pairs in band {n_band} (listed {n_band_got})")


def _one_atom(r):
    rows = torch.tensor([[4.0, 0.0, 0.0], [1.0, 11.0, 0.0], [2.0, -1.0, 12.0]], dtype=torch.float64)  # sees itself along a
    return LCase("one-periodic", torch.tensor([[0.3, 0.2, 0.1]], dtype=torch.float64), rows, (T, T, T), r)


def _empty(r, periodic):
    cell = torch.eye(3, dtype=torch.float64) * 9.0 if periodic else None
    return LCase("empty", torch.zeros(0, 3, dtype=torch.float64), cell, (periodic,) * 3, r)


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_one_batch_of_every_case(dtype):
    """one batch per r_max: every case, empty frames at the start, middle and end, a one-atom periodic frame; each frame's
    rows and shifts bitwise those of the frame alone, in either frame order"""
    by_r = {}
    for c in CASES:
        by_r.setdefault(c.r_max, []).append(c)
    for r, cs in by_r.items():
        h = len(cs) // 2
        frames = [_empty(r, False)] + cs[:h] + [_one_atom(r), _empty(r, True)] + cs[h:] + [_empty(r, False)]
        alone = {}
        for f in frames:
            csr, sv, _ = _search([f], dtype, r)
            alone[id(f)] = (csr.row_ptr.cpu(), csr.nbr.cpu(), sv.cpu())
        for order in (frames, frames[::-1]):
            csr, sv, fp = _search(order, dtype, r)
            row_ptr, nbr, sv = csr.row_ptr.cpu(), csr.nbr.cpu(), sv.cpu()
            assert int(row_ptr[-1]) == sum(int(a[0][-1]) for a in alone.values())
            for b, f in enumerate(order):
                a0, a1 = int(fp[b]), int(fp[b + 1])
                e0, e1 = int(row_ptr[a0]), int(row_ptr[a1])
                rp1, nbr1, sv1 = alone[id(f)]
                assert torch.equal(row_ptr[a0 : a1 + 1] - e0, rp1), (r, f.name)
                assert torch.equal(nbr[e0:e1] - a0, nbr1), (r, f.name)
                assert torch.equal(sv[e0:e1], sv1), (r, f.name)
        print(f"\n[nlist-frames batch] r_max {r} {str(dtype)[6:]}: {len(frames)} frames, {int(row_ptr[-1])} edges")


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_frames_list_matches_the_cell_list(case, dtype):
    """the two device searches list the same (i, j, s); only pairs inside the band may differ"""
    n, r = case.pos.shape[0], case.r_max
    rows = _rows(case, dtype)
    rows_a, _, _ = _listed(case, dtype)
    pos = case.pos.to(dtype).to(DEV)
    csr, sv = D.neighbor_csr(pos, r, None if case.cell is None else case.cell.to(DEV), case.pbc)
    rows_b = _image_rows(csr.ctr.cpu().long(), csr.nbr.cpu().long(), sv, rows, case.pbc, dtype)
    ka, kb = O.keys(rows_a, n), O.keys(rows_b, n)
    diff = np.setxor1d(ka, kb)
    print(f"\n[nlist-frames vs cell list] {case.name} {str(dtype)[6:]}: E={ka.size} differing rows {diff.size}")
    if diff.size:
        p64 = case.pos.to(dtype).double().numpy()
        both = np.concatenate([rows_a, rows_b])
        centres = np.unique(both[np.isin(O.keys(both, n), diff), 0])
        band = LO.band_for(p64, rows, r, fp32=dtype == torch.float32)
        ref, dist = LO.pairs(p64, rows, case.pbc, r, centres=centres, reach=band)
        rk = O.keys(ref, n)
        assert np.isin(diff, rk).all() and (np.abs(dist[np.isin(rk, diff)] - r) <= band).all()


# --------------------------------------------------------------------------- #
# the model on a batch
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def models():
    from test_gpu_model import _pair

    oracle, model64, _ = _pair("c2", 3, "float64")
    _, model32, _ = _pair("c2", 3, "float32")
    return oracle, {"float64": model64, "float32": model32}


PERIODIC = ["L1-hcp-120deg", "L2-graphite-c6.7", "L2-height-0.4r", "L1-left-handed", "one-periodic"]
OPEN = ["L3-tilted-sheet-TTF", "L4-ase-sheet-zero-c", "L4-ase-wire-zero-ab", "L4-cluster-cell-None", "empty"]


def _model_frames(names, dtype):
    """(case, single-frame dict) per name, positions in the model's dtype on the device"""
    by = {c.name: c for c in nlist_lattice_cases.cases(full_size=False)}
    by["one-periodic"], by["empty"] = _one_atom(5.0), _empty(5.0, False)
    out = []
    for name in names:
        c = by[name]
        f = {D.POSITIONS_KEY: c.pos.to(dtype).to(DEV), D.ATOM_TYPE_KEY: torch.zeros(c.pos.shape[0], dtype=torch.long, device=DEV)}
        if c.cell is not None:
            f[D.CELL_KEY], f[D.PBC_KEY] = c.cell.to(DEV), torch.tensor(c.pbc)
        out.append((c, f))
    return out


def _rel(a, b):
    """relative to max |b|; absolute where b is 0 (the one-atom frame's forces cancel by symmetry)"""
    return float((a - b).abs().max()) / (float(b.abs().max()) or 1.0)


def _check_frames(oracle, cases, parts, tol, stress):
    for c, p in zip(cases, parts):
        n = c.pos.shape[0]
        if n == 0:
            assert float(p[D.TOTAL_ENERGY_KEY].abs().max()) == 0.0 and p[D.CSR_KEY].num_edges == 0
            continue
        pos = p[D.POSITIONS_KEY].double().cpu()  # what the search and the model saw
        ref = _exact(oracle, pos, c.cell, torch.zeros(n, dtype=torch.long), c.pbc, c.r_max)
        e, er = p[D.PER_ATOM_ENERGY_KEY].double().cpu(), ref[D.PER_ATOM_ENERGY_KEY]
        f, fr = p[D.FORCE_KEY].double().cpu(), ref[D.FORCE_KEY]
        errs = [_rel(e, er), _rel(f, fr), abs(float(p[D.TOTAL_ENERGY_KEY].double().sum()) - float(er.sum())) / float(er.abs().sum())]
        if stress:
            errs += [_rel(p[D.STRESS_KEY].double().cpu().reshape(3, 3), ref[D.STRESS_KEY].reshape(3, 3)),
                     _rel(p[D.VIRIAL_KEY].double().cpu().reshape(3, 3), ref[D.VIRIAL_KEY].reshape(3, 3))]
        print(f"\n[frames model] {c.name}: relative errors {['%.2e' % x for x in errs]}")
        assert all(x < tol for x in errs), (c.name, errs)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_model_on_a_batch_matches_the_oracle(models, dtype):
    oracle, by_dtype = models
    inner = getattr(by_dtype[dtype], "model", by_dtype[dtype])
    tol = 1e-9 if dtype == "float64" else 1e-4
    cases, frames = zip(*_model_frames(PERIODIC + OPEN, getattr(torch, dtype)))
    batch = collate(list(frames), 5.0)
    out = inner.energy_and_forces_frames(batch, False)
    _check_frames(oracle, cases, split(out), tol, False)
    # stress needs a volume: refused on the same batch (zero-row sheet and wire, a frame without a cell)
    with pytest.raises(ValueError, match="non-singular"):
        inner.energy_and_forces_frames(batch, True)
    # the periodic subset with stress
    cases, frames = zip(*_model_frames(PERIODIC, getattr(torch, dtype)))
    out = inner.energy_and_forces_frames(collate(list(frames), 5.0), True)
    _check_frames(oracle, cases, split(out), tol, True)
    # a sheet whose open row lies 1e-15 rad from the plane of the periodic rows: the list completes that row, the stress
    # has no volume to divide by
    c, f = _model_frames(["L3-tilted-sheet-TTF"], getattr(torch, dtype))[0]
    rows = c.cell.clone()
    rows[2] = rows[0] + torch.tensor([0.0, 0.0, 1e-14], dtype=torch.float64)
    assert not D.is_regular_cell(rows.to(getattr(torch, dtype)))
    f[D.CELL_KEY] = rows.to(DEV)
    batch = collate(list(frames) + [f], 5.0)
    out = inner.energy_and_forces_frames(batch, False)
    _check_frames(oracle, list(cases) + [LCase("near-coplanar-open-row", c.pos, rows, c.pbc, 5.0)], split(out), tol, False)
    with pytest.raises(ValueError, match="non-singular"):
        inner.energy_and_forces_frames(batch, True)
