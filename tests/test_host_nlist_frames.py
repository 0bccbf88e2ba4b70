"""The host side of the batched-frames neighbour list (``data.neighbor_csr_frames`` / ``data.frames_geometry``) on a
CPU-only box: the cells it refuses before any search, the cells it accepts, and the image counts it hands to
ab2_nl_frames_count / fill.

The search itself is the torch restatement of those kernels in tests/test_host_frames.py; on accepted frames its rows
are held to the fp64 pair search of nlist_lattice_oracle.  A refused frame must never reach ``_lib.nl_frames`` or an
``ab2_nl_frames_*`` entry point: a cell the kernels cannot bound (a height of 1e-30 asks for 2^31 images per axis)
would otherwise run on the device for as long as the walk takes."""
import math

import numpy as np
import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
from allegro_b200 import _lib
from allegro_b200 import data as D
from test_host_frames import nl_frames as spec_nl_frames

DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]
T, F = True, False


class _NoFramesKernels:
    """load() stand-in: reaching an ab2_nl_frames_* entry point fails the test"""

    def __init__(self, load):
        self._load = load

    def __getattr__(self, name):
        if name.startswith("ab2_nl_frames"):
            raise AssertionError(f"{name} was reached")
        return getattr(self._load(), name)


@pytest.fixture()
def searches(monkeypatch):
    """_lib.nl_frames replaced by the torch restatement; every call's arguments are recorded"""
    calls = []

    def spy(*args):
        calls.append(args)
        return spec_nl_frames(*args)

    stub = _NoFramesKernels(_lib.load)
    monkeypatch.setattr(_lib, "load", lambda: stub)
    monkeypatch.setattr(_lib, "nl_frames", spy)
    return calls


def _one(pos, cell, pbc, r, dtype):
    """one-frame batch as collate builds it: cell [1,3,3] in the positions' dtype (or None), pbc [1,3]"""
    p = pos.to(dtype)
    c = None if cell is None else cell.reshape(1, 3, 3).to(dtype)
    return p, torch.tensor([0, p.shape[0]]), c, torch.tensor([pbc])


# --------------------------------------------------------------------------- #
# refused before any search
# --------------------------------------------------------------------------- #
def _refused():
    r = 5.0
    good = torch.tensor([[10.0, 0, 0], [1.0, 11.0, 0], [0.5, -1.0, 12.0]], dtype=torch.float64)
    out = []
    for what, v in (("nan", float("nan")), ("inf", float("inf"))):
        c = good.clone()
        c[1, 1] = v
        out.append((f"{what}-periodic-row", c, (T, T, T), r, "not finite"))
        out.append((f"{what}-periodic-row-TTF", c, (T, T, F), r, "not finite"))
    c = good.clone()
    c[1] = 0.0
    out.append(("zero-periodic-row", c, (T, T, T), r, "near-coplanar"))
    out.append(("zero-periodic-row-TFF", torch.tensor([[0.0, 0, 0], [0, 9, 0], [0, 0, 0]], dtype=torch.float64), (T, F, F), r,
                "near-coplanar"))
    out.append(("zero-periodic-row-TTF", c, (T, T, F), r, "near-coplanar"))  # the periodic rows have no normal to complete
    out.append(("coplanar-1e-30", torch.tensor([[5.0, 0, 0], [0, 5.0, 0], [5.0, 5.0, 1e-30]], dtype=torch.float64), (T, T, T), r,
                "near-coplanar"))
    # rows 1e-13 rad from a common plane: |det| = 1e-13 |a| |b| |c| sin(angle of a, b) < 1e-12 |a| |b| |c|
    a, b = good[0], good[1]
    u = torch.linalg.cross(a, b)
    cc = 0.6 * a - 0.3 * b + 1e-13 * float(a.norm()) * u / u.norm()
    out.append(("coplanar-1e-13-rad", torch.stack([a, b, cc]), (T, T, T), r, "near-coplanar"))
    out.append(("coplanar-periodic-rows-TTF", torch.stack([a, 2.0 * a, good[2]]), (T, T, F), r, "near-coplanar"))
    # past the image budget: heights 0.002 r_max on every axis (2001^3 images), one axis 1e-6 r_max (2e6 + 1)
    out.append(("budget-0.002r", torch.eye(3, dtype=torch.float64) * (0.002 * r), (T, T, T), r, "images per pair"))
    out.append(("budget-one-axis", torch.diag(torch.tensor([16.0, 16.0, 1e-6 * r], dtype=torch.float64)), (T, T, T), r,
                "images per pair"))
    # (2 * 51 + 1)^3 = 1092727 > 2^20: heights 0.125, r_max 51 * 0.125
    out.append(("budget-51-per-axis", torch.eye(3, dtype=torch.float64) * 0.125, (T, T, T), 51 * 0.125, "images per pair"))
    return out


REFUSED = _refused()


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("name,cell,pbc,r,match", REFUSED, ids=[c[0] for c in REFUSED])
def test_refused_before_any_search(name, cell, pbc, r, match, dtype, searches):
    pos = torch.tensor([[0.1, 0.2, 0.3], [1.0, 1.5, 0.5]], dtype=torch.float64)
    with pytest.raises(ValueError, match=match):
        D.neighbor_csr_frames(*_one(pos, cell, pbc, r, dtype), r)
    # and inside a batch: frame 1 of three, the others fine
    good = torch.eye(3, dtype=torch.float64) * 12.0
    cells = torch.stack([good, cell, good]).to(dtype)
    pbcs = torch.tensor([(T, T, T), pbc, (F, F, F)])
    pos3 = torch.cat([pos, pos, pos]).to(dtype)
    with pytest.raises(ValueError, match="frame 1 "):
        D.neighbor_csr_frames(pos3, torch.tensor([0, 2, 4, 6]), cells, pbcs, r)
    with pytest.raises(ValueError, match=match):
        D.frames_geometry(cell.reshape(1, 3, 3), torch.tensor([pbc]), r, dtype)
    assert searches == []


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("name,cell,pbc,r,match", [c for c in REFUSED if "budget" in c[0] or "1e-30" in c[0]],
                         ids=[c[0] for c in REFUSED if "budget" in c[0] or "1e-30" in c[0]])
def test_the_kernel_wrapper_refuses_before_any_launch(name, cell, pbc, r, match, dtype, monkeypatch):
    """_lib.nl_frames called directly (not through neighbor_csr_frames) still computes and bounds the image counts on the
    host: no ab2_nl_frames_* entry point is reached"""
    stub = _NoFramesKernels(_lib.load)
    monkeypatch.setattr(_lib, "load", lambda: stub)
    pos = torch.tensor([[0.1, 0.2, 0.3], [1.0, 1.5, 0.5]], dtype=dtype)
    c = cell.to(dtype).reshape(1, 3, 3)
    with pytest.raises(ValueError, match=match):
        _lib.nl_frames(pos, torch.tensor([0, 2], dtype=torch.int32), c, torch.zeros_like(c), torch.tensor([pbc], dtype=torch.int32), r)


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_periodic_frames_need_a_cell(dtype, searches):
    pos = torch.rand(3, 3, dtype=dtype)
    with pytest.raises(ValueError, match="need a cell"):
        D.neighbor_csr_frames(pos, torch.tensor([0, 3]), None, (T, F, F), 5.0)
    with pytest.raises(ValueError, match="need a cell"):
        D.neighbor_csr_frames(torch.cat([pos, pos]), torch.tensor([0, 3, 6]), None, torch.tensor([(F, F, F), (F, T, F)]), 5.0)
    assert searches == []


def test_the_budget_is_inclusive(searches):
    # (2 * 50 + 1)^3 = 1030301 <= 2^20 images: accepted (geometry only; the search is not run)
    rows, nimg = D.frames_geometry((torch.eye(3, dtype=torch.float64) * 0.125).reshape(1, 3, 3), torch.tensor([(T, T, T)]), 6.25)
    assert nimg.tolist() == [[50, 50, 50]] and math.prod(2 * k + 1 for k in nimg[0].tolist()) <= D.FRAMES_MAX_IMAGES
    _, nimg = D.frames_geometry(torch.diag(torch.tensor([0.125, 16.0, 16.0], dtype=torch.float64)).reshape(1, 3, 3),
                                torch.tensor([(T, T, T)]), 6.25)
    assert nimg.tolist() == [[50, 1, 1]]


# --------------------------------------------------------------------------- #
# accepted: ASE zero open rows, cell=None, degenerate open rows; the restated search against the oracle
# --------------------------------------------------------------------------- #
def _accepted():
    by_name = {c.name: c for c in nlist_lattice_cases.cases(full_size=False)}
    out = [(n, by_name[n].pos, by_name[n].cell, by_name[n].pbc, by_name[n].r_max)
           for n in ("L4-ase-sheet-zero-c", "L4-ase-wire-zero-ab", "L4-cluster-cell-None", "L3-tilted-sheet-TTF")]
    pos, rows = nlist_lattice_cases.tilted_sheet(21)
    bad = rows.clone()
    bad[2] = float("inf")
    out.append(("TTF-inf-open-row", pos, bad, (T, T, F), 5.0))
    bad = rows.clone()
    bad[2] = rows[0] + rows[1]  # open row in the plane of the periodic ones
    out.append(("TTF-coplanar-open-row", pos, bad, (T, T, F), 5.0))
    bad = torch.full((3, 3), float("nan"), dtype=torch.float64)
    out.append(("FFF-nan-cell", nlist_lattice_cases.cluster(), bad, (F, F, F), 5.0))
    pos, rows = nlist_lattice_cases.tilted_wire(22, zero_rows=True)
    out.append(("FTF-zero-rows", pos[:, [0, 2, 1]], rows[:, [0, 2, 1]][[0, 2, 1]], (F, T, F), 5.0))
    return out


ACCEPTED = _accepted()


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("name,pos,cell,pbc,r", ACCEPTED, ids=[c[0] for c in ACCEPTED])
def test_accepted_frames_list_the_oracle_pairs(name, pos, cell, pbc, r, dtype, searches):
    p, fp, c, pb = _one(pos, cell, pbc, r, dtype)
    csr, sv = D.neighbor_csr_frames(p, fp, c, pb, r)
    assert len(searches) == 1
    rows_seen, _, pbc_seen, r_seen = searches[0][2:]
    assert float(r_seen) == r and pbc_seen.tolist() == [list(pbc)]
    assert bool(torch.isfinite(rows_seen).all())  # completed: no zero, non-finite or coplanar open row is searched
    # the kernels' image counts (_lib.nl_frames): the completed rows unchanged, images on the periodic axes only
    rows2, nimg = D.frames_geometry(rows_seen, pbc_seen != 0, r, dtype)
    assert torch.equal(rows2.to(dtype), rows_seen)
    for a in range(3):
        assert (int(nimg[0, a]) > 0) == pbc[a]
    # the oracle completes zero rows; a non-finite open row is as good as none
    rows = LO.complete(None if c is None else np.nan_to_num(c[0].double().numpy(), nan=0.0, posinf=0.0, neginf=0.0), pbc)
    img, dev = LO.images_of(sv.double().numpy(), rows)
    assert dev <= (1e-5 if dtype == torch.float32 else 1e-12), dev
    for a in range(3):
        if not pbc[a]:
            assert (img[:, a] == 0).all(), a
    if not any(pbc):
        assert bool((sv == 0).all())
    got = np.concatenate([csr.ctr.long().numpy()[:, None], csr.nbr.long().numpy()[:, None], img], 1)
    p64 = p.double().numpy()
    band = LO.band_for(p64, rows, r, fp32=dtype == torch.float32)
    ref, dist = LO.pairs(p64, rows, pbc, r, reach=band)
    assert ref.shape[0] > 0
    LO.compare(got, ref, dist, r, band, p64.shape[0])


# --------------------------------------------------------------------------- #
# image counts
# --------------------------------------------------------------------------- #
def _all_cases():
    out = []
    for c in nlist_cases.cases(full_size=False):
        out.append((c.name, c.pos, c.cell, c.pbc, c.r_max))
    for c in nlist_lattice_cases.cases(full_size=False):
        out.append((c.name, c.pos, c.cell, c.pbc, c.r_max))
    return out


ALL = _all_cases()


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_image_counts_cover_every_oracle_pair(dtype):
    """nimg = ceil(r_max / H) with H from the oracle's heights, and no oracle pair needs an image beyond it (images counted
    from the search's own wrap: floor of the fractional coordinates in the rows it is given)"""
    for name, pos, cell, pbc, r in ALL:
        if not any(pbc):
            continue
        rows, nimg = D.frames_geometry(cell.reshape(1, 3, 3), torch.tensor([pbc]), r, dtype)
        rows, nimg = rows[0].numpy(), nimg[0].tolist()
        H = LO.heights(rows)
        for a in range(3):
            if not pbc[a]:
                assert nimg[a] == 0, (name, a)
                continue
            q = r / H[a]
            if abs(q - round(q)) > 8 * np.spacing(q):
                assert nimg[a] == math.ceil(q), (name, a, nimg[a], q)
            else:  # an integer ratio, to within the rounding of two fp64 height formulas
                assert nimg[a] in (round(q), round(q) + 1), (name, a, nimg[a], q)
        p64 = pos.to(dtype).double().numpy()
        if p64.shape[0] == 0:
            continue
        ref, _ = LO.pairs(p64, LO.complete(rows, pbc), pbc, r)
        frac = np.linalg.solve(rows.T, p64.T).T
        img0 = np.where(pbc, np.floor(frac), 0).astype(np.int64)
        need = ref[:, 2:] + img0[ref[:, 1]] - img0[ref[:, 0]]  # image of the wrapped neighbour
        assert (np.abs(need) <= np.array(nimg)).all(), (name, np.abs(need).max(0).tolist(), nimg)


def _nextafter(x, toward, dtype):
    if dtype == torch.float32:
        return float(np.nextafter(np.float32(x), np.float32(toward)))
    return float(np.nextafter(x, toward))


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_image_counts_at_integer_ratios(dtype):
    """r_max / H an integer k, and H one ulp (of the positions' dtype) either side: k, k, k + 1 images.  An fp64 ulp is
    lost when the cell is rounded to fp32, so fp32 positions then search k."""
    r = 5.0
    for k in (1, 2, 4, 8):
        h = r / k  # exact
        heights = [(h, k), (_nextafter(h, math.inf, dtype), k), (_nextafter(h, 0.0, dtype), k + 1)]
        if dtype == torch.float32:
            heights += [(_nextafter(h, math.inf, torch.float64), k), (_nextafter(h, 0.0, torch.float64), k)]
        for hh, want in heights:
            for axis in range(3):
                d = [8.0, 16.0, 32.0]  # powers of two: every height of the cell is exact in fp64
                d[axis] = hh
                cell = torch.diag(torch.tensor(d, dtype=torch.float64))
                _, nimg = D.frames_geometry(cell.reshape(1, 3, 3), torch.tensor([(T, T, T)]), r, dtype)
                assert nimg[0, axis] == want, (k, hh, axis, nimg.tolist())
                # the oracle's height agrees to its last bits (its determinant is an LU product, not exact here)
                H = LO.heights(cell.to(dtype).double().numpy())
                assert abs(H[axis] - float(torch.tensor(hh).to(dtype))) <= 4 * np.spacing(hh)
                assert nimg[0].tolist() == [want if a == axis else 1 for a in range(3)]


def test_batched_regularity_is_the_single_frame_one():
    cells = [c for _, _, c, _, _ in ALL if c is not None]
    g = torch.Generator().manual_seed(3)
    cells += [torch.randn(3, 3, generator=g, dtype=torch.float64) for _ in range(50)]
    cells += [c for _, c, _, _, _ in REFUSED]
    h = torch.stack(cells)
    regular, heights = D._lattice_metrics_batched(h)
    for b, c in enumerate(cells):
        _, hs, reg = D._lattice_metrics(c.tolist())
        assert bool(regular[b]) == reg == D.is_regular_cell(c)
        if reg:
            assert heights[b].tolist() == hs  # bitwise: the same operations in the same order
    assert torch.equal(D.regular_cells(h), regular)
