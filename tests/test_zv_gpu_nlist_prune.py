"""ab2_nl_prune_count / fill through ``data.prune_csr`` on every geometry of nlist_cases and nlist_lattice_cases, in fp64 and
fp32: bitwise the torch restatement (tests/nlist_prune_spec.py), each row an ordered subsequence of the unpruned row, the
kept pairs those of the fp64 oracle away from the band of their own cutoff, a table at r_max everywhere a no-op, a
second call the same bits; rows for n_centres < n, empty frames, one atom and zero-edge lists; and ``collate(...,
cutoffs)`` on a mixed batch, frame by frame against the pruned single-frame list."""
import numpy as np
import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
import nlist_prune_spec as PS
from allegro_b200 import data as D

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _geometries():
    """(name, pos, cell or None, oracle rows, pbc, r_max, n_centres, ref_centres)"""
    out = []
    for c in nlist_cases.cases():
        out.append((c.name, c.pos, c.cell, c.cell.numpy(), c.pbc, c.r_max, c.n_centres, c.ref_centres))
    for c in nlist_lattice_cases.cases():
        rows = LO.complete(None if c.cell is None else c.cell.numpy(), c.pbc)
        out.append((c.name, c.pos, c.cell, rows, c.pbc, c.r_max, None, c.ref_centres))
    return out


GEOMS = _geometries()


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_prune_kernel(geom, dtype):
    name, pos64, cell, rows, pbc, r, nc, ref_centres = geom
    pos = pos64.to(dtype)
    n = pos.shape[0]
    nc = n if nc is None else nc
    posd = pos.to(DEV)
    celld = None if cell is None else cell.to(DEV)
    csr, sv = D.neighbor_csr(posd, r, celld, pbc, n_centres=nc)
    assert csr.radius == r
    T = 3
    seed = sum(map(ord, name))
    types, table = PS.random_types(n, T, seed), PS.random_table(T, r, seed + 1)
    td, tabd = types.to(DEV), table.to(DEV)
    out, sv_p = D.prune_csr(csr, sv, posd, td, tabd)
    got = (out.row_ptr, out.nbr, sv_p)
    # bitwise the restatement, on the device
    want = PS.nl_prune(posd, csr.row_ptr, csr.nbr, sv, td.to(torch.int32), tabd * tabd)
    assert _same(got, want), name
    assert sv_p.dtype == dtype and out.num_atoms == nc and out.num_edges == out.nbr.shape[0] <= csr.num_edges
    counts = (out.row_ptr[1:] - out.row_ptr[:-1]).long()
    assert torch.equal(out.ctr, torch.repeat_interleave(torch.arange(nc, device=DEV, dtype=torch.int32), counts))
    assert out.max_degree == (int(counts.max()) if nc else 0)
    # a second call: the same bits
    again, sv_a = D.prune_csr(csr, sv, posd, td, tabd)
    assert _same(got, (again.row_ptr, again.nbr, sv_a))
    # a table at r_max everywhere: the unpruned list, bitwise.  The search decides its pairs on wrapped positions (in fp32
    # for an fp32 orthorhombic frame), this test on the raw ones in fp64, so a pair within the band of r_max (the lattice
    # with r_max on its nearest-neighbour shell) may go; nothing else may.
    p64 = pos.double()
    band = LO.band_for(p64.numpy(), rows, r, fp32=dtype == torch.float32)
    full, sv_f = D.prune_csr(csr, sv, posd, td, torch.full((T, T), r, dtype=torch.float64, device=DEV))
    if not _same((full.row_ptr, full.nbr, sv_f), (csr.row_ptr, csr.nbr, sv)):
        assert PS.is_ordered_subsequence(csr.row_ptr, csr.nbr, sv, full.row_ptr, full.nbr, sv_f), name
        pd = posd.double()
        d = ((pd[csr.nbr.long()] + sv.double()) - pd[csr.ctr.long()]).norm(dim=-1)
        n_dropped = csr.num_edges - full.num_edges
        assert int(((d - r).abs() <= band).sum()) >= n_dropped > 0 and bool((d[d >= r] - r <= band).all()), name
        print(f"\n[prune] {name} {str(dtype)[6:]}: a table at r_max drops {n_dropped} edges within the band of r_max")
    # ordered subsequences (checked directly on the smaller frames; on the larger ones it follows from the restatement,
    # a masked selection)
    if csr.num_edges <= 50_000:
        assert PS.is_ordered_subsequence(csr.row_ptr, csr.nbr, sv, out.row_ptr, out.nbr, sv_p)
    # kept pairs against the fp64 oracle, outside the band of their own cutoff
    centres = np.arange(nc)
    if ref_centres is not None:
        centres = np.sort(np.random.default_rng(0).choice(nc, ref_centres, replace=False))
    ref, dist = LO.pairs(p64.numpy(), rows, pbc, r, centres=centres, reach=band)
    ctr = out.ctr.cpu().long().numpy()
    img, dev = LO.images_of(sv_p.double().cpu().numpy(), rows)
    got_rows = np.concatenate([ctr[:, None], out.nbr.cpu().long().numpy()[:, None], img], 1)
    n_band, kept = PS.compare_pruned(got_rows[np.isin(ctr, centres)], ref, dist, types.numpy(), table.numpy(), band, n)
    print(f"\n[prune] {name} {str(dtype)[6:]}: E {csr.num_edges} -> {out.num_edges}, in band {n_band} (kept {kept})")


def test_zero_centres_zero_edges_and_one_atom():
    cell = torch.eye(3, dtype=torch.float64, device=DEV) * 30
    for n, nc in ((0, 0), (1, 1), (5, 0)):
        pos = torch.rand(n, 3, dtype=torch.float64, device=DEV) * 10
        csr, sv = D.neighbor_csr(pos, 3.0, cell, (False, False, False), n_centres=nc)
        out, sv_p = D.prune_csr(csr, sv, pos, torch.zeros(n, dtype=torch.long, device=DEV), torch.full((1, 1), 2.0, dtype=torch.float64))
        assert out.num_atoms == nc and out.num_edges == 0 and sv_p.shape == (0, 3) and torch.equal(out.row_ptr, csr.row_ptr)
    # centres whose rows are all empty (atoms far apart), then a list whose every edge goes
    pos = torch.tensor([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0], [20.0, 0.0, 0.0], [21.0, 0.0, 0.0]], dtype=torch.float32, device=DEV)
    csr, sv = D.neighbor_csr(pos, 3.0, None, (False, False, False))
    assert csr.num_edges == 2
    types = torch.tensor([0, 1, 0, 1], device=DEV)
    tab = torch.tensor([[3.0, 0.5], [3.0, 3.0]], dtype=torch.float64)  # 2 -> 3 (type 0 -> 1) dropped, 3 -> 2 kept
    out, sv_p = D.prune_csr(csr, sv, pos, types, tab)
    assert out.row_ptr.tolist() == [0, 0, 0, 0, 1] and out.nbr.tolist() == [2] and out.ctr.tolist() == [3]
    out, sv_p = D.prune_csr(csr, sv, pos, types, torch.full((2, 2), 0.5, dtype=torch.float64))
    assert out.num_edges == 0 and out.row_ptr.tolist() == [0] * 5 and out.max_degree == 0


def test_neighbor_csr_with_cutoffs_is_search_then_prune():
    pos, cell, types = (t.to(DEV) for t in __import__("allegro_b200.systems", fromlist=["x"]).make_positions("c3", 8))
    tab = torch.tensor([[4.0, 5.0, 5.5], [5.0, 4.5, 6.0], [5.5, 5.5, 5.5]], dtype=torch.float64)
    for dt in (torch.float64, torch.float32):
        p = pos.to(dt)
        csr, sv = D.neighbor_csr(p, 6.0, cell, (True, True, True))
        a, sva = D.neighbor_csr(p, 6.0, cell, (True, True, True), types=types, cutoffs=tab)
        b, svb = D.prune_csr(csr, sv, p, types, tab)
        assert _same((a.row_ptr, a.nbr, sva), (b.row_ptr, b.nbr, svb)) and a.num_edges < csr.num_edges


def _batch_frames():
    """frames of the geometry matrix a batched search takes: periodic and open, orthorhombic and triclinic, a cluster
    without a cell, one atom"""
    want = {"G3-pbcTTT", "G3-pbcTFT", "G4-graphene-TTF", "G4-one-FFF", "G6-dense"}
    frames = []
    for c in nlist_cases.cases(full_size=False):
        if c.name in want:
            frames.append((c.pos, c.cell, c.pbc))
    for c in nlist_lattice_cases.cases():
        if c.pos.shape[0] <= 1500 and len(frames) < 9:
            pbc = torch.tensor(c.pbc).view(1, 3)
            try:  # the frames the batched search takes (few enough images per pair)
                D.frames_geometry(None if c.cell is None else c.cell.view(1, 3, 3), pbc, 5.0)
            except ValueError:
                continue
            frames.append((c.pos, c.cell, c.pbc))
    return frames


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
def test_collate_with_cutoffs_frame_by_frame(dtype):
    from allegro_b200.batch import collate, split

    r = 5.0
    T = 3
    table = PS.random_table(T, r, 77)
    frames = []
    for k, (pos, cell, pbc) in enumerate(_batch_frames()):
        f = {D.POSITIONS_KEY: pos.to(DEV, dtype), D.ATOM_TYPE_KEY: PS.random_types(pos.shape[0], T, 100 + k).to(DEV),
             D.PBC_KEY: torch.tensor(pbc)}
        if cell is not None:
            f[D.CELL_KEY] = cell.to(DEV, dtype)
        frames.append(f)
    assert len(frames) >= 8
    batch = collate(frames, r, cutoffs=table)
    full = collate(frames, r)
    assert batch[D.CSR_KEY].num_edges < full[D.CSR_KEY].num_edges
    for f, part in zip(frames, split(batch)):
        one = collate([f], r, cutoffs=table)
        csr, one_csr = part[D.CSR_KEY], one[D.CSR_KEY]
        assert torch.equal(csr.row_ptr, one_csr.row_ptr) and torch.equal(csr.nbr, one_csr.nbr) and torch.equal(csr.ctr, one_csr.ctr)
        assert torch.equal(part[D.EDGE_SHIFT_VEC_KEY], one[D.EDGE_SHIFT_VEC_KEY])
