"""Per-edge-type pruning of the neighbour list on the HOST side, without a GPU.

* The torch restatement of ab2_nl_prune_count / fill (tests/nlist_prune_spec.py) against the fp64 numpy pair search of
  nlist_lattice_oracle, on the geometries of nlist_cases and nlist_lattice_cases (frames of at most 3000 atoms: the
  all-pairs oracle), with seeded random types and directed tables spanning 0.4 - 1.0 r_max.
* Every refusal of ``data.prune_csr`` / ``neighbor_csr`` / ``neighbor_csr_frames`` / ``collate`` is raised before any
  launch: the wrappers are replaced by functions that fail the test.
* ``collate(..., cutoffs)`` and ``AllegroCalculator(prune_edges=True)`` with the restatement and tests/kernel_spec.py
  swapped in (as tests/test_host_pipeline.py does): the pruned lists give the energies, forces and stress of the
  unpruned ones and of the reference-pinned oracle on exact r_max lists.
The kernels themselves are checked on the GPU (tests/test_zv_gpu_nlist_prune.py).
"""
import numpy as np
import pytest
import torch

import kernel_spec
import nlist_cases
import nlist_lattice_cases
import nlist_lattice_oracle as LO
import nlist_prune_spec as PS
from golden_util import load_models, unpack_state_dict

MODELS = {r["name"]: r for r in load_models()}


def _geometries():
    """(name, pos, search cell or None, oracle rows, pbc, r_max, n_centres) of every frame of at most 3000 atoms"""
    out = []
    for c in nlist_cases.cases(full_size=False):
        out.append((c.name, c.pos, c.cell, c.cell.numpy(), c.pbc, c.r_max, c.n_centres))
    for c in nlist_lattice_cases.cases():
        if c.pos.shape[0] <= 3000:
            rows = LO.complete(None if c.cell is None else c.cell.numpy(), c.pbc)
            out.append((c.name, c.pos, c.cell, rows, c.pbc, c.r_max, None))
    return out


GEOMS = _geometries()


def _oracle_list(pos, rows, pbc, r_max, nc, band):
    """unpruned rows of centres [0, nc) from the oracle (pairs within r_max + band), as the device lists carry them"""
    ref, dist = LO.pairs(pos.double().numpy(), rows, pbc, r_max, centres=np.arange(nc), reach=band)
    sel = dist < r_max
    rows_in = ref[sel]
    order = np.argsort(rows_in[:, 0], kind="stable")
    rows_in = rows_in[order]
    row_ptr = torch.zeros(nc + 1, dtype=torch.int32)
    row_ptr[1:] = torch.cumsum(torch.bincount(torch.from_numpy(rows_in[:, 0]), minlength=nc), 0).to(torch.int32)
    nbr = torch.from_numpy(rows_in[:, 1]).to(torch.int32)
    shift = (torch.from_numpy(rows_in[:, 2:]).double() @ torch.from_numpy(np.asarray(rows, dtype=np.float64))).to(pos.dtype).contiguous()
    return row_ptr, nbr, shift, ref, dist


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_restatement_matches_the_oracle(geom, dtype):
    name, pos64, _, rows, pbc, r, nc = geom
    pos = pos64.to(dtype)
    n = pos.shape[0]
    nc = n if nc is None else nc
    band = LO.band_for(pos.double().numpy(), rows, r, fp32=dtype == torch.float32)
    row_ptr, nbr, shift, ref, dist = _oracle_list(pos, rows, pbc, r, nc, band)
    T = 3
    seed = sum(map(ord, name))
    types, table = PS.random_types(n, T, seed), PS.random_table(T, r, seed + 1)
    rp, nb, sh = PS.nl_prune(pos, row_ptr, nbr, shift, types.to(torch.int32), table * table)
    assert rp.dtype == torch.int32 and nb.dtype == torch.int32 and sh.dtype == dtype
    assert PS.is_ordered_subsequence(row_ptr, nbr, shift, rp, nb, sh)
    ctr = torch.repeat_interleave(torch.arange(nc), (rp[1:] - rp[:-1]).long())
    img, dev = LO.images_of(sh.double().numpy(), rows)
    assert dev <= (1e-5 if dtype == torch.float32 else 1e-12) * max(1.0, float(np.abs(rows).max()) * 10)
    got = np.concatenate([ctr.numpy()[:, None], nb.long().numpy()[:, None], img], 1)
    n_band, kept = PS.compare_pruned(got, ref, dist, types.numpy(), table.numpy(), band, n)
    print(f"\n[prune] {name} {str(dtype)[6:]}: E {nbr.shape[0]} -> {nb.shape[0]}, in band {n_band} (kept {kept})")
    if nbr.shape[0]:
        # the table spans 0.4 - 1.0 r_max: something goes unless every pair is short
        assert nb.shape[0] <= nbr.shape[0]


def test_restatement_with_table_at_r_max_keeps_everything():
    name, pos, _, rows, pbc, r, nc = next(g for g in GEOMS if g[0].startswith("G6-dense"))
    n = pos.shape[0]
    band = LO.band_for(pos.numpy(), rows, r, fp32=False)
    row_ptr, nbr, shift, _, dist = _oracle_list(pos, rows, pbc, r, n, band)
    # the oracle's pairs are those with fp64 distance < r_max; the restatement's d2 < r^2 agrees away from the boundary
    assert not np.any(np.abs(dist[dist < r] - r) < 1e-9)
    tab = torch.full((2, 2), r, dtype=torch.float64)
    rp, nb, sh = PS.nl_prune(pos, row_ptr, nbr, shift, PS.random_types(n, 2, 1).to(torch.int32), tab * tab)
    assert torch.equal(rp, row_ptr) and torch.equal(nb, nbr) and torch.equal(sh, shift)


# --------------------------------------------------------------------------- #
# refusals: raised before anything is launched
# --------------------------------------------------------------------------- #
@pytest.fixture()
def no_launch(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200 import data as D

    def launched(*a, **k):
        raise AssertionError("a kernel was launched")

    for name in ("nl_prune", "neighbor_csr", "neighbor_csr_lattice", "nl_frames"):
        monkeypatch.setattr(_lib, name, launched)
    # neighbor_csr takes CPU positions here (its search is replaced above)
    monkeypatch.setattr(D, "_csr_grid", lambda pos, r_max, cell, pbc: D.search_grid(pos, r_max, cell, pbc))


def _small():
    from allegro_b200 import data as D

    g = torch.Generator().manual_seed(5)
    cell = torch.eye(3, dtype=torch.float64) * 16.0
    pos = torch.rand(40, 3, generator=g, dtype=torch.float64) * 16.0
    types = torch.randint(0, 2, (40,), generator=g)
    ei, sh = D.neighbor_list(pos, 5.0, cell, (True, True, True))
    csr = D.build_csr(ei, 40)
    return pos, cell, types, csr, (sh @ cell).contiguous()


BAD_TABLES = {
    "not_square": torch.full((2, 3), 4.0, dtype=torch.float64),
    "one_dim": torch.full((4,), 4.0, dtype=torch.float64),
    "empty": torch.zeros(0, 0, dtype=torch.float64),
    "nan": torch.tensor([[4.0, float("nan")], [4.0, 4.0]], dtype=torch.float64),
    "inf": torch.tensor([[4.0, float("inf")], [4.0, 4.0]], dtype=torch.float64),
    "zero": torch.tensor([[4.0, 0.0], [4.0, 4.0]], dtype=torch.float64),
    "negative": torch.tensor([[4.0, 4.0], [-1.0, 4.0]], dtype=torch.float64),
    "above_r_list": torch.tensor([[4.0, 4.0], [5.0 + 1e-12, 4.0]], dtype=torch.float64),
}


@pytest.mark.parametrize("bad", list(BAD_TABLES), ids=list(BAD_TABLES))
def test_bad_tables_are_refused_before_any_launch(bad, no_launch):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    pos, cell, types, csr, sv = _small()
    tab = BAD_TABLES[bad]
    with pytest.raises(ValueError):
        D.prune_csr(csr, sv, pos, types, tab, r_list=5.0)
    with pytest.raises(ValueError):
        D.neighbor_csr(pos, 5.0, cell, (True, True, True), types=types, cutoffs=tab)
    with pytest.raises(ValueError):
        D.neighbor_csr_frames(pos, torch.tensor([0, 40]), cell.view(1, 3, 3), (True, True, True), 5.0, types=types, cutoffs=tab)
    with pytest.raises(ValueError):
        collate([{"pos": pos, "atom_types": types, "cell": cell}], 5.0, cutoffs=tab)


def test_bad_types_and_missing_arguments_are_refused_before_any_launch(no_launch):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    pos, cell, types, csr, sv = _small()
    tab = torch.full((2, 2), 4.0, dtype=torch.float64)
    for t in (types[:-1], torch.cat([types, types[:1]]), torch.full_like(types, 2), torch.full_like(types, -1), types.double()):
        with pytest.raises(ValueError):
            D.prune_csr(csr, sv, pos, t, tab, r_list=5.0)
        with pytest.raises(ValueError):
            D.neighbor_csr(pos, 5.0, cell, (True, True, True), types=t, cutoffs=tab)
    with pytest.raises(ValueError):  # the radius of a list built from a COO edge_index is not known
        D.prune_csr(csr, sv, pos, types, tab)
    with pytest.raises(ValueError):
        D.neighbor_csr(pos, 5.0, cell, (True, True, True), cutoffs=tab)
    with pytest.raises(ValueError):
        D.neighbor_csr(pos, 5.0, cell, (True, True, True), types=types)
    ei, sh = D.neighbor_list(pos, 5.0, cell, (True, True, True))
    with pytest.raises(ValueError):  # frames that bring their own list
        collate([{"pos": pos, "atom_types": types, "cell": cell, "edge_index": ei, "edge_cell_shift": sh}], 5.0, cutoffs=tab)


def test_prune_csr_rebuilds_ctr_and_max_degree(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200 import data as D

    monkeypatch.setattr(_lib, "nl_prune", PS.nl_prune)
    pos, cell, types, csr, sv = _small()
    tab = torch.tensor([[3.0, 4.5], [2.5, 5.0]], dtype=torch.float64)
    out, sv2 = D.prune_csr(csr, sv, pos, types, tab, r_list=5.0)
    counts = out.row_ptr[1:] - out.row_ptr[:-1]
    assert out.num_atoms == 40 and out.num_edges == out.nbr.shape[0] == sv2.shape[0] < csr.num_edges
    assert torch.equal(out.ctr, torch.repeat_interleave(torch.arange(40, dtype=torch.int32), counts.long()))
    assert out.max_degree == int(counts.max()) and out.perm is None and out.radius is None
    assert out.ctr.dtype == torch.int32 and out.nbr.dtype == torch.int32


# --------------------------------------------------------------------------- #
# collate and the MD calculator with the restated kernels
# --------------------------------------------------------------------------- #
@pytest.fixture()
def spec_kernels(monkeypatch):
    import test_host_frames as HF
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    for name, fn in HF.BATCH_SPEC.items():
        monkeypatch.setattr(_lib, name, fn)
    monkeypatch.setattr(_lib, "nl_prune", PS.nl_prune)
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))
    monkeypatch.setattr(FusedAllegroEnergy, "energy_and_forces",
                        lambda self, data, stress=False, atomic_virial=False, heat_current=False: self._energy_and_forces(data, stress, atomic_virial, heat_current))


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0) if b.numel() else 0.0


@pytest.mark.parametrize("name", ["per_edge_type_cutoff", "spline_embed_per_edge_type_cutoff"])
def test_collate_with_cutoffs(name, spec_kernels):
    import test_host_frames as HF
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    rec = MODELS[name]
    kw = rec["kwargs"]
    _, model = HF._models(kw, unpack_state_dict(rec["state_dict"]))
    frames = HF._mixed_frames(rec["data"], kw["r_max"], len(kw["type_names"]), seed=4, periodic_only=True)
    frames = [{k: v for k, v in f.items() if k not in (D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY)} for f in frames]
    tab = model.edge_norm.rmax_table
    full = collate(frames, kw["r_max"])
    pruned = collate(frames, kw["r_max"], cutoffs=tab)
    assert 0 < pruned[D.CSR_KEY].num_edges < full[D.CSR_KEY].num_edges
    types = full[D.ATOM_TYPE_KEY].to(torch.int32)
    rp, nb, sh = PS.nl_prune(full[D.POSITIONS_KEY], full[D.CSR_KEY].row_ptr, full[D.CSR_KEY].nbr, full[D.EDGE_SHIFT_VEC_KEY], types, tab * tab)
    assert torch.equal(pruned[D.CSR_KEY].row_ptr, rp) and torch.equal(pruned[D.CSR_KEY].nbr, nb) and torch.equal(pruned[D.EDGE_SHIFT_VEC_KEY], sh)
    a = model._energy_and_forces_frames(full, True)
    b = model._energy_and_forces_frames(pruned, True)
    for k in (D.TOTAL_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.STRESS_KEY):
        assert _rel(b[k], a[k]) < 1e-12, (k, _rel(b[k], a[k]))


def test_calculator_prune_edges_under_the_md_driver(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.calculator import AllegroCalculator
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    rec = MODELS["per_edge_type_cutoff"]
    sd = unpack_state_dict(rec["state_dict"])
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(sd, strict=True)
    oracle = AllegroOracle(**rec["kwargs"])
    oracle.load_state_dict(sd, strict=True)
    r_max = rec["kwargs"]["r_max"]
    d = rec["data"]
    pos, cell, types = d[D.POSITIONS_KEY], d[D.CELL_KEY], d[D.ATOM_TYPE_KEY]
    calc = AllegroCalculator(model, r_max, skin=0.5, use_graph=False, compute_stress=True, prune_edges=True)
    plain = AllegroCalculator(model, r_max, skin=0.5, use_graph=False, compute_stress=True)
    tab = model.model.edge_norm.rmax_table
    assert torch.equal(calc._cutoffs, tab + 0.5) and calc.r_list == float(tab.max()) + 0.5
    g = torch.Generator().manual_seed(8)
    p = pos.clone()
    for _ in range(4):
        out = calc.compute(p, cell, types)
        out_plain = plain.compute(p, cell, types)
        assert calc.num_edges < plain.num_edges
        ei, sh = D.neighbor_list(p, r_max, cell, (True, True, True))
        ref = oracle({D.POSITIONS_KEY: p, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh})
        for k, rk in (("forces", "forces"), ("atomic_energy", "atomic_energy"), ("stress", "stress")):
            assert _rel(out[k], ref[rk]) < 1e-10, k
            assert _rel(out[k], out_plain[k]) < 1e-12, k
        p = p + 0.1 * torch.randn(p.shape, generator=g, dtype=p.dtype)
    assert calc.n_rebuilds == plain.n_rebuilds >= 1


def test_prune_edges_without_a_per_type_table_changes_nothing():
    from allegro_b200.calculator import AllegroCalculator
    from allegro_b200.model import AllegroModel

    rec = MODELS["c2_lmax2_L2"]
    model = AllegroModel(**rec["kwargs"])
    calc = AllegroCalculator(model, rec["kwargs"]["r_max"], skin=0.5, prune_edges=True)
    assert calc._cutoffs is None and calc.r_list == rec["kwargs"]["r_max"] + 0.5
