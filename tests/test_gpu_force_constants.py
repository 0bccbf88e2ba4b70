"""phonons.force_constants on the GPU: the ab2_fc_* kernels against tests/fc_spec.py, the locality argument on the device
(fp64 models equal full-frame central differences of energy_and_forces across the architecture grid and the cell kinds),
the fp64 oracle's Hessian, the properties of a force-constant matrix, determinism across chunkings and atom subsets,
every refusal, and a 10 976-atom frame in many chunks."""
import math

import pytest
import torch

import fc_spec
from fc_oracle import hessian_rows, rel, synthetic_list
from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from allegro_b200.phonons import force_constants
from oracle.model_ref import AllegroOracle

pytestmark = pytest.mark.gpu
DEV = "cuda"

SMALL = dict(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16,
             scalar_embed_mlp_hidden_layers_width=16, allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=8)
CUTOFFS = {"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}
ZBL = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]}


# ---- kernels against the restatement -----------------------------------------------------------------------------------
def _dev_csr(row_ptr, ctr, nbr):
    n = row_ptr.shape[0] - 1
    return D.EdgeCSR(n, ctr.to(DEV, torch.int32).contiguous(), nbr.to(DEV, torch.int32).contiguous(), row_ptr.to(DEV, torch.int32).contiguous(),
                     None, int((row_ptr[1:] - row_ptr[:-1]).max()) if n else 0)


@pytest.mark.parametrize("pdt,adt", [(torch.float64, torch.float64), (torch.float32, torch.float32), (torch.float64, torch.float32)])
@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (1, 2, 1), (2, 7, 2), (3, 40, 3), (5, 6, 5)])
def test_kernels_match_the_spec(seed, n, isolated, pdt, adt):
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated, dtype=pdt)
    g = torch.Generator().manual_seed(seed + 7)
    atoms = torch.randperm(n, generator=g)
    csr = _dev_csr(row_ptr, ctr, nbr)
    h = float(torch.tensor(0.0625, dtype=pdt))
    cptr, cen, coff, ea = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    fptr, col = fc_spec.columns(cptr, cen, row_ptr, nbr, n)
    atoms_d = atoms.to(DEV)
    dc = _lib.fc_centres(atoms_d, csr, n)
    for got, ref in zip(dc, (cptr, cen, coff, ea)):
        assert torch.equal(got.cpu().long(), ref.long())
    dfp, dcol = _lib.fc_columns(dc[0], dc[1], csr, n)
    assert torch.equal(dfp.cpu(), fptr) and torch.equal(dcol.cpu().long(), col)
    Cp, Ep = fc_spec.unit_prefix(cptr, ea)
    U = 3 * n
    blocks = torch.full((col.shape[0], 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    gref = torch.Generator().manual_seed(seed + 11)
    for u0, u1 in ((0, U), (0, 1), (1, U)) if U > 1 else ((0, U),):
        Cb, Eb = int(2 * (Cp[u1] - Cp[u0])), int(2 * (Ep[u1] - Ep[u0]))
        ref = fc_spec.gather(pos, shift, h, adt, atoms, cptr, cen, coff, ea, row_ptr, nbr, u0, u1)
        gvec = torch.randn(Eb, 3, generator=gref, dtype=torch.float64).to(adt)
        if Eb:
            got = _lib.fc_gather(pos.to(DEV), shift.to(DEV), h, adt, atoms_d, *dc, csr, Cp.to(DEV), Ep.to(DEV), u0, u1, Cb, Eb)
            for a, b in zip(got[:4], ref[:4]):
                assert torch.equal(a.cpu().long(), b.long())
            assert torch.equal(got[4].cpu(), ref[4])  # the same operations in the positions' dtype, one rounding
        _lib.fc_fold(gvec.to(DEV), h, *dc, csr, n, dfp, dcol, Ep.to(DEV), u0, u1, blocks)
        want = fc_spec.fold(gvec, h, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, u0, u1)
        bl = blocks.cpu()
        for (p, alpha), v in want.items():
            torch.testing.assert_close(bl[p, alpha], v, rtol=1e-12, atol=1e-12)


# ---- models and frames ---------------------------------------------------------------------------------------------------
ARCH = {
    "c2_small": ("c2", {}),
    "lmax0": ("c2", dict(l_max=0, num_layers=2)),
    "lmax1_L3": ("c2", dict(l_max=1, num_layers=3)),
    "lmax3": ("c2", dict(l_max=3, num_layers=2)),
    "no_coupling": ("c2", dict(tp_path_channel_coupling=False)),
    "mish": ("c2", dict(allegro_mlp_nonlinearity="mish", readout_mlp_nonlinearity="mish", scalar_embed_mlp_nonlinearity="mish")),
    "gelu": ("c2", dict(allegro_mlp_nonlinearity="gelu", readout_mlp_nonlinearity="gelu", scalar_embed_mlp_nonlinearity="gelu")),
    "scales": ("c2", dict(per_type_energy_scales=[2.5], per_type_energy_shifts=[-1.25])),
    "per_edge_cutoff": ("c3", dict(per_edge_type_cutoff=CUTOFFS, per_type_energy_shifts=[0.5, -1.0, 0.25])),
    "zbl": ("c3", dict(per_edge_type_cutoff=CUTOFFS, pair_potential=ZBL)),
}


def _model(name, dtype, arch=None):
    if arch == "spline":
        from golden_util import load_models

        kw = dict({r["name"]: r for r in load_models()}["spline_embed_per_edge_type_cutoff"]["kwargs"])
    else:
        sysname, over = ARCH[arch or "c2_small"]
        kw = systems.model_kwargs(sysname, 30.0, "float64")
        kw.update(SMALL)
        kw.update(over)
    if arch in ("mish", "gelu"):  # the oracle takes silu MLPs only; these compare against the model's own full frames
        return None, AllegroModel(**dict(kw, model_dtype=dtype)).to(DEV), kw
    oracle = AllegroOracle(**kw)
    m = AllegroModel(**dict(kw, model_dtype=dtype))
    m.load_state_dict(oracle.state_dict())
    return oracle, m.to(DEV), kw


def _cell_frame(kind, kw, dtype=torch.float64, seed=0):
    """(pos, cell, types, pbc) of a small frame of the model's species."""
    g = torch.Generator().manual_seed(seed)
    T = len(kw["type_names"])
    if kind == "ortho":
        pos, cell = systems._lattice(systems._FCC, 3.6, (2, 2, 3), 0.08, g)
    elif kind == "hcp":
        a, c = 2.9, 4.7
        cell = torch.tensor([[a, 0.0, 0.0], [-a / 2, a * math.sqrt(3) / 2, 0.0], [0.0, 0.0, c]], dtype=torch.float64) * torch.tensor([[2.0], [2.0], [2.0]], dtype=torch.float64)
        frac = torch.tensor([[0.0, 0.0, 0.0], [1 / 3, 2 / 3, 0.5]], dtype=torch.float64)
        reps = torch.stack(torch.meshgrid(*[torch.arange(2.0, dtype=torch.float64)] * 3, indexing="ij"), -1).reshape(-1, 3)
        f = ((frac.unsqueeze(0) + reps.unsqueeze(1)) / 2).reshape(-1, 3)
        pos = f @ cell + 0.05 * torch.randn(f.shape[0], 3, generator=g, dtype=torch.float64)
    elif kind == "short":
        # a 2-atom cell shorter than r_max: every atom sees its own images
        a = 3.7
        cell = torch.tensor([[0.0, a / 2, a / 2], [a / 2, 0.0, a / 2], [a, a, 0.0]], dtype=torch.float64)
        pos = torch.tensor([[0.03, -0.02, 0.01], [0.9, 0.95, 0.02]], dtype=torch.float64)
    elif kind == "open":
        # no cell: a small cluster and one isolated atom far away
        pos = 2.4 * torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0.2], [0.6, 0.4, 1.1], [9, 9, 9]], dtype=torch.float64)
        pos = pos + 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
        cell = None
    else:
        raise KeyError(kind)
    types = torch.randint(0, T, (pos.shape[0],), generator=g)
    return pos.to(DEV, dtype), (None if cell is None else cell.to(DEV, dtype)), types.to(DEV), kind != "open"


def _full_fd(model, pos, cell, types, pbc, atoms, h, r_list, cutoffs=None):
    """-(F(r + h e) - F(r - h e)) / (2h) of whole displaced frames from energy_and_forces, on a fixed list at r_list."""
    inner = model.model
    prune = {} if cutoffs is None else dict(types=types.to(torch.int32), cutoffs=cutoffs)
    csr, sv = D.neighbor_csr(pos, r_list, cell, (pbc,) * 3, **prune)
    n = pos.shape[0]
    out = torch.zeros(len(atoms), n, 3, 3, dtype=torch.float64)
    for a, j in enumerate(atoms):
        for alpha in range(3):
            fs = []
            for s in (1.0, -1.0):
                q = pos.clone()
                q[j, alpha] += s * h
                d = {D.POSITIONS_KEY: q, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
                if cell is not None:
                    d[D.CELL_KEY] = cell
                fs.append(inner.energy_and_forces(d)[D.FORCE_KEY].double().cpu())
            out[a, :, alpha] = -(fs[0] - fs[1]) / (2 * h)
    return out


def _dense_rows(fc):
    return fc.dense().cpu()


@pytest.mark.parametrize("arch", list(ARCH) + ["spline"])
def test_fp64_equals_full_frame_differences_across_the_grid(arch):
    oracle, model, kw = _model(None, "float64", arch)
    kind = "ortho" if arch != "spline" else "open"
    pos, cell, types, pbc = _cell_frame(kind, kw)
    if arch == "spline":
        pos = pos[:6] * 0.6
        types = types[:6]
    h = 0.01
    atoms = [0, 3, pos.shape[0] - 1]
    fc = force_constants(model, pos, cell, types, pbc=pbc, atoms=torch.tensor(atoms), displacement=h)
    from allegro_b200.calculator import prune_table

    ref = _full_fd(model, pos, cell, types, pbc, atoms, h, kw["r_max"] + h, prune_table(model, h))
    err = rel(_dense_rows(fc), ref)
    print(f"{arch}: force_constants vs full-frame differences rel {err:.2e}")
    assert err <= 1e-9, err


@pytest.mark.parametrize("kind", ["ortho", "hcp", "short", "open"])
def test_fp64_equals_full_frame_differences_across_cells(kind):
    oracle, model, kw = _model(None, "float64")
    pos, cell, types, pbc = _cell_frame(kind, kw)
    h = 0.01
    atoms = list(range(pos.shape[0])) if pos.shape[0] <= 8 else [0, 1, 5, pos.shape[0] - 1]
    fc = force_constants(model, pos, cell, types, pbc=pbc, atoms=torch.tensor(atoms), displacement=h)
    ref = _full_fd(model, pos, cell, types, pbc, atoms, h, kw["r_max"] + h)
    err = rel(_dense_rows(fc), ref)
    print(f"{kind}: force_constants vs full-frame differences rel {err:.2e}")
    assert err <= 1e-9, err
    if kind == "open":  # the isolated atom: one zero diagonal block
        a = atoms.index(pos.shape[0] - 1)
        r = slice(int(fc.row_ptr[a]), int(fc.row_ptr[a + 1]))
        assert fc.col[r].tolist() == [pos.shape[0] - 1] and bool((fc.blocks[r] == 0).all())


def _oracle_hessian(oracle, pos, cell, types, atoms, r_max):
    p, c = pos.double().cpu(), cell.double().cpu()
    ei, sh = D.neighbor_list(p, r_max, c, (True, True, True))
    return hessian_rows(oracle, p, types.cpu(), ei[0], ei[1], sh.double() @ c, torch.tensor(atoms))


def test_against_the_oracle_hessian():
    oracle, m64, kw = _model(None, "float64")
    _, m32, _ = _model(None, "float32")
    pos, cell, types, pbc = _cell_frame("ortho", kw)
    pos, types = pos[:32].contiguous(), types[:32].contiguous()
    cell = cell.clone()
    atoms = [0, 7, 19]
    H = _oracle_hessian(oracle, pos, cell, types, atoms, kw["r_max"])
    e64 = rel(_dense_rows(force_constants(m64, pos, cell, types, atoms=torch.tensor(atoms), displacement=1e-4)), H)
    e32 = rel(_dense_rows(force_constants(m32, pos.float(), cell.float(), types, atoms=torch.tensor(atoms), displacement=0.01)), H)
    print(f"vs oracle Hessian: fp64 model h=1e-4 rel {e64:.2e}; fp32 model h=1e-2 rel {e32:.2e} (tolerance 2e-3, measured 5.3e-4)")
    assert e64 < 1e-5, e64
    assert e32 < 2e-3, e32


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_properties_and_determinism(dtype):
    _, model, kw = _model(None, dtype)
    pdt = torch.float64 if dtype == "float64" else torch.float32
    pos, cell, types, pbc = _cell_frame("hcp", kw, pdt)
    n = pos.shape[0]
    h = 0.01 if dtype == "float32" else 1e-4
    full = force_constants(model, pos, cell, types, displacement=h)
    assert torch.equal(full.atoms.cpu(), torch.arange(n))
    Dn = full.dense()
    scale = float(full.blocks.abs().max())
    # acoustic sum rule (translation invariance of the energy) and symmetry to O(h^2)
    asr = float(Dn.sum(1).abs().max()) / scale
    sym = float((Dn - Dn.permute(1, 0, 3, 2)).abs().max()) / scale
    print(f"{dtype}: acoustic sum rule {asr:.2e}, asymmetry {sym:.2e}")
    assert asr < (1e-12 if dtype == "float64" else 1e-4)
    assert sym < (1e-6 if dtype == "float64" else 5e-3)
    for a in range(n):
        r = slice(int(full.row_ptr[a]), int(full.row_ptr[a + 1]))
        assert torch.equal(Dn[a, full.col[r]], full.blocks[r])
    # a subset, and other chunkings, give the same rows (fp64 at h = 0.01: the atomics' rounding is divided by 2h)
    if dtype == "float64":
        h = 0.01
        full = force_constants(model, pos, cell, types, displacement=h)
        scale = float(full.blocks.abs().max())
    sub = torch.tensor([n - 1, 3, 0])
    tol = 0.0 if dtype == "float32" else 1e-13

    def same(fc, rows):
        for b, a in enumerate(rows):
            ra = slice(int(full.row_ptr[a]), int(full.row_ptr[a + 1]))
            rb = slice(int(fc.row_ptr[b]), int(fc.row_ptr[b + 1]))
            assert torch.equal(fc.col[rb], full.col[ra])
            d = float((fc.blocks[rb] - full.blocks[ra]).abs().max()) / scale
            assert d <= tol, (a, d)

    same(force_constants(model, pos, cell, types, atoms=sub, displacement=h), sub.tolist())
    one = int(2 * (_lib.fc_centres(torch.arange(n, device=DEV), D.neighbor_csr(pos, kw["r_max"] + h, cell)[0], n)[3].max()))
    for cap in (one, 3 * one + 1, 50 * one):
        same(force_constants(model, pos, cell, types, displacement=h, max_edges=cap), list(range(n)))


def test_refusals():
    _, model, kw = _model(None, "float64")
    pos, cell, types, pbc = _cell_frame("ortho", kw)
    n = pos.shape[0]
    from allegro_b200.committee import Committee

    with pytest.raises(TypeError):
        force_constants(Committee([model.model]), pos, cell, types)
    with pytest.raises(TypeError):
        force_constants(object(), pos, cell, types)
    with pytest.raises(RuntimeError):
        force_constants(model, pos.cpu(), cell, types)
    with pytest.raises(RuntimeError):
        force_constants(model, pos, cell, types.cpu())
    for h in (0.0, -0.01, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            force_constants(model, pos, cell, types, displacement=h)
    for atoms in (torch.tensor([[0, 1]]), torch.tensor([0.0, 1.0]), torch.tensor([-1]), torch.tensor([n]), torch.tensor([2, 2])):
        with pytest.raises(ValueError):
            force_constants(model, pos, cell, types, atoms=atoms)
    for bad in (pos[:, :2].contiguous(), pos.to(torch.float16), pos.unsqueeze(0)):
        with pytest.raises(ValueError):
            force_constants(model, bad, cell, types)
    for bad in (types[:-1], types.unsqueeze(-1), types.double()):
        with pytest.raises(ValueError):
            force_constants(model, pos, cell, bad)
    flat = cell.clone()
    flat[2] = flat[0] + flat[1]
    for c in (None, flat):
        with pytest.raises(ValueError):
            force_constants(model, pos, c, types)
    with pytest.raises(ValueError):
        force_constants(model, pos, cell, types, max_edges=0)


def test_c2_frame_in_many_chunks():
    """The 10 976-atom c2 frame, fp32 model: 16 random displaced atoms in small chunks against full-frame differences."""
    pos, cell, types = systems.make_positions("c2")
    kw = systems.model_kwargs("c2", 42.0, "float32")
    m = AllegroModel(**kw).to(DEV)
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    g = torch.Generator().manual_seed(5)
    atoms = torch.randperm(pos.shape[0], generator=g)[:16]
    h = 0.01
    fc = force_constants(m, pos, cell, types, atoms=atoms, displacement=h, max_edges=20_000)
    ref = _full_fd(m, pos, cell, types, True, atoms.tolist(), h, kw["r_max"] + h)
    err = rel(_dense_rows(fc), ref)
    print(f"c2 fp32, 16 atoms in chunks of <= 20k edges: rel {err:.2e}")
    assert err < 1e-3, err
