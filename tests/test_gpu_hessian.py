"""Forward-mode second derivatives on the GPU (nn._hessian, phonons.hessian_vector_product / analytic_force_constants):
the tangent kernels against tests/hvp_spec.py in fp64 and fp32 (ragged lists, isolated atoms, E = 0), analytic force
constants against the fp64 oracle's Hessian rows across the architecture grid and the cell kinds, the Hessian-vector
product against central differences of energy_and_forces, the properties of the blocks, determinism across chunkings and
atom subsets, every refusal, and the 10 976-atom c2 frame in several chunks."""
import pytest
import torch

import hvp_spec
import fc_spec
from fc_oracle import frame_list, hessian_rows, rel, synthetic_list
from test_gpu_force_constants import ARCH, SMALL, _cell_frame, _dev_csr, _full_fd
from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from allegro_b200.phonons import analytic_force_constants, force_constants, hessian_vector_product
from oracle.model_ref import AllegroOracle

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---- kernels against the restatement -----------------------------------------------------------------------------------
def _edges(seed, E, T=3, dtype=torch.float64, r_lo=0.6, r_hi=5.5):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(E, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True) * (r_lo + (r_hi - r_lo) * torch.rand(E, 1, generator=g, dtype=torch.float64))
    vdot = torch.randn(E, 3, generator=g, dtype=torch.float64)
    types = torch.randint(0, T, (E + 1,), generator=g, dtype=torch.int32)
    ctr = torch.randint(0, E + 1, (E,), generator=g, dtype=torch.int32)
    nbr = torch.randint(0, E + 1, (E,), generator=g, dtype=torch.int32)
    return d.to(dtype), vdot.to(dtype), types, ctr, nbr, g


def _close(got, want, dtype, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if want.numel() == 0:
        return
    tol = 1e-11 if dtype == torch.float64 else 2e-4
    err = rel(got, want)
    assert err <= tol, (what, err)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("E", [0, 1, 300])
def test_sh_and_act_kernels_match_the_spec(dtype, E):
    vec, vdot, _, _, _, g = _edges(1 + E, E, dtype=dtype)
    for lmax in range(5):
        D_ = (lmax + 1) ** 2
        gY = torch.randn(E, D_, generator=g, dtype=torch.float64).to(dtype)
        got = _lib.sh_jvp(vec.to(DEV), vdot.to(DEV), lmax).cpu()
        _close(got, hvp_spec.sh_jvp(vec.double(), vdot.double(), lmax), dtype, f"sh_jvp l={lmax}")
        base = torch.randn(E, 3, generator=g, dtype=torch.float64)
        out = base.to(dtype).to(DEV)
        _lib.sh_hvp(vec.to(DEV), vdot.to(DEV), gY.to(DEV), lmax, out)
        want = base.clone()
        hvp_spec.sh_hvp(vec.double(), vdot.double(), gY.double(), lmax, want)
        _close(out.cpu() - base.to(dtype), want - base, dtype, f"sh_hvp l={lmax}")
    n = 7 * E
    for code in (_lib.NL_SILU, _lib.NL_MISH, _lib.NL_GELU):
        ga, gad, pre, pd = [(4 * torch.randn(n, generator=g, dtype=torch.float64)).to(dtype) for _ in range(4)]
        for gd in (gad, None):
            got = _lib.act_bwd_jvp(None if gd is None else gd.to(DEV), ga.to(DEV), pre.to(DEV), pd.to(DEV), code).cpu()
            want = hvp_spec.act_bwd_jvp(None if gd is None else gd.double(), ga.double(), pre.double(), pd.double(), code)
            _close(got, want, dtype, f"act_bwd_jvp {code}")


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("E", [0, 1, 257])
def test_radial_and_zbl_kernels_match_the_spec(dtype, E):
    T = 3
    vec, vdot, types, ctr, nbr, g = _edges(11 + E, E, T=T, dtype=dtype)
    rmax = (4.0 + torch.rand(T, T, generator=g, dtype=torch.float64)).to(dtype)  # some edges lie beyond r_max
    if E > 1:  # one edge at r_max (alone it would be the scale of the comparison, and its terms vanish there)
        vec[0] = vec[0] / vec[0].norm() * rmax[types[ctr[0]], types[nbr[0]]]
    bw8 = (torch.arange(1, 9, dtype=torch.float64) + 0.1 * torch.randn(8, generator=g, dtype=torch.float64)).to(dtype)
    S = 40
    PQ = torch.randn(T * T, 8, S, generator=g, dtype=torch.float64).to(dtype)
    g_out, aux = [torch.randn(E, S, generator=g, dtype=torch.float64).to(dtype) for _ in range(2)]
    d = lambda t: t.to(DEV)  # noqa: E731
    args = (d(vec), d(vdot), d(ctr), d(nbr), d(types), d(rmax), d(bw8), d(PQ))
    got = _lib.radial_pq_jvp(dtype, S, 6.0, *args).cpu()
    _close(got, hvp_spec.radial_pq_jvp(torch.float64, S, 6.0, vec.double(), vdot.double(), ctr, nbr, types, rmax.double(), bw8.double(), PQ.double()),
           dtype, "radial_pq_jvp")
    for a, code in ((None, _lib.NL_SILU), (aux, _lib.NL_SILU), (aux, _lib.NL_MISH), (aux, _lib.NL_GELU)):
        out = torch.zeros(E, 3, dtype=dtype, device=DEV)
        _lib.radial_pq_hvp(dtype, S, 6.0, *args, d(g_out), None if a is None else d(a), out, code)
        want = torch.zeros(E, 3, dtype=torch.float64)
        hvp_spec.radial_pq_hvp(torch.float64, S, 6.0, vec.double(), vdot.double(), ctr, nbr, types, rmax.double(), bw8.double(), PQ.double(),
                               g_out.double(), None if a is None else a.double(), want, code)
        _close(out.cpu(), want, dtype, f"radial_pq_hvp {code}")
    # the generic route: 5 Bessel functions, S_rc = 12
    bw5 = bw8[:5].contiguous()
    Wb = torch.randn(5, 12, generator=g, dtype=torch.float64).to(dtype)
    cemb, nemb = [torch.randn(T, 6, generator=g, dtype=torch.float64).to(dtype) for _ in range(2)]
    ge0 = torch.randn(E, 12, generator=g, dtype=torch.float64).to(dtype)
    gargs = (d(vec), d(vdot), d(ctr), d(nbr), d(types), d(rmax), d(bw5), d(Wb), d(cemb), d(nemb))
    hargs = (vec.double(), vdot.double(), ctr, nbr, types, rmax.double(), bw5.double(), Wb.double(), cemb.double(), nemb.double())
    _close(_lib.radial_jvp(dtype, 12, 6.0, *gargs).cpu(), hvp_spec.radial_jvp(torch.float64, 12, 6.0, *hargs), dtype, "radial_jvp")
    out = torch.zeros(E, 3, dtype=dtype, device=DEV)
    _lib.radial_hvp(dtype, 12, 6.0, *gargs, d(ge0), out)
    want = torch.zeros(E, 3, dtype=torch.float64)
    hvp_spec.radial_hvp(torch.float64, 12, 6.0, *hargs, ge0.double(), want)
    _close(out.cpu(), want, dtype, "radial_hvp")
    Z = torch.tensor([3.0, 15.0, 16.0], dtype=dtype)
    out = torch.zeros(E, 3, dtype=dtype, device=DEV)
    _lib.zbl_hvp(6.0, 7.2, d(vec), d(vdot), d(ctr), d(nbr), d(types), d(Z), d(rmax.reshape(-1)), out)
    want = torch.zeros(E, 3, dtype=torch.float64)
    hvp_spec.zbl_hvp(6.0, 7.2, vec.double(), vdot.double(), ctr, nbr, types, Z.double(), rmax.double(), want)
    _close(out.cpu(), want, dtype, "zbl_hvp")
    if E:  # beyond r_max every term is exactly zero
        r = vec.double().norm(dim=-1)
        far = r > rmax.double()[types[ctr].long(), types[nbr].long()] * (1 + 1e-9)
        assert far.any()
        out = torch.zeros(E, 3, dtype=dtype, device=DEV)
        _lib.radial_pq_hvp(dtype, S, 6.0, *args, d(g_out), None, out)
        _lib.zbl_hvp(6.0, 7.2, d(vec), d(vdot), d(ctr), d(nbr), d(types), d(Z), d(rmax.reshape(-1)), out)
        assert bool((out.cpu()[far] == 0).all())
        assert bool((_lib.radial_pq_jvp(dtype, S, 6.0, *args).cpu()[far] == 0).all())


@pytest.mark.parametrize("pdt,adt", [(torch.float64, torch.float64), (torch.float32, torch.float32), (torch.float64, torch.float32)])
@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (1, 2, 1), (2, 7, 2), (3, 40, 3), (5, 6, 5)])
def test_fc_tangent_mode_matches_the_spec(seed, n, isolated, pdt, adt):
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated, dtype=pdt)
    g = torch.Generator().manual_seed(seed + 7)
    atoms = torch.randperm(n, generator=g)
    csr = _dev_csr(row_ptr, ctr, nbr)
    cptr, cen, coff, ea = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    fptr, col = fc_spec.columns(cptr, cen, row_ptr, nbr, n)
    atoms_d = atoms.to(DEV)
    dc = _lib.fc_centres(atoms_d, csr, n)
    dfp, dcol = _lib.fc_columns(dc[0], dc[1], csr, n)
    Cp = _lib._prefix((dc[0][1:] - dc[0][:-1]).repeat_interleave(3))
    Ep = _lib._prefix(dc[3].repeat_interleave(3))
    Cp_h, Ep_h = Cp.cpu(), Ep.cpu()
    U = 3 * n
    blocks = torch.full((col.shape[0], 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    for u0, u1 in ((0, U), (0, 1), (1, U)) if U > 1 else ((0, U),):
        Cb, Eb = int(Cp_h[u1] - Cp_h[u0]), int(Ep_h[u1] - Ep_h[u0])
        ref = hvp_spec.fc_gather_tangent(pos, shift, adt, atoms, cptr, cen, coff, ea, row_ptr, nbr, u0, u1)
        gd = torch.randn(Eb, 3, generator=g, dtype=torch.float64).to(adt)
        if Eb:
            got = _lib.fc_gather_tangent(pos.to(DEV), shift.to(DEV), adt, atoms_d, *dc, csr, Cp, Ep, u0, u1, Cb, Eb)
            for a, b in zip(got[:4], ref[:4]):
                assert torch.equal(a.cpu().long(), b.long())
            assert torch.equal(got[4].cpu(), ref[4]) and torch.equal(got[5].cpu(), ref[5])
        _lib.fc_fold_tangent(gd.to(DEV), *dc, csr, n, dfp, dcol, Ep, u0, u1, blocks)
        want = hvp_spec.fc_fold_tangent(gd, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, u0, u1)
        bl = blocks.cpu()
        for (p, alpha), v in want.items():
            torch.testing.assert_close(bl[p, alpha], v, rtol=1e-12, atol=1e-12)


# ---- models against the oracle -----------------------------------------------------------------------------------------
GRID = dict(ARCH)
GRID.update({
    "lmax4": ("c2", dict(l_max=4, num_layers=2)),
    "one_layer": ("c2", dict(num_layers=1)),
    "bessel5": ("c2", dict(radial_chemical_embed={"_target_": "allegro.nn.TwoBodyBesselScalarEmbed", "num_bessels": 5,
                                                  "polynomial_cutoff_p": 6})),
})


def _oracle_model(arch, dtype):
    """(fp64 oracle, model on the device, kwargs); mish / gelu take tests/nonlin_oracle.py."""
    if arch == "spline":
        from golden_util import load_models

        kw = dict({r["name"]: r for r in load_models()}["spline_embed_per_edge_type_cutoff"]["kwargs"])
    elif arch == "c2_widths":
        kw = systems.model_kwargs("c2", 30.0, "float64")
    else:
        sysname, over = GRID[arch]
        kw = systems.model_kwargs(sysname, 30.0, "float64")
        kw.update(SMALL)
        kw.update(over)
    if arch in ("mish", "gelu"):
        import nonlin_oracle

        oracle = nonlin_oracle.oracle(**kw)
    else:
        oracle = AllegroOracle(**kw)
    m = AllegroModel(**dict(kw, model_dtype=dtype))
    m.load_state_dict(oracle.state_dict())
    return oracle, m.to(DEV), kw


def _oracle_rows(oracle, pos, cell, types, pbc, atoms, r_max):
    p = pos.double().cpu()
    c = None if cell is None else cell.double().cpu()
    _, ctr, nbr, sv = frame_list(p, c, (pbc,) * 3, r_max)
    return hessian_rows(oracle, p, types.cpu(), ctr, nbr, sv, torch.tensor(atoms))


@pytest.mark.parametrize("arch", list(GRID) + ["spline", "c2_widths"])
def test_analytic_force_constants_against_the_oracle_grid(arch):
    oracle, m64, kw = _oracle_model(arch, "float64")
    kind = "open" if arch == "spline" else "ortho"
    pos, cell, types, pbc = _cell_frame(kind, kw)
    if arch == "spline":
        pos, types = pos[:6] * 0.6, types[:6]
    atoms = [0, 3, pos.shape[0] - 1]
    H = _oracle_rows(oracle, pos, cell, types, pbc, atoms, kw["r_max"])
    e64 = rel(analytic_force_constants(m64, pos, cell, types, pbc=pbc, atoms=torch.tensor(atoms)).dense(), H)
    msg = f"{arch}: fp64 analytic vs oracle Hessian rel {e64:.2e}"
    if arch in ("c2_small", "c2_widths", "mish", "zbl", "lmax4", "spline"):
        _, m32, _ = _oracle_model(arch, "float32")
        p32, c32 = pos.float(), None if cell is None else cell.float()
        e32 = rel(analytic_force_constants(m32, p32, c32, types, pbc=pbc, atoms=torch.tensor(atoms)).dense(), H)
        efd = rel(force_constants(m32, p32, c32, types, pbc=pbc, atoms=torch.tensor(atoms), displacement=1e-2).dense(), H)
        msg += f"; fp32 analytic {e32:.2e}, fp32 finite difference (h = 1e-2) {efd:.2e}"
        assert e32 <= 1e-3 and e32 < efd, (e32, efd)
    print(msg)
    assert e64 <= 1e-10, e64


@pytest.mark.parametrize("kind", ["ortho", "hcp", "short", "open"])
def test_analytic_force_constants_across_cells(kind):
    oracle, m64, kw = _oracle_model("c2_small", "float64")
    pos, cell, types, pbc = _cell_frame(kind, kw)
    atoms = list(range(pos.shape[0])) if pos.shape[0] <= 8 else [0, 1, 5, pos.shape[0] - 1]
    H = _oracle_rows(oracle, pos, cell, types, pbc, atoms, kw["r_max"])
    fc = analytic_force_constants(m64, pos, cell, types, pbc=pbc, atoms=torch.tensor(atoms))
    err = rel(fc.dense(), H)
    print(f"{kind}: fp64 analytic vs oracle Hessian rel {err:.2e}")
    assert err <= 1e-10, err
    if kind == "open":  # the isolated atom: one zero diagonal block
        a = atoms.index(pos.shape[0] - 1)
        r = slice(int(fc.row_ptr[a]), int(fc.row_ptr[a + 1]))
        assert fc.col[r].tolist() == [pos.shape[0] - 1] and bool((fc.blocks[r] == 0).all())


# ---- the Hessian-vector product ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["ortho", "short", "open"])
@pytest.mark.parametrize("arch", ["c2_small", "zbl", "spline"])
def test_hessian_vector_product_fp64(arch, kind):
    if arch == "spline" and kind != "open":
        pytest.skip("the spline model's species fit the open cluster")
    _, model, kw = _oracle_model(arch, "float64")
    pos, cell, types, pbc = _cell_frame(kind, kw)
    if arch == "spline":
        pos, types = pos[:6] * 0.6, types[:6]
    n = pos.shape[0]
    g = torch.Generator().manual_seed(3)
    v, w = [torch.randn(n, 3, generator=g, dtype=torch.float64).to(DEV) for _ in range(2)]
    Hv = hessian_vector_product(model, pos, cell, types, v, pbc=pbc)
    Hw = hessian_vector_product(model, pos, cell, types, w, pbc=pbc)
    # central differences of energy_and_forces along v on a fixed list
    eps = 1e-4
    from allegro_b200.calculator import prune_table

    cut = prune_table(model, 2 * eps)
    prune = {} if cut is None else dict(types=types.to(torch.int32), cutoffs=cut)
    csr, sv = D.neighbor_csr(pos, kw["r_max"] + 2 * eps, cell, (pbc,) * 3, **prune)
    fs = []
    for s in (1.0, -1.0):
        d = {D.POSITIONS_KEY: pos + s * eps * v, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
        if cell is not None:
            d[D.CELL_KEY] = cell
        fs.append(model.model.energy_and_forces(d)[D.FORCE_KEY].double())
    fd = -(fs[0] - fs[1]) / (2 * eps)
    e_fd = rel(Hv, fd)
    sym = abs(float((v * Hw).sum() - (w * Hv).sum())) / max(float((v * Hw).sum().abs()), 1e-300)
    fc = analytic_force_constants(model, pos, cell, types, pbc=pbc).dense()
    j, alpha = n // 2, 1
    e = torch.zeros(n, 3, dtype=torch.float64, device=DEV)
    e[j, alpha] = 1.0
    e_fc = rel(hessian_vector_product(model, pos, cell, types, e, pbc=pbc), fc[j, :, alpha])
    print(f"{arch}/{kind}: HVP vs central differences {e_fd:.2e}, v'Hw - w'Hv {sym:.2e}, vs analytic fc row {e_fc:.2e}")
    assert e_fd <= 1e-6 and sym <= 1e-11 and e_fc <= 1e-12, (e_fd, sym, e_fc)


# ---- properties, determinism, refusals -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_properties_and_determinism(dtype):
    _, model, kw = _oracle_model("c2_small", dtype)
    pdt = torch.float64 if dtype == "float64" else torch.float32
    pos, cell, types, pbc = _cell_frame("hcp", kw, pdt)
    n = pos.shape[0]
    full = analytic_force_constants(model, pos, cell, types)
    Dn = full.dense()
    scale = float(full.blocks.abs().max())
    asr = float(Dn.sum(1).abs().max()) / scale
    sym = float((Dn - Dn.permute(1, 0, 3, 2)).abs().max()) / scale
    print(f"{dtype}: acoustic sum rule {asr:.2e}, asymmetry {sym:.2e}")
    assert asr < (1e-12 if dtype == "float64" else 1e-4)
    assert sym < (1e-12 if dtype == "float64" else 1e-4)
    tol = 0.0 if dtype == "float32" else 1e-10

    def same(fc, rows):
        for b, a in enumerate(rows):
            ra = slice(int(full.row_ptr[a]), int(full.row_ptr[a + 1]))
            rb = slice(int(fc.row_ptr[b]), int(fc.row_ptr[b + 1]))
            assert torch.equal(fc.col[rb], full.col[ra])
            d = float((fc.blocks[rb] - full.blocks[ra]).abs().max()) / scale
            assert d <= tol, (a, d)

    sub = torch.tensor([n - 1, 3, 0])
    same(analytic_force_constants(model, pos, cell, types, atoms=sub), sub.tolist())
    one = int(_lib.fc_centres(torch.arange(n, device=DEV), D.neighbor_csr(pos, kw["r_max"], cell)[0], n)[3].max())
    for cap in (one, 3 * one + 1, 50 * one):
        same(analytic_force_constants(model, pos, cell, types, max_edges=cap), list(range(n)))


def test_refusals():
    _, model, kw = _oracle_model("c2_small", "float64")
    pos, cell, types, pbc = _cell_frame("ortho", kw)
    n = pos.shape[0]
    v = torch.ones(n, 3, dtype=torch.float64, device=DEV)
    from allegro_b200.committee import Committee

    for fn, extra in ((analytic_force_constants, ()), (hessian_vector_product, (v,))):
        with pytest.raises(TypeError):
            fn(Committee([model.model]), pos, cell, types, *extra)
        with pytest.raises(TypeError):
            fn(object(), pos, cell, types, *extra)
        with pytest.raises(RuntimeError):
            fn(model, pos.cpu(), cell, types, *extra)
        with pytest.raises(RuntimeError):
            fn(model, pos, cell, types.cpu(), *extra)
        for bad in (types[:-1], types.unsqueeze(-1), types.double()):
            with pytest.raises(ValueError):
                fn(model, pos, cell, bad, *extra)
        flat = cell.clone()
        flat[2] = flat[0] + flat[1]
        for c in (None, flat):
            with pytest.raises(ValueError):
                fn(model, pos, c, types, *extra)
    for bad in (pos[:, :2].contiguous(), pos.to(torch.float16), pos.unsqueeze(0)):
        with pytest.raises(ValueError):
            analytic_force_constants(model, bad, cell, types)
        with pytest.raises(ValueError):
            hessian_vector_product(model, bad, cell, types, v)
    for atoms in (torch.tensor([[0, 1]]), torch.tensor([0.0, 1.0]), torch.tensor([-1]), torch.tensor([n]), torch.tensor([2, 2])):
        with pytest.raises(ValueError):
            analytic_force_constants(model, pos, cell, types, atoms=atoms)
    with pytest.raises(ValueError):
        analytic_force_constants(model, pos, cell, types, max_edges=0)
    with pytest.raises(ValueError):
        analytic_force_constants(model, pos, cell, types, max_edges=1)
    for bad in (v.cpu(), v[:-1], v.long(), v.reshape(-1), v[:, :2], "v"):
        with pytest.raises(ValueError):
            hessian_vector_product(model, pos, cell, types, bad)
    # a frame without edges: zeros
    far = torch.tensor([[0.0, 0.0, 0.0], [20.0, 0.0, 0.0]], dtype=torch.float64, device=DEV)
    hv = hessian_vector_product(model, far, None, types[:2], torch.ones(2, 3, dtype=torch.float64, device=DEV), pbc=False)
    assert hv.shape == (2, 3) and bool((hv == 0).all())


def test_c2_frame_in_several_chunks():
    """The 10 976-atom c2 frame, fp32 model: 8 random displaced atoms in small chunks against full-frame differences,
    and the full-frame Hessian-vector product against the analytic rows."""
    pos, cell, types = systems.make_positions("c2")
    kw = systems.model_kwargs("c2", 42.0, "float32")
    m = AllegroModel(**kw).to(DEV)
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    g = torch.Generator().manual_seed(5)
    atoms = torch.randperm(pos.shape[0], generator=g)[:8]
    fc = analytic_force_constants(m, pos, cell, types, atoms=atoms, max_edges=5_000)
    ref = _full_fd(m, pos, cell, types, True, atoms.tolist(), 0.01, kw["r_max"] + 0.01)
    err = rel(fc.dense(), ref)
    one = analytic_force_constants(m, pos, cell, types, atoms=atoms[:2])
    d = float((one.dense() - fc.dense()[:2]).abs().max())
    e = torch.zeros(pos.shape[0], 3, dtype=torch.float32, device=DEV)
    e[int(atoms[0]), 2] = 1.0
    e_hv = rel(hessian_vector_product(m, pos, cell, types, e), fc.dense()[0, :, 2])
    print(f"c2 fp32, 8 atoms in chunks of <= 5k edges: vs full-frame differences rel {err:.2e}, vs one chunk {d:.1e}, "
          f"HVP vs the rows {e_hv:.2e}")
    assert err < 1e-3 and d == 0.0 and e_hv < 1e-4, (err, d, e_hv)
