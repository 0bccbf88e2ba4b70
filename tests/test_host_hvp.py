"""The tangent kernels' restatements (tests/hvp_spec.py) against forward-mode / double autograd of the fp64 oracle's
functions, and the whole tangent sequencing (nn._hessian) run on the restatements against the oracle's Hessian rows, on
the CPU.  The kernels themselves are checked against these restatements on the GPU (tests/test_gpu_hessian.py)."""
import os

import pytest
import torch

import fc_spec
import hvp_spec
import kernel_spec
from fc_oracle import frame_list, hessian_rows, rel, synthetic_list
from allegro_b200 import _lib
from oracle import o3_ref

BAR = 1e-12
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _edges(seed, E, T=3, r_lo=0.5, r_hi=5.5):
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(E, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True) * (r_lo + (r_hi - r_lo) * torch.rand(E, 1, generator=g, dtype=torch.float64))
    vdot = torch.randn(E, 3, generator=g, dtype=torch.float64)
    types = torch.randint(0, T, (E + 1,), generator=g, dtype=torch.int32)
    ctr = torch.randint(0, E + 1, (E,), generator=g, dtype=torch.int32)
    nbr = torch.randint(0, E + 1, (E,), generator=g, dtype=torch.int32)
    return d, vdot, types, ctr, nbr, g


def _vjp_jvp(f, vec, vdot, gout):
    """d/de [J_f(vec + e vdot)^T gout] by forward over reverse autograd."""
    return torch.func.jvp(lambda v: torch.func.vjp(f, v)[1](gout)[0], (vec,), (vdot,))[1]


@pytest.mark.parametrize("lmax", [0, 1, 2, 3, 4])
def test_sh_tangents(lmax):
    vec, vdot, _, _, _, g = _edges(lmax, 200)
    sh = lambda v: o3_ref.spherical_harmonics(lmax, v, method="explicit" if lmax <= 3 else "recursive")  # noqa: E731
    want = torch.func.jvp(sh, (vec,), (vdot,))[1]
    assert rel(hvp_spec.sh_jvp(vec, vdot, lmax), want) <= BAR
    gY = torch.randn(200, (lmax + 1) ** 2, generator=g, dtype=torch.float64)
    got = torch.zeros(200, 3, dtype=torch.float64)
    hvp_spec.sh_hvp(vec, vdot, gY, lmax, got)
    want = _vjp_jvp(sh, vec, vdot, gY)
    assert float((got - want).abs().max()) <= BAR * max(float(want.abs().max()), 1.0)


@pytest.mark.parametrize("code", [_lib.NL_SILU, _lib.NL_MISH, _lib.NL_GELU])
def test_nonlinearity_second_derivatives(code):
    phi = {_lib.NL_SILU: torch.nn.functional.silu, _lib.NL_MISH: torch.nn.functional.mish, _lib.NL_GELU: torch.nn.functional.gelu}[code]
    x = torch.linspace(-15.0, 19.0, 3001, dtype=torch.float64).requires_grad_(True)
    (d1,) = torch.autograd.grad(phi(x).sum(), x, create_graph=True)
    (d2,) = torch.autograd.grad(d1.sum(), x)
    assert float((hvp_spec.d2phi(code, x.detach()) - d2).abs().max()) <= BAR
    g = torch.Generator().manual_seed(code)
    ga, gad, pd = [torch.randn(3001, generator=g, dtype=torch.float64) for _ in range(3)]
    want = ga * d2 * pd + gad * d1.detach()
    assert float((hvp_spec.act_bwd_jvp(gad, ga, x.detach(), pd, code) - want).abs().max()) <= 10 * BAR


def _radial_case(seed, E, nb):
    T = 3
    vec, vdot, types, ctr, nbr, g = _edges(seed, E, T=T)
    rmax = 4.0 + torch.rand(T, T, generator=g, dtype=torch.float64)
    vec[0] = vec[0] / vec[0].norm() * rmax[types[ctr[0]].long(), types[nbr[0]].long()]  # exactly at r_max
    bw = torch.arange(1, nb + 1, dtype=torch.float64) + 0.1 * torch.randn(nb, generator=g, dtype=torch.float64)
    return vec, vdot, types, ctr, nbr, rmax, bw, g


def test_bessel_and_cutoff_tangents_pq_route():
    vec, vdot, types, ctr, nbr, rmax, bw, g = _radial_case(3, 300, 8)
    S = 24
    PQ = torch.randn(9, 8, S, generator=g, dtype=torch.float64)
    f = lambda v: kernel_spec._radial_pq(6.0, v, ctr, nbr, types, rmax, bw, PQ)  # noqa: E731
    want = torch.func.jvp(f, (vec,), (vdot,))[1]
    got = hvp_spec.radial_pq_jvp(torch.float64, S, 6.0, vec, vdot, ctr, nbr, types, rmax, bw, PQ)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())
    gout, aux = [torch.randn(300, S, generator=g, dtype=torch.float64) for _ in range(2)]
    for a in (None, aux):
        gg = gout if a is None else gout * kernel_spec._dsilu(a)
        want = _vjp_jvp(f, vec, vdot, gg)
        got = torch.zeros(300, 3, dtype=torch.float64)
        hvp_spec.radial_pq_hvp(torch.float64, S, 6.0, vec, vdot, ctr, nbr, types, rmax, bw, PQ, gout, a, got)
        assert float((got - want).abs().max()) <= BAR * float(want.abs().max())
    far = vec.norm(dim=-1) >= rmax[types[ctr].long(), types[nbr].long()]
    assert far.sum() > 1 and bool((got[far] == 0).all())


def test_bessel_and_cutoff_tangents_generic_route():
    vec, vdot, types, ctr, nbr, rmax, bw, g = _radial_case(4, 300, 5)
    Wb = torch.randn(5, 12, generator=g, dtype=torch.float64)
    cemb, nemb = [torch.randn(3, 6, generator=g, dtype=torch.float64) for _ in range(2)]
    f = lambda v: kernel_spec._radial(torch.float64, 12, 6.0, v, ctr, nbr, types, rmax, bw, Wb, cemb, nemb)  # noqa: E731
    want = torch.func.jvp(f, (vec,), (vdot,))[1]
    got = hvp_spec.radial_jvp(torch.float64, 12, 6.0, vec, vdot, ctr, nbr, types, rmax, bw, Wb, cemb, nemb)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())
    ge0 = torch.randn(300, 12, generator=g, dtype=torch.float64)
    want = _vjp_jvp(f, vec, vdot, ge0)
    got = torch.zeros(300, 3, dtype=torch.float64)
    hvp_spec.radial_hvp(torch.float64, 12, 6.0, vec, vdot, ctr, nbr, types, rmax, bw, Wb, cemb, nemb, ge0, got)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())


def test_zbl_hessian():
    vec, vdot, types, ctr, nbr, g = _edges(5, 300, r_lo=0.3)
    rmax = 4.0 + torch.rand(3, 3, generator=g, dtype=torch.float64)
    Z = torch.tensor([3.0, 15.0, 16.0], dtype=torch.float64)
    f = lambda v: kernel_spec._zbl(6.0, 7.2, v, ctr, nbr, types, Z, rmax)  # noqa: E731
    want = _vjp_jvp(f, vec, vdot, torch.ones(300, dtype=torch.float64))
    got = torch.zeros(300, 3, dtype=torch.float64)
    hvp_spec.zbl_hvp(6.0, 7.2, vec, vdot, ctr, nbr, types, Z, rmax, got)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())


def test_spline_tangents():
    from allegro_b200.nn._spline import spline_backward, spline_forward, spline_hvp, spline_jvp

    vec, vdot, types, ctr, nbr, g = _edges(6, 200, T=2, r_lo=0.2, r_hi=4.5)
    K, C = 6, 10
    lower = torch.linspace(0.0, 0.8, K, dtype=torch.float64)
    upper = lower + 0.35
    w = torch.randn(4 * K, C, generator=g, dtype=torch.float64)
    rmax = torch.tensor([[4.0, 3.5], [3.5, 4.2]], dtype=torch.float64)
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    f = lambda v: spline_forward(v, tc, tn, rmax, lower, upper, 2 * torch.pi / 0.35, w, 2, torch.float64)[0]  # noqa: E731
    want = torch.func.jvp(f, (vec,), (vdot,))[1]
    got = spline_jvp(vec, vdot, tc, tn, rmax, lower, upper, 2 * torch.pi / 0.35, w, 2, torch.float64)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())
    ge0 = torch.randn(200, C, generator=g, dtype=torch.float64)
    want = _vjp_jvp(f, vec, vdot, ge0)
    got = spline_hvp(vec, vdot, tc, tn, rmax, lower, upper, 2 * torch.pi / 0.35, w, 2, ge0)
    assert float((got - want).abs().max()) <= BAR * float(want.abs().max())
    # the hand-written adjoint the tangent shares
    _, saved = spline_forward(vec, tc, tn, rmax, lower, upper, 2 * torch.pi / 0.35, w, 2, torch.float64)
    assert rel(spline_backward(saved, ge0, w, 2), torch.func.vjp(f, vec)[1](ge0)[0]) <= BAR


@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (2, 7, 2), (3, 20, 3)])
def test_fc_tangent_mode_is_the_fold_of_one_job(seed, n, isolated):
    """The tangent gather holds the undisplaced rows with vdot = e_alpha ([nbr = j] - [ctr = j]); its fold of gvec_dot is
    -F_dot, the limit of fc_spec's central difference of a displaced pair of jobs whose gradients are g +- h gvec_dot."""
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated)
    atoms = torch.randperm(n, generator=torch.Generator().manual_seed(seed))
    cptr, cen, coff, ea = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    fptr, col = fc_spec.columns(cptr, cen, row_ptr, nbr, n)
    U = 3 * n
    rp, cb, cz, nz, vb, vd = hvp_spec.fc_gather_tangent(pos, shift, torch.float64, atoms, cptr, cen, coff, ea, row_ptr, nbr, 0, U)
    h = 0.25
    _, _, _, _, vfd = fc_spec.gather(pos, shift, h, torch.float64, atoms, cptr, cen, coff, ea, row_ptr, nbr, 0, U)
    gd = torch.randn(vb.shape[0], 3, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64)
    # unit by unit: the displaced pair is vec +- h vdot, and g(vec) = vec . A for a linear g gives gd = vdot . A
    e = 0
    pairs = []
    for u in range(U):
        Eu = int(ea[u // 3])
        assert torch.equal(vfd[2 * e : 2 * e + Eu], vb[e : e + Eu] + h * vd[e : e + Eu])
        assert torch.equal(vfd[2 * e + Eu : 2 * e + 2 * Eu], vb[e : e + Eu] - h * vd[e : e + Eu])
        pairs += [gd[e : e + Eu] * h, -gd[e : e + Eu] * h]
        e += Eu
    g_fd = torch.cat(pairs) if pairs else torch.zeros(0, 3, dtype=torch.float64)
    want = fc_spec.fold(g_fd, h, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, 0, U)
    got = hvp_spec.fc_fold_tangent(gd, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, 0, U)
    assert set(got) == set(want)
    for k in got:
        torch.testing.assert_close(got[k], want[k], rtol=1e-13, atol=1e-13)


# ---- the whole tangent sequencing on the restatements -------------------------------------------------------------------
HVP_KERNELS = ("sh_jvp", "sh_hvp", "act_bwd_jvp", "radial_pq_jvp", "radial_jvp", "radial_pq_hvp", "radial_hvp", "zbl_hvp")


@pytest.fixture()
def spec_kernels(monkeypatch):
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    for name in HVP_KERNELS:
        monkeypatch.setattr(_lib, name, getattr(hvp_spec, name))
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))


@pytest.mark.parametrize("variant", ["default", "nofold", "product_embed", "zbl", "lmax3_L3"])
def test_composed_tangent_equals_the_oracle_hessian(variant, spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel
    from allegro_b200.nn._hessian import edge_energy_grad_tangent
    from allegro_b200.phonons import _energy_terms
    from oracle.model_ref import AllegroOracle

    small = dict(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16, scalar_embed_mlp_hidden_layers_width=16,
                 allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=8)
    sysname = "c3" if variant == "zbl" else "c2"
    kw = systems.model_kwargs(sysname, 30.0, "float64")
    kw.update(small)
    if variant == "zbl":
        kw.update(pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]},
                  per_type_energy_scales=[1.5, 0.5, 2.0])
    if variant == "lmax3_L3":
        kw.update(l_max=3, num_layers=3)
    if variant == "nofold":  # two hidden layers: the per-type-pair radial kernel without the first layer folded in
        kw.update(scalar_embed_mlp_hidden_layers_depth=2)
    if variant == "product_embed":  # not 8 Bessels: the product-embedding radial kernel
        kw.update(radial_chemical_embed=dict(kw["radial_chemical_embed"], num_bessels=5))
    oracle = AllegroOracle(**kw)
    model = AllegroModel(**dict(kw, model_dtype="float64"))
    model.load_state_dict(oracle.state_dict())
    inner = model.model
    g = torch.Generator().manual_seed(1)
    n = 6
    pos = 1.7 * torch.randn(n, 3, generator=g, dtype=torch.float64)
    types = torch.randint(0, len(kw["type_names"]), (n,), generator=g)
    row_ptr, ctr, nbr, sv = frame_list(pos, None, (False,) * 3, kw["r_max"])
    csr = D.EdgeCSR(n, ctr.to(torch.int32), nbr.to(torch.int32), row_ptr.to(torch.int32), None, int((row_ptr[1:] - row_ptr[:-1]).max()))
    core = inner.core()
    up = inner._upstream
    if variant == "nofold":
        assert up.PQ is not None and not up.fold_radial
    if variant == "product_embed":
        assert up.PQ is None
    types_i32 = types.to(torch.int32)
    gscale, pair = _energy_terms(inner, core, types, torch.device("cpu"))
    vec = pos[nbr] - pos[ctr] + sv
    atoms = torch.tensor([0, 2, 5])
    H = hessian_rows(oracle, pos, types, ctr, nbr, sv, atoms)
    rows = torch.zeros_like(H)
    for a, j in enumerate(atoms.tolist()):
        for alpha in range(3):
            vdot = torch.zeros_like(vec)
            vdot[:, alpha] = (nbr == j).double() - (ctr == j).double()
            _, gvd = edge_energy_grad_tangent(core, inner._upstream, csr, vec, vdot, types_i32, gscale, pair)
            rows[a, :, alpha] = -kernel_spec.force_scatter(gvd, csr, n)
    err = rel(rows, H)
    assert err <= 1e-10, err


def test_new_symbols_in_header_and_library():
    hdr = open(os.path.join(ROOT, "include", "allegro_b200.h")).read()
    names = HVP_KERNELS + ("fc_gather_tangent", "fc_fold_tangent")
    for name in names:
        assert f"int ab2_{name}(" in hdr, name
        assert f"ab2_{name}" in _lib.exported_symbols()
    so = _lib.lib_path()
    if not os.path.exists(so):
        pytest.skip("the shared library is not built")
    import ctypes

    lib = ctypes.CDLL(so)
    for name in names:
        assert hasattr(lib, f"ab2_{name}"), name
