"""Per-atom virials and the heat current on the GPU: the two kernels (ab2_force_virial_scatter, ab2_frame_heat_current)
against fp64 restatements, and W / J of the model against checks that do not trust the code under test -- the oracle's
edge-vector gradients, the position Jacobian of the oracle's per-atom energies, the existing virial output, and central
differences of sum_i r_i E_i along the velocities."""
import pytest
import torch

from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.batch import collate, split

from golden_util import load_models, unpack_state_dict
from test_host_atomic_virial import oracle_w_j

pytestmark = pytest.mark.gpu
DEV = "cuda"
SMALL = dict(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16,
             scalar_embed_mlp_hidden_layers_width=16, allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=8)
ZBL = dict(SMALL, readout_mlp_hidden_layers_width=16, per_type_energy_scales=[0.7, 1.3, 0.9], per_type_energy_shifts=[0.1, -0.2, 0.3],
           pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0) if a.numel() else 0.0


def _dev(d):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


# --------------------------------------------------------------------------- #
# the kernels
# --------------------------------------------------------------------------- #
def _ragged(N, n_total, seed):
    """Random CSR: empty centres, a few long rows, neighbours drawn from a pool that leaves 10 % of the atoms (owned and
    ghost) nobody's neighbour."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 40, (N,), generator=g)
    deg[torch.rand(N, generator=g) < 0.2] = 0
    deg[torch.randperm(N, generator=g)[:5]] = 400
    row_ptr = torch.zeros(N + 1, dtype=torch.int32)
    row_ptr[1:] = deg.cumsum(0).to(torch.int32)
    E = int(row_ptr[-1])
    ctr = torch.repeat_interleave(torch.arange(N, dtype=torch.int32), deg)
    atoms = torch.randperm(n_total, generator=g)
    pool = atoms[: n_total * 9 // 10]
    nbr = pool[torch.randint(0, pool.numel(), (E,), generator=g)].to(torch.int32)
    lonely = atoms[n_total * 9 // 10:]
    csr = D.EdgeCSR(N, ctr.to(DEV), nbr.to(DEV), row_ptr.to(DEV), None, int(deg.max()))
    return csr, ctr, nbr, lonely, g


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["float64", "float32"])
def test_force_virial_scatter_kernel(dtype):
    N, n_total = 3000, 3500
    csr, ctr, nbr, lonely, g = _ragged(N, n_total, 3)
    E = ctr.numel()
    vec = torch.randn(E, 3, generator=g, dtype=torch.float64).to(dtype)
    gv = torch.randn(E, 3, generator=g, dtype=torch.float64).to(dtype)
    F, W = _lib.force_virial_scatter(vec.to(DEV), gv.to(DEV), csr, n_total)
    assert F.shape == (n_total, 3) and W.shape == (n_total, 3, 3) and W.dtype == dtype
    assert torch.equal(F, _lib.force_scatter(gv.to(DEV), csr, n_total))           # F bitwise today's
    F2, W2 = _lib.force_virial_scatter(vec.to(DEV), gv.to(DEV), csr, n_total)
    assert torch.equal(W, W2) and torch.equal(F, F2)                                # fixed order: bitwise reproducible
    outer = vec.double().unsqueeze(2) * gv.double().unsqueeze(1)
    W_ref = torch.zeros(n_total, 3, 3, dtype=torch.float64).index_add_(0, nbr.long(), -outer)
    tol = 1e-12 if dtype == torch.float64 else 1e-6
    assert _rel(W, W_ref) < tol
    assert bool((W.cpu()[lonely] == 0).all())                                        # no column: exactly 0
    assert bool((W.cpu()[N:] != 0).any())                                            # ghost rows get their columns
    # no edge at all
    empty = D.EdgeCSR(N, torch.zeros(0, dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV),
                      torch.zeros(N + 1, dtype=torch.int32, device=DEV), None, 0)
    z = torch.zeros(0, 3, dtype=dtype, device=DEV)
    F0, W0 = _lib.force_virial_scatter(z, z, empty, n_total)
    assert bool((F0 == 0).all()) and bool((W0 == 0).all())


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["float64", "float32"])
def test_frame_heat_current_kernel(dtype):
    g = torch.Generator().manual_seed(5)
    sizes = torch.tensor([0, 0] + [7] * 2000 + [0] + [int(torch.randint(1, 40, (1,), generator=g)) for _ in range(300)]
                         + [120_000] + [0, 2047, 2048, 2049, 1])
    B, n = sizes.shape[0], int(sizes.sum())
    ptr = torch.cat([torch.zeros(1, dtype=torch.long), sizes.cumsum(0)])
    e = torch.randn(n, generator=g, dtype=torch.float64).to(dtype)
    v = torch.randn(n, 3, generator=g, dtype=torch.float64).to(dtype)
    W = torch.randn(n, 3, 3, generator=g, dtype=torch.float64).to(dtype)
    fp = ptr.to(DEV, torch.int32)
    J = _lib.frame_heat_current(e.to(DEV), v.to(DEV), W.to(DEV), fp)
    assert J.shape == (B, 3) and J.dtype == dtype
    assert torch.equal(J, _lib.frame_heat_current(e.to(DEV), v.to(DEV), W.to(DEV), fp))
    per = e.double().unsqueeze(1) * v.double() + (W.double() @ v.double().unsqueeze(2)).squeeze(2)
    seg = torch.repeat_interleave(torch.arange(B), sizes)
    ref = torch.zeros(B, 3, dtype=torch.float64).index_add_(0, seg, per)
    scale = torch.zeros(B, 3, dtype=torch.float64).index_add_(0, seg, e.double().abs().unsqueeze(1) * v.double().abs()
                                                                 + (W.double().abs() @ v.double().abs().unsqueeze(2)).squeeze(2))
    tol = 1e-13 if dtype == torch.float64 else 1e-7
    assert bool(((J.double().cpu() - ref).abs() <= tol * scale.clamp(min=1e-300)).all())
    assert bool((J.cpu()[sizes == 0] == 0).all())
    # a frame's J does not change when the other frames change, nor when it is evaluated alone
    e2, v2, W2 = e.clone(), v.clone(), W.clone()
    big = int((sizes == 120_000).nonzero()[0, 0])
    keep = torch.zeros(n, dtype=torch.bool)
    for b in (big, 5):
        keep[int(ptr[b]):int(ptr[b + 1])] = True
    e2[~keep] = torch.randn(int((~keep).sum()), generator=g, dtype=torch.float64).to(dtype)
    v2[~keep] *= 2
    W2[~keep] *= -3
    J2 = _lib.frame_heat_current(e2.to(DEV), v2.to(DEV), W2.to(DEV), fp)
    for b in (big, 5):
        assert torch.equal(J2[b], J[b])
        p0, p1 = int(ptr[b]), int(ptr[b + 1])
        alone = _lib.frame_heat_current(e[p0:p1].to(DEV), v[p0:p1].to(DEV), W[p0:p1].to(DEV),
                                        torch.tensor([0, p1 - p0], dtype=torch.int32, device=DEV))
        assert torch.equal(alone[0], J[b])


# --------------------------------------------------------------------------- #
# the model's W against the oracle's edge-vector gradients
# --------------------------------------------------------------------------- #
def _pair(name, scale, dtype, **over):
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    d = systems.make_system(name, scale)
    kw = systems.model_kwargs(name, d[D.EDGE_INDEX_KEY].shape[1] / d[D.POSITIONS_KEY].shape[0], "float64")
    kw.update(over)
    if "r_max" in over:
        d[D.EDGE_INDEX_KEY], d[D.EDGE_CELL_SHIFT_KEY] = D.neighbor_list(d[D.POSITIONS_KEY], over["r_max"], d[D.CELL_KEY])
    oracle = AllegroOracle(**kw)
    kwm = dict(kw, model_dtype=dtype)
    model = AllegroModel(**kwm)
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to(DEV).model, d


def _golden(name):
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    rec = {r["name"]: r for r in load_models()}[name]
    sd = unpack_state_dict(rec["state_dict"])
    oracle = AllegroOracle(**rec["kwargs"])
    oracle.load_state_dict(sd, strict=True)
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(sd, strict=True)
    return oracle, model.to(DEV).model, dict(rec["data"])


def _zbl_pair(dtype="float64"):
    d = systems.make_system("c3", 2)
    return _pair("c3", 2, dtype, **dict(ZBL, avg_num_neighbors=d[D.EDGE_INDEX_KEY].shape[1] / 8))


ORACLE_CASES = {
    "c2_s3_f64": lambda: _pair("c2", 3, "float64"),
    "c2_s3_f32": lambda: _pair("c2", 3, "float32"),
    "c5_small_f64": lambda: _pair("c5", 2, "float64", **SMALL),
    "spline_f64": lambda: _golden("spline_embed_reftest_cfg"),
    "zbl_f64": lambda: _zbl_pair(),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_atomic_virial_against_edge_oracle(case):
    oracle, model, d = ORACLE_CASES[case]()
    n = d[D.POSITIONS_KEY].shape[0]
    vel = torch.randn(n, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    W_ref, J_ref, e_ref = oracle_w_j(oracle, d, vel)
    inp = _dev(d)
    inp[D.VELOCITY_KEY] = vel.to(DEV)
    out = model.energy_and_forces(inp, stress=True, heat_current=True)
    tol = 1e-9 if model.model_dtype == torch.float64 else 1e-4
    assert _rel(out[D.ATOMIC_VIRIAL_KEY], W_ref) < tol, _rel(out[D.ATOMIC_VIRIAL_KEY], W_ref)
    assert _rel(out[D.HEAT_CURRENT_KEY][0], J_ref) < tol, (out[D.HEAT_CURRENT_KEY], J_ref)
    # the symmetric part of the sum is today's virial output (on the scale of the summed terms: the sum cancels)
    W = out[D.ATOMIC_VIRIAL_KEY].double().cpu()
    Ws = W.sum(0)
    err = float((0.5 * (Ws + Ws.T) - out[D.VIRIAL_KEY][0].double().cpu()).abs().max())
    assert err <= (1e-12 if model.model_dtype == torch.float64 else 1e-5) * float(W.abs().sum(0).max()), err


def test_atomic_virial_against_the_position_jacobian():
    """No edge decomposition: W[j] = sum_{i != j} (r_i - r_j)_image (x) dE_i/dr_j from the oracle's per-atom energies,
    on a cell wider than 2 r_max along every axis (every pair has at most one image within r_max)."""
    r_max = 4.0
    oracle, model, d = _pair("c2", 3, "float64", r_max=r_max)
    cell = d[D.CELL_KEY].view(3, 3)
    widths = torch.linalg.det(cell).abs() / torch.stack([torch.linalg.cross(cell[(a + 1) % 3], cell[(a + 2) % 3]).norm() for a in range(3)])
    assert bool((widths > 2 * r_max).all()), widths
    n = d[D.POSITIONS_KEY].shape[0]
    out = model.energy_and_forces(_dev(d), atomic_virial=True)
    pos = d[D.POSITIONS_KEY].double().clone().requires_grad_(True)
    inp = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: d[D.ATOM_TYPE_KEY], D.EDGE_INDEX_KEY: d[D.EDGE_INDEX_KEY],
           D.EDGE_CELL_SHIFT_KEY: d[D.EDGE_CELL_SHIFT_KEY], D.CELL_KEY: cell}
    with torch.enable_grad():
        e = oracle.model(inp)[D.PER_ATOM_ENERGY_KEY].reshape(-1)
        jac = torch.stack([torch.autograd.grad(e[i], pos, retain_graph=True)[0] for i in range(n)])  # [i, j, 3]
    p = pos.detach()
    diff = p.unsqueeze(1) - p.unsqueeze(0)                                    # [i, j] = r_i - r_j
    frac = diff @ torch.linalg.inv(cell)
    diff = (frac - torch.round(frac)) @ cell                                  # the minimum image
    W_ref = torch.einsum("ija,ijb->jab", diff, jac)
    assert _rel(out[D.ATOMIC_VIRIAL_KEY], W_ref) < 1e-9, _rel(out[D.ATOMIC_VIRIAL_KEY], W_ref)


# --------------------------------------------------------------------------- #
# heat current by central differences, and ghosts against the periodic frame
# --------------------------------------------------------------------------- #
def _cluster(n=24, seed=3, r_min=2.0, half=5.0):
    g = torch.Generator().manual_seed(seed)
    pts = []
    while len(pts) < n:
        p = (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * half
        if all(float((p - q).norm()) > r_min for q in pts):
            pts.append(p)
    return torch.stack(pts)


def _ghost(d):
    """data.to_ghost_format(d) and the owner of every ghost."""
    g = D.to_ghost_format(d)
    g.pop("num_local_atoms")
    owners = d[D.EDGE_INDEX_KEY][1, d[D.EDGE_CELL_SHIFT_KEY].abs().sum(-1) != 0]
    return g, owners


def _fd_case(kind):
    if kind == "cluster":
        oracle, model, d = _pair("c2", 3, "float64")
        pos = _cluster()
        types = torch.zeros(pos.shape[0], dtype=torch.long)
    elif kind == "zbl_cluster":
        oracle, model, d = _zbl_pair()
        pos = _cluster(n=20, seed=4, r_min=1.9, half=4.0)
        types = torch.arange(pos.shape[0]) % 3
    else:  # the ghost format of a periodic c2 frame: ghosts move with their owners
        oracle, model, d = _pair("c2", 3, "float64")
        g, owners = _ghost(d)
        n = d[D.POSITIONS_KEY].shape[0]
        v = torch.randn(n, 3, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
        return model, g, torch.cat([v, v[owners]])
    ei = D.neighbor_list(pos, model.r_max, None, (False,) * 3)[0]
    v = torch.randn(pos.shape[0], 3, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    return model, {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei}, v


@pytest.mark.parametrize("kind", ["cluster", "ghost_c2", "zbl_cluster"])
def test_heat_current_by_central_differences(kind):
    """d/dt sum_i r_i E_i = sum_i E_i v_i + sum_i W[i] v_i - sum_i r_i (F_i . v_i) along r(t) = r + t v (no cell, one fixed
    list), with only atomic_energy and forces on the left-hand side."""
    model, d, v = _fd_case(kind)
    dd = _dev(d)
    vd = v.to(DEV)

    def G(t):
        x = dict(dd)
        x[D.POSITIONS_KEY] = dd[D.POSITIONS_KEY] + t * vd
        e = model.energy_and_forces(x)[D.PER_ATOM_ENERGY_KEY].double().reshape(-1, 1)
        return (x[D.POSITIONS_KEY][: e.shape[0]].double() * e).sum(0)

    h = 1e-4
    lhs = (G(h) - G(-h)) / (2 * h)
    x = dict(dd)
    x[D.VELOCITY_KEY] = vd
    out = model.energy_and_forces(x, heat_current=True)
    F = out[D.FORCE_KEY].double()
    rhs = out[D.HEAT_CURRENT_KEY][0].double() - (dd[D.POSITIONS_KEY].double() * (F * vd).sum(-1, keepdim=True)).sum(0)
    assert float((lhs - rhs).abs().max()) <= 1e-6 * float(rhs.abs().max()), (lhs, rhs)


def test_ghost_format_against_periodic():
    oracle, model, d = _pair("c2", 3, "float64")
    n = d[D.POSITIONS_KEY].shape[0]
    vel = torch.randn(n, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(DEV)
    per = _dev(d)
    per[D.VELOCITY_KEY] = vel
    ref = model.energy_and_forces(per, heat_current=True)
    g, owners = _ghost(d)
    g = _dev(g)
    owners = owners.to(DEV)
    vg = torch.cat([vel, vel[owners]])
    ga = dict(g, **{D.VELOCITY_KEY: vg})                                   # appended ghosts as edge_index
    gb = {D.POSITIONS_KEY: g[D.POSITIONS_KEY], D.ATOM_TYPE_KEY: g[D.ATOM_TYPE_KEY], D.VELOCITY_KEY: vg,
          D.CSR_KEY: D.build_csr(g[D.EDGE_INDEX_KEY], n)}                 # rows for the owned atoms only
    for o in (model.energy_and_forces(ga, heat_current=True), model.energy_and_forces(gb, heat_current=True)):
        W = o[D.ATOMIC_VIRIAL_KEY]
        folded = W[:n].clone().index_add_(0, owners, W[n:])
        assert _rel(folded, ref[D.ATOMIC_VIRIAL_KEY]) < 1e-10
        assert _rel(o[D.HEAT_CURRENT_KEY], ref[D.HEAT_CURRENT_KEY]) < 1e-10  # ghosts carry no energy in this model


# --------------------------------------------------------------------------- #
# batches, graph replay, calculator, opt-out
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_batch_equals_single_frames(dtype):
    from test_gpu_frames import _model, _model_frames

    oracle, model, kw = _model("c2", dtype)
    g = torch.Generator().manual_seed(43)
    frames = _model_frames("c2", 1, g, periodic_only=False)
    frames.append({D.POSITIONS_KEY: torch.tensor([[0.0, 0, 0], [9.0, 0, 0]], dtype=torch.float64), D.ATOM_TYPE_KEY: torch.zeros(2, dtype=torch.long)})
    for i, f in enumerate(frames):
        f[D.VELOCITY_KEY] = torch.randn(f[D.POSITIONS_KEY].shape[0], 3, generator=g, dtype=torch.float64)
    batch = collate([_dev(f) for f in frames], kw["r_max"])
    out = model.energy_and_forces_frames(batch, heat_current=True)
    assert out[D.HEAT_CURRENT_KEY].shape == (len(frames), 3)
    fp64 = dtype == "float64"
    for b, (fin, fo) in enumerate(zip(split(batch), split(out))):
        one = model.model.energy_and_forces(fin, heat_current=True)
        for k in (D.ATOMIC_VIRIAL_KEY, D.HEAT_CURRENT_KEY):
            if fp64:  # tp_bwd adds with fp64 atomics: not bitwise (DESIGN section 4.4)
                assert _rel(fo[k], one[k]) < 1e-12, (b, k)
            else:
                assert torch.equal(fo[k], one[k]), (b, k, _rel(fo[k], one[k]))
        if fin[D.CSR_KEY].num_edges == 0:  # the one-atom frame and the two isolated atoms
            assert bool((fo[D.ATOMIC_VIRIAL_KEY] == 0).all())
            ev = (fo[D.PER_ATOM_ENERGY_KEY].double() * fin[D.VELOCITY_KEY].double()).sum(0)
            assert _rel(fo[D.HEAT_CURRENT_KEY][0], ev) < 1e-6


def test_calculator_and_graph_replay_random_walk():
    from allegro_b200.calculator import AllegroCalculator

    oracle, model, d = _pair("c2", 3, "float64")
    wrapped = model  # FusedAllegroEnergy: the calculator takes the energy model itself too
    pos, cell, types = d[D.POSITIONS_KEY], d[D.CELL_KEY], d[D.ATOM_TYPE_KEY]
    calcs = [AllegroCalculator(wrapped, 5.0, skin=0.6, use_graph=ug, compute_atomic_virial=True, compute_heat_current=True) for ug in (True, False)]
    g = torch.Generator().manual_seed(4)
    p = pos.clone()
    for step in range(4):
        vel = torch.randn(p.shape, generator=g, dtype=torch.float64)
        res = [c.compute(p.to(DEV), cell.to(DEV), types.to(DEV), velocities=vel.to(DEV)) for c in calcs]
        ei, sh = D.neighbor_list(p, 5.0, cell, (True, True, True))
        W_ref, J_ref, _ = oracle_w_j(oracle, {D.POSITIONS_KEY: p, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei,
                                             D.EDGE_CELL_SHIFT_KEY: sh}, vel)
        for r in res:
            assert _rel(r["atomic_virial"], W_ref) < 1e-9, (step, _rel(r["atomic_virial"], W_ref))
            assert _rel(r["heat_current"][0], J_ref) < 1e-9, step
        assert _rel(res[0]["atomic_virial"], res[1]["atomic_virial"]) < 1e-12
        assert _rel(res[0]["heat_current"], res[1]["heat_current"]) < 1e-12
        p = p + 0.1 * torch.randn(p.shape, generator=g, dtype=p.dtype)
    assert calcs[0].n_evaluations == 4 and calcs[0].num_edges > ei.shape[1]  # the skin list is longer than the exact one


def test_opt_out_fp32():
    oracle, model, d = _pair("c2", 3, "float32")
    dd = _dev(d)
    plain = model.energy_and_forces(dd, stress=True)
    assert D.ATOMIC_VIRIAL_KEY not in plain and D.HEAT_CURRENT_KEY not in plain
    withv = dict(dd, **{D.VELOCITY_KEY: torch.randn(d[D.POSITIONS_KEY].shape, dtype=torch.float64).to(DEV)})
    full = model.energy_and_forces(withv, stress=True, heat_current=True)
    for k in (D.FORCE_KEY, D.PER_ATOM_ENERGY_KEY, D.STRESS_KEY):
        assert torch.equal(plain[k], full[k]), k
    again = model.energy_and_forces(withv, stress=True)  # velocities present, flags off: no new keys
    assert set(again) == set(plain) | {D.VELOCITY_KEY}
