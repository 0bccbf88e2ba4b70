"""world_size-2/3 gloo tests (CPU) of the slab decomposition on triclinic cells: slabs cut in fractional coordinates along
lattice row 0 (``halo.SlabGeometry``).

* The torch restatement of ab2_slab_plan_count_lattice below against a one-atom-at-a-time Python brute force, on slanted
  and tilted faces, a LAMMPS box at large tilt, hcp, a left-handed and a rotated cell, with atoms on the faces, one ulp
  below 1, 100 cells out and at negative coordinates.
* ``SlabDecomposition`` + ``DistributedAllegro(stress, atomic_virial, heat_current)`` on those cells against the fp64
  oracle on an exact r_max list (tests/nlist_lattice_oracle.py), and the same crystal in three bases and in a rotated
  frame.
* ``DistributedCalculator`` velocity-Verlet trajectories on a slanted-face and a rotated cell, checked at every step.
* Refusals on every rank before any exchange: singular and near-coplanar cells, slabs whose height (not row length) is
  below r_max + skin, an atom that moved more than one slab in s_0.

Each rank runs the fused model through the spec kernels (as in tests/test_halo_gloo_md.py); the device kernels are
checked against the restatement in tests/test_gpu_slab_md_lattice.py."""
import math

import numpy as np
import pytest
import torch

from allegro_b200 import data as D
from allegro_b200 import systems

from test_halo_gloo_md import R_MAX, SKIN, _nz, _rel, _spawn, md_frame

F64 = torch.float64


# ---- torch restatement of ab2_slab_plan_count_lattice (csrc/slab_md.cu) ------------------------------------------------
def lattice_inverse(rows):
    """(h, hinv[x][a], H_0) as lattice.cuh computes them, in Python floats"""
    h = [[float(v) for v in r] for r in (rows.tolist() if torch.is_tensor(rows) else rows)]
    cr = [D._cross(h[(a + 1) % 3], h[(a + 2) % 3]) for a in range(3)]
    det = h[0][0] * cr[0][0] + h[0][1] * cr[0][1] + h[0][2] * cr[0][2]
    hinv = [[cr[a][x] / det for a in range(3)] for x in range(3)]
    return h, hinv, D._lattice_metrics(h)[1][0]


def _frac(p, hinv, a):
    """s_a = (p_0 hinv[0][a] + p_1 hinv[1][a]) + p_2 hinv[2][a], fp64, no FMA"""
    return (p[:, 0] * hinv[0][a] + p[:, 1] * hinv[1][a]) + p[:, 2] * hinv[2][a]


def slab_wrap_classify_lattice_spec(pos, image, rows, rank, world, jump=float("inf")):
    """mode 0: img_a = floor(s_a), pos <- pos - sum_a img_a h_a in fp64 rounded once, image += img; classify by
    clamp(floor(s_0 world), 0, world - 1) of the wrapped position, refuse by the unwrapped s_0"""
    h, hinv, _ = lattice_inverse(rows)
    p = pos.double()
    img = [torch.floor(_frac(p, hinv, a)) for a in range(3)]
    s0 = _frac(p, hinv, 0)
    for x in range(3):
        shift = (img[0] * h[0][x] + img[1] * h[1][x]) + img[2] * h[2][x]
        pos[:, x] = (p[:, x] - shift).to(pos.dtype)
    for a in range(3):
        image[:, a] += img[a].to(torch.int32)
    lo, hi = rank / world, (rank + 1) / world
    s = torch.floor(_frac(pos.double(), hinv, 0) * float(world)).long().clamp(0, world - 1)
    d = (s - rank) % world
    far = (s0 < lo - jump) | (s0 >= hi + jump)
    move = ~far & (d != 0)
    if world == 2:
        left, right = move & (s0 < lo), move & ~(s0 < lo)
    else:
        left, right = move & (d == world - 1), move & (d == 1)
        far = far | (move & ~left & ~right)
    return _nz(~far & (d == 0)), _nz(left), _nz(right), int(far.sum())


def slab_faces_lattice_spec(pos, rows, rank, world, r_list):
    """mode 1: s_0 < lo + r_list / H_0 and s_0 >= hi - r_list / H_0, fp64"""
    _, hinv, H0 = lattice_inverse(rows)
    s0 = _frac(pos.double(), hinv, 0)
    lo, hi = rank / world, (rank + 1) / world
    return _nz(s0 < lo + r_list / H0), _nz(s0 >= hi - r_list / H0)


def _brute_plan(pos, rows, rank, world, jump, r_list):
    """one atom at a time in Python floats (fp64 frames): the same rules, lists built by appending in atom order"""
    h, hinv, H0 = lattice_inverse(rows)
    lo, hi = rank / world, (rank + 1) / world
    stay, left, right, far, wrapped, images, low, high = [], [], [], 0, [], [], [], []
    for i, p in enumerate(pos.tolist()):
        fr = lambda q, a: (q[0] * hinv[0][a] + q[1] * hinv[1][a]) + q[2] * hinv[2][a]  # noqa: E731
        img = [math.floor(fr(p, a)) for a in range(3)]
        w = [p[x] - ((img[0] * h[0][x] + img[1] * h[1][x]) + img[2] * h[2][x]) for x in range(3)]
        wrapped.append(w)
        images.append(img)
        s0 = fr(p, 0)
        s = min(max(math.floor(fr(w, 0) * world), 0), world - 1)
        d = (s - rank) % world
        if s0 < lo - jump or s0 >= hi + jump:
            far += 1
        elif d == 0:
            stay.append(i)
        elif world == 2:
            (left if s0 < lo else right).append(i)
        elif d == world - 1:
            left.append(i)
        elif d == 1:
            right.append(i)
        else:
            far += 1
        sw = fr(w, 0)
        if sw < lo + r_list / H0:
            low.append(i)
        if sw >= hi - r_list / H0:
            high.append(i)
    return stay, left, right, far, wrapped, images, low, high


def _rotation(seed=3):
    g = torch.Generator().manual_seed(seed)
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=F64))
    q = q * torch.sign(torch.diagonal(r))
    return q if float(torch.det(q)) > 0 else -q


def plan_cells():
    """(name, rows): the faces of the first two are the same planes x = const and slanted planes, H_0 = L / sqrt 2"""
    L = 18.0
    a, b, c = torch.tensor([L, 0.0, 0.0], dtype=F64), torch.tensor([0.0, L, 0.0], dtype=F64), torch.tensor([0.0, 0.0, 12.0], dtype=F64)
    import nlist_lattice_cases as NC

    slanted = torch.stack([a, b + a, c])
    return [("tilted image (a+b, b, c)", torch.stack([a + b, b, c])), ("slanted faces (a, b+a, c)", slanted),
            ("lammps large tilt", NC.lammps(36.0, 18.0, 15.0, 17.9, -17.9, 8.9)), ("hcp", NC.hcp(reps=(6, 4, 3))[1]),
            ("left-handed", torch.stack([a, c, b + 0.3 * a])), ("rotated", slanted @ _rotation().T)]


def plan_atoms(rows, world, seed=5):
    """(name, fp64 positions, jump): random in and around the cell, the faces s_0 = k / world, s = 1 - ulp, 100 cells
    out, negative coordinates, everyone emigrating (jump one slab), none"""
    g = torch.Generator().manual_seed(seed)
    one_ulp = 1.0 - 2.0**-53
    rnd = (torch.rand(200, 3, generator=g, dtype=F64) * 1.4 - 0.2) @ rows
    faces = torch.tensor([[k / world, 0.3, 0.6] for k in range(world + 1)] + [[k / world, -0.0, 1.0] for k in range(world + 1)], dtype=F64) @ rows
    ulp = torch.tensor([[one_ulp, 0.5, 0.5], [0.25, one_ulp, one_ulp], [-2.0**-60, 0.5, -1e-18], [one_ulp, one_ulp, one_ulp]], dtype=F64) @ rows
    far = (torch.rand(20, 3, generator=g, dtype=F64) + torch.tensor([100.0, -100.0, 100.0], dtype=F64)) @ rows
    neg = -torch.rand(20, 3, generator=g, dtype=F64) * 15.0
    mid = (0.5 + 0.5 / world) * torch.ones(30, 1, dtype=F64)
    emig = torch.cat([mid + 0.1 / world * torch.rand(30, 1, generator=g, dtype=F64), torch.rand(30, 2, generator=g, dtype=F64)], 1) @ rows
    return [("random", rnd, None), ("faces", faces, None), ("one ulp below 1", ulp, None), ("100 cells out", far, None), ("negative", neg, None),
            ("all emigrate", emig, "slab"), ("empty", torch.zeros(0, 3, dtype=F64), None)]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("cell", range(6))
def test_lattice_plan_restatement_matches_brute_force(world, cell):
    cname, rows = plan_cells()[cell]
    h64 = rows.double()
    for name, pos, jump in plan_atoms(rows, world):
        jump = {None: float("inf"), "slab": 1.0 / world}[jump]
        for rank in range(world):
            p = pos.clone()
            image = torch.zeros(p.shape[0], 3, dtype=torch.int32)
            stay, left, right, far = slab_wrap_classify_lattice_spec(p, image, rows, rank, world, jump)
            b = _brute_plan(pos, rows, rank, world, jump, R_MAX + SKIN)
            assert (stay.tolist(), left.tolist(), right.tolist(), far) == b[:4], (cname, name, rank)
            assert p.tolist() == b[4] and image.tolist() == b[5], (cname, name)
            low, high = slab_faces_lattice_spec(p, rows, rank, world, R_MAX + SKIN)
            assert (low.tolist(), high.tolist()) == b[6:], (cname, name, rank)
            if p.shape[0]:
                s = p @ torch.linalg.inv(h64)
                assert bool((s > -1e-12).all() and (s < 1 + 1e-12).all()), (cname, name)  # wrapped into the cell
                assert torch.allclose(p + image.double() @ h64, pos, rtol=0, atol=1e-9 * (1 + float(pos.abs().max()))), (cname, name)
        if name == "all emigrate":
            b = _brute_plan(pos, rows, world - 2, world, jump, 0.0)  # the slab below theirs
            assert len(b[0]) == 0 and len(b[1]) + len(b[2]) + b[3] == pos.shape[0] and len(b[1]) + len(b[2]) > 0, cname


# ---- the distributed runs ---------------------------------------------------------------------------------------------
def _install():
    from test_halo_gloo_md import _install as install_md

    from allegro_b200 import _lib

    install_md()
    _lib.slab_wrap_classify_lattice = slab_wrap_classify_lattice_spec
    _lib.slab_faces_lattice = slab_faces_lattice_spec


def _init(rank, world, port):
    import os

    import torch.distributed as dist

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    _install()


def _model():
    from test_halo_gloo_md import _model as md_model
    from test_halo_gloo_virial import _kwargs

    return md_model(_kwargs("c2"))


def _np(t):
    return t.detach().double().cpu().numpy().copy()


def _grid_gas(rows, n, seed):
    """a jittered fractional grid n0 x n1 x n2 in the cell (every pair some Angstrom apart)"""
    g = torch.Generator().manual_seed(seed)
    ijk = torch.stack(torch.meshgrid(*[torch.arange(k, dtype=F64) for k in n], indexing="ij"), -1).reshape(-1, 3)
    return (ijk + 0.5) / torch.tensor(n, dtype=F64) @ rows + 0.05 * torch.randn(int(np.prod(n)), 3, generator=g, dtype=F64)


def static_frames():
    """(name, pos, rows, vel): the c2 crystal (6, 6, 3) in its cubic basis, two tilted bases, a left-handed one and a
    rotated frame; a LAMMPS box at large tilt and hcp"""
    import nlist_lattice_cases as NC

    pos, cell, _ = systems.make_positions("c2", (6, 6, 3))
    g = torch.Generator().manual_seed(11)
    pos = pos + 0.1 * torch.randn(pos.shape, generator=g, dtype=F64)
    vel = torch.randn(pos.shape, generator=g, dtype=F64)
    A, B, C = cell.double()
    R = _rotation()
    out = [("cubic", pos, cell.double(), vel), ("(a+b, b, c)", pos, torch.stack([A + B, B, C]), vel),
           ("(a, b+a, c)", pos, torch.stack([A, B + A, C]), vel), ("left-handed (a, c, b)", pos, torch.stack([A, C, B]), vel),
           ("rotated (a, b+a, c)", pos @ R.T, torch.stack([A, B + A, C]) @ R.T, vel @ R.T)]
    lam = NC.lammps(36.0, 18.0, 15.0, 17.9, -17.9, 8.9)
    hp, hrows = NC.hcp(reps=(6, 4, 3))
    for name, p, rows in (("lammps large tilt", _grid_gas(lam, (12, 8, 6), 12), lam), ("hcp", hp, hrows)):
        out.append((name, p, rows, torch.randn(p.shape, generator=g, dtype=F64)))
    return out


def _static_worker(rank, world, port, q):
    import torch.distributed as dist

    try:
        _init(rank, world, port)
        from allegro_b200.halo import DistributedAllegro, SlabDecomposition

        model = _model()
        res = {}
        for name, pos, rows, vel in static_frames():
            types = torch.zeros(pos.shape[0], dtype=torch.long)
            dec = SlabDecomposition(pos, rows, types, R_MAX, rank, world)
            pos_owned = dec.local_positions_from_global(pos)[: dec.n_owned]
            r = DistributedAllegro(model, dec, stress=True, atomic_virial=True, heat_current=True).evaluate(pos_owned, vel[dec.owned])
            res[name] = {"owned": dec.owned.numpy().copy(), "diagonal": dec.geom.diagonal, **{k: _np(v) for k, v in r.items()}}
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def oracle(pos, rows, vel):
    """fp64 oracle on the whole periodic frame, exact r_max list: E, F, stress, virial, atomic energies, W and J"""
    import nlist_lattice_oracle as LO
    from test_halo_gloo_virial import _kwargs
    from test_host_atomic_virial import oracle_w_j

    from oracle.model_ref import AllegroOracle

    pr, _ = LO.pairs(pos.numpy(), rows.numpy(), (True, True, True), R_MAX)
    pr = torch.from_numpy(pr)
    d = {D.POSITIONS_KEY: pos, D.CELL_KEY: rows.double(), D.ATOM_TYPE_KEY: torch.zeros(pos.shape[0], dtype=torch.long),
         D.EDGE_INDEX_KEY: pr[:, :2].T.contiguous(), D.EDGE_CELL_SHIFT_KEY: pr[:, 2:].double()}
    orc = AllegroOracle(**_kwargs("c2"))
    ref = orc(d)
    W, J, _ = oracle_w_j(orc, d, vel)
    return ref, W, J


def _assemble(res, key, n):
    """the per-rank rows of one result put in global order: F, E_atom, W, and how often each atom was owned"""
    F, Ea, W = torch.zeros(n, 3, dtype=F64), torch.zeros(n, 1, dtype=F64), torch.zeros(n, 3, 3, dtype=F64)
    seen = torch.zeros(n, dtype=torch.long)
    for _, r in res:
        r = r[key]
        ids = torch.from_numpy(r["owned"] if "owned" in r else r["ids"]).long()
        seen[ids] += 1
        F[ids], Ea[ids], W[ids] = torch.from_numpy(r[D.FORCE_KEY]), torch.from_numpy(r[D.PER_ATOM_ENERGY_KEY]), torch.from_numpy(r[D.ATOMIC_VIRIAL_KEY])
    return F, Ea, W, seen


@pytest.mark.parametrize("world", [2, 3])
def test_static_decomposition_matches_oracle_on_triclinic_cells(world):
    res = _spawn(_static_worker, world)
    R = _rotation()
    got = {}
    for name, pos, rows, vel in static_frames():
        n = pos.shape[0]
        assert res[0][1][name]["diagonal"] == (name == "cubic"), name  # only the diagonal cell takes the orthorhombic path
        ref, W_ref, J_ref = oracle(pos, rows, vel)
        F, Ea, W, seen = _assemble(res, name, n)
        assert bool((seen == 1).all()), name  # every atom owned exactly once
        for _, r in res:
            r = r[name]
            assert _rel(r[D.TOTAL_ENERGY_KEY].reshape(-1), ref[D.TOTAL_ENERGY_KEY].reshape(-1)) < 1e-10, name
            assert _rel(r[D.VIRIAL_KEY], ref[D.VIRIAL_KEY]) < 1e-10 and _rel(r[D.STRESS_KEY], ref[D.STRESS_KEY]) < 1e-10, name
            assert _rel(r[D.HEAT_CURRENT_KEY][0], J_ref) < 1e-10, name
        assert _rel(F, ref[D.FORCE_KEY]) < 1e-10 and _rel(Ea, ref[D.PER_ATOM_ENERGY_KEY]) < 1e-10 and _rel(W, W_ref) < 1e-10, name
        got[name] = (res[0][1][name], F, W)
    # the same crystal in three bases (and a left-handed one): the same numbers to 1e-12
    base, F0, W0 = got["cubic"]
    for name in ("(a+b, b, c)", "(a, b+a, c)", "left-handed (a, c, b)"):
        r, F, W = got[name]
        assert _rel(r[D.TOTAL_ENERGY_KEY], base[D.TOTAL_ENERGY_KEY]) < 1e-12, name
        assert _rel(F, F0) < 1e-12 and _rel(W, W0) < 1e-12 and _rel(r[D.VIRIAL_KEY], base[D.VIRIAL_KEY]) < 1e-12, name
        assert _rel(r[D.HEAT_CURRENT_KEY], base[D.HEAT_CURRENT_KEY]) < 1e-12, name
    # the rotated frame: the same energy, forces and J rotated, W and the virial rotated on both sides
    r, F, W = got["rotated (a, b+a, c)"]
    assert _rel(r[D.TOTAL_ENERGY_KEY], base[D.TOTAL_ENERGY_KEY]) < 1e-12
    assert _rel(F, F0 @ R.T) < 1e-11 and _rel(W, R @ W0 @ R.T) < 1e-11
    assert _rel(torch.from_numpy(r[D.VIRIAL_KEY])[0], R @ torch.from_numpy(base[D.VIRIAL_KEY])[0] @ R.T) < 1e-11
    assert _rel(torch.from_numpy(r[D.HEAT_CURRENT_KEY])[0], R @ torch.from_numpy(base[D.HEAT_CURRENT_KEY])[0]) < 1e-11


# ---- molecular dynamics -----------------------------------------------------------------------------------------------
STEPS = 40


def md_case(kind):
    """(pos, rows, types, vel) of a trajectory: the sheared c2 frame of tests/test_halo_gloo_md.py in slanted-face rows
    (a, b+a, c) of a (5, 5, 3) supercell (H_0 / 2 = 6.4 > r_max + skin), or its (6, 3, 3) box rotated"""
    if kind == "slanted":
        pos, cell, types, vel = md_frame(reps=(5, 5, 3))
        A, B, C = cell
        return pos, torch.stack([A, B + A, C]), types, vel
    pos, cell, types, vel = md_frame()
    R = _rotation()
    return pos @ R.T, cell @ R.T, types, vel @ R.T


def _md_worker(rank, world, port, q, kind):
    import torch.distributed as dist

    from test_halo_gloo_md import run_trajectory

    try:
        _init(rank, world, port)
        from allegro_b200.halo import DistributedCalculator

        pos, rows, types, vel = md_case(kind)
        calc = DistributedCalculator(_model(), rows, R_MAX, SKIN, rank, world, device="cpu", transport="nccl", stress=True, heat_current=True)
        assert not calc.geom.diagonal
        steps = []

        def record(step, out, local):
            frame = calc.gather(local)
            steps.append({"ids": _np(local.ids), "frame": None if frame is None else {k: _np(v) for k, v in frame.items()},
                          **{k: _np(v) for k, v in out.items()}})

        run_trajectory(calc, pos, types, vel, STEPS, record)
        stats = dict(rebuilds=calc.n_rebuilds, redone=calc.n_redone, left=calc.n_sent_left, right=calc.n_sent_right)
        try:
            calc.compute(None, cell=rows * 1.01)
            stats["cell"] = "accepted"
        except ValueError as e:
            stats["cell"] = str(e)
        q.put((rank, steps, stats))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("kind,world", [("slanted", 2), ("rotated", 3)])
def test_md_trajectory_on_triclinic_cell_matches_oracle_at_every_step(kind, world):
    res = _spawn(_md_worker, world, kind)
    pos, rows, types, _ = md_case(kind)
    n = types.shape[0]
    st = [r[2] for r in res]
    assert all("fixed" in s["cell"] for s in st), st
    assert all(s["rebuilds"] == st[0]["rebuilds"] and s["redone"] == st[0]["redone"] for s in st)  # every rank rebuilt together
    assert st[0]["rebuilds"] >= 3 and st[0]["redone"] >= 2, st[0]
    assert sum(s["left"] for s in st) > 0 and sum(s["right"] for s in st) > 0, st  # migrations in both directions
    img0 = [res[0][1][s]["frame"]["image"][:, 0] for s in range(STEPS + 1)]
    assert any((img0[s] != img0[0]).any() for s in range(STEPS + 1))  # an atom crossed the periodic face of row 0
    for s in range(STEPS + 1):
        frame = res[0][1][s]["frame"]
        assert frame["ids"].tolist() == list(range(n))
        ref, W_ref, J_ref = oracle(torch.from_numpy(frame["pos"]), rows, torch.from_numpy(frame["velocities"]))
        F, Ea, W, seen = _assemble([(r[0], {"x": r[1][s]}) for r in res], "x", n)
        assert bool((seen == 1).all()), s  # every atom owned exactly once
        for _, steps, _ in res:
            r = steps[s]
            assert _rel(r[D.TOTAL_ENERGY_KEY].reshape(-1), ref[D.TOTAL_ENERGY_KEY].reshape(-1)) < 1e-10, s
            assert _rel(r[D.STRESS_KEY], ref[D.STRESS_KEY]) < 1e-10 and _rel(r[D.VIRIAL_KEY], ref[D.VIRIAL_KEY]) < 1e-10, s
            assert _rel(r[D.HEAT_CURRENT_KEY][0], J_ref) < 1e-10, s
        assert _rel(F, ref[D.FORCE_KEY]) < 1e-10 and _rel(Ea, ref[D.PER_ATOM_ENERGY_KEY]) < 1e-10 and _rel(W, W_ref) < 1e-10, s


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _refusal_worker(rank, world, port, q):
    import torch.distributed as dist

    try:
        _init(rank, world, port)
        from allegro_b200.halo import DistributedCalculator

        model = _model()
        pos, cell, types, vel = md_frame()
        A, B, C = cell
        got = {}
        cells = {"singular": torch.stack([A, B, A + B]), "near-coplanar": torch.stack([A, B, A + B + 1e-14 * C]),
                 # |h_0| / 3 = 7.2 >= r_max + skin, but H_0 / 3 = 3.2 is not
                 "thin": torch.stack([A, B + A, C])}
        for k, c in cells.items():
            try:
                DistributedCalculator(model, c, R_MAX, SKIN, rank, world, device="cpu", transport="nccl")
                got[k] = "accepted"
            except ValueError as e:
                got[k] = str(e)
        rows = md_case("rotated")[1]
        calc = DistributedCalculator(model, rows, R_MAX, SKIN, rank, world, device="cpu", transport="nccl")
        local = calc.distribute(*md_case("rotated")[:1], types, velocities=md_case("rotated")[3])
        calc.compute(local)
        if rank == 0:  # one atom two slabs further along s_0: the rebuild this triggers must refuse it on every rank
            local.pos[0] += (2.0 / world) * rows[0]
        try:
            calc.compute(local)
            got["far"] = "accepted"
        except ValueError as e:
            got["far"] = str(e)
        q.put((rank, got))
    finally:
        dist.destroy_process_group()


def test_lattice_refusals_raise_on_every_rank():
    res = _spawn(_refusal_worker, 3)
    for _, got in res:
        assert "not regular" in got["singular"] and "not regular" in got["near-coplanar"], got
        assert "H_0" in got["thin"] and "r_max + skin" in got["thin"], got["thin"]
        assert "time step or the skin" in got["far"], got["far"]
