"""world_size-2/3 gloo tests (CPU) of ``DistributedCalculator``: molecular dynamics on a slab decomposition that migrates
atoms and rebuilds its halo as they move.

Each rank runs the package's fused model on the CPU (``_energy_and_forces`` with the spec kernels, as in
tests/test_halo_gloo_virial.py) and the torch restatement of ab2_slab_plan below, so what is checked here is the host
protocol: the rebuild check riding the vector reduction, redone steps, wrap / migration / ghost selection, the
re-partition of ``LocalAtoms`` and ``gather``.  At every step of a velocity-Verlet trajectory whose atoms cross slab
faces in both directions and the periodic x boundary, the gathered frame is evaluated by the fp64 oracle on an exact
r_max list.  The kernels and the peer-memory transport are checked on the GPU (tests/test_gpu_slab_md.py)."""
import math
import os
import queue
import time

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from allegro_b200 import data as D
from allegro_b200 import systems

R_MAX, SKIN, STEPS, DT, MASS = 5.0, 0.5, 40, 1.0, 1000.0


# ---- torch restatement of ab2_slab_plan (csrc/slab_md.cu) ---------------------------------------------------------------
def _nz(m):
    return torch.nonzero(m).reshape(-1)


def slab_wrap_classify_spec(pos, image, box, rank, world, width, jump=float("inf")):
    """mode 0: wrap in place (x - floor(x / L) L, one correction either way, in the positions' dtype), image += boxes
    removed, classify by clamp(floor(x / width), 0, world - 1)"""
    dt = pos.dtype
    xd = pos[:, 0].double().clone()
    for a in range(3):
        L = torch.tensor(box[a], dtype=dt, device=pos.device)
        x = pos[:, a]
        img = torch.floor(x / L)
        w = x - img * L
        neg = w < 0
        w, img = torch.where(neg, w + L, w), torch.where(neg, img - 1, img)
        big = w >= L
        w, img = torch.where(big, w - L, w), torch.where(big, img + 1, img)
        pos[:, a] = w
        image[:, a] += img.to(torch.int32)
    lo, hi = rank * width, (rank + 1) * width
    s = (pos[:, 0] / torch.tensor(width, dtype=dt, device=pos.device)).long().clamp(0, world - 1)
    d = (s - rank) % world
    far = (xd < lo - jump) | (xd >= hi + jump)
    move = ~far & (d != 0)
    if world == 2:
        left, right = move & (xd < lo), move & ~(xd < lo)
    else:
        left, right = move & (d == world - 1), move & (d == 1)
        far = far | (move & ~left & ~right)
    return _nz(~far & (d == 0)), _nz(left), _nz(right), int(far.sum())


def slab_faces_spec(pos, box, rank, world, width, r_list):
    """mode 1: atoms within r_list of the low face and of the high face, compared in fp64"""
    x = pos[:, 0].double()
    lo, hi = rank * width, (rank + 1) * width
    return _nz(x < lo + r_list), _nz(x >= hi - r_list)


def _brute_plan(pos, box, rank, world, width, jump=float("inf")):
    """one atom at a time in Python floats (fp64 frames): the same rules, lists built by appending in atom order"""
    stay, left, right, far, wrapped, images = [], [], [], 0, [], []
    lo, hi = rank * width, (rank + 1) * width
    for i, p in enumerate(pos.tolist()):
        w3, im3 = [], []
        for a in range(3):
            L = box[a]
            img = math.floor(p[a] / L)
            w = p[a] - img * L
            if w < 0:
                w, img = w + L, img - 1
            if w >= L:
                w, img = w - L, img + 1
            w3.append(w)
            im3.append(img)
        wrapped.append(w3)
        images.append(im3)
        x = p[0]
        s = min(max(int(w3[0] / width), 0), world - 1)
        d = (s - rank) % world
        if x < lo - jump or x >= hi + jump:
            far += 1
        elif d == 0:
            stay.append(i)
        elif world == 2:
            (left if x < lo else right).append(i)
        elif d == world - 1:
            left.append(i)
        elif d == 1:
            right.append(i)
        else:
            far += 1
    return stay, left, right, far, wrapped, images


def plan_cases():
    """(name, fp64 positions, box, jump): faces, x == Lx after the wrap, negative x, everyone emigrating, empty"""
    box = [21.69, 10.845, 10.845]
    g = torch.Generator().manual_seed(5)
    rnd = (torch.rand(200, 3, generator=g, dtype=torch.float64) * 1.4 - 0.2) * torch.tensor(box, dtype=torch.float64)
    faces = torch.tensor([[k * box[0] / 3, 1.0, 2.0] for k in range(4)] + [[k * box[0] / 2, -0.0, box[2]] for k in range(3)], dtype=torch.float64)
    at_l = torch.tensor([[-1e-17, 3.0, 3.0], [box[0] * (1 - 1e-17), 1.0, -1e-18], [box[0], box[1], 0.0], [-2 * box[0], -box[1], 3 * box[2]]],
                        dtype=torch.float64)
    neg = -torch.rand(20, 3, generator=g, dtype=torch.float64) * 15.0
    emig = torch.cat([box[0] / 2 + torch.rand(30, 1, generator=g, dtype=torch.float64) * box[0] / 7, torch.rand(30, 2, generator=g, dtype=torch.float64)], 1)
    return [("random", rnd, box, None), ("faces", faces, box, None), ("x == Lx after the wrap", at_l, box, None), ("negative x", neg, box, None),
            ("all emigrate", emig, box, "width"), ("empty", torch.zeros(0, 3, dtype=torch.float64), box, None)]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", range(6))
def test_plan_restatement_matches_brute_force(world, case):
    name, pos, box, jump = plan_cases()[case]
    width = box[0] / world
    jump = {None: float("inf"), "width": width}[jump]
    for rank in range(world):
        p = pos.clone()
        image = torch.zeros(p.shape[0], 3, dtype=torch.int32)
        stay, left, right, far = slab_wrap_classify_spec(p, image, box, rank, world, width, jump)
        b_stay, b_left, b_right, b_far, b_w, b_img = _brute_plan(pos, box, rank, world, width, jump)
        assert stay.tolist() == b_stay and left.tolist() == b_left and right.tolist() == b_right and far == b_far, (name, rank)
        assert p.tolist() == b_w and image.tolist() == b_img, name
        assert bool(((p >= 0) & (p < torch.tensor(box, dtype=torch.float64))).all()), name
        assert torch.allclose(p + image.double() * torch.tensor(box, dtype=torch.float64), pos, rtol=0, atol=1e-12), name
        low, high = slab_faces_spec(p, box, rank, world, width, 5.5)
        x = p[:, 0].tolist()
        assert low.tolist() == [i for i in range(len(x)) if x[i] < rank * width + 5.5], name
        assert high.tolist() == [i for i in range(len(x)) if x[i] >= (rank + 1) * width - 5.5], name
    if name == "all emigrate":
        assert len(_brute_plan(pos, box, 0, world, width, jump)[0]) == 0
    if name == "empty":
        assert all(len(v) == 0 for v in slab_wrap_classify_spec(pos.clone(), torch.zeros(0, 3, dtype=torch.int32), box, 0, world, width)[:3])


# ---- the distributed runs ---------------------------------------------------------------------------------------------
def _install():
    from test_halo_gloo_virial import _install_spec_kernels

    from allegro_b200 import _lib

    _install_spec_kernels()
    _lib.slab_wrap_classify = slab_wrap_classify_spec
    _lib.slab_faces = slab_faces_spec


def _model(kw):
    from test_halo_gloo_virial import _CpuFused
    from test_host_frames import _models

    from oracle.model_ref import AllegroOracle

    return _CpuFused(_models(kw, AllegroOracle(**kw).state_dict())[1])


def md_frame(reps=(6, 3, 3), dtype=torch.float64, seed=7, world=1, spread=0.0):
    """displaced c2 frame with a shear flow: v_x ~ sin(2 pi y / Ly) plus thermal noise, so atoms cross slab faces in both
    directions and the periodic x boundary within a few tens of steps.  ``spread`` adds v_x = -spread sin(2 pi x world /
    Lx), which carries atoms from the middle of each of ``world`` slabs towards its faces (the ghost lists grow)."""
    pos, cell, types = systems.make_positions("c2", reps)
    g = torch.Generator().manual_seed(seed)
    pos = pos + 0.1 * torch.randn(pos.shape, generator=g, dtype=pos.dtype)
    Ly = float(cell.view(3, 3)[1, 1])
    vel = 0.01 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
    vel[:, 0] += 0.05 * torch.sin(2 * math.pi * pos[:, 1] / Ly)
    vel[:, 0] -= spread * torch.sin(2 * math.pi * pos[:, 0] * world / float(cell.view(3, 3)[0, 0]))
    return pos.to(dtype), cell.to(dtype), types, vel.to(dtype)


def run_trajectory(calc, pos, types, vel, steps, record):
    """velocity Verlet; ``record(step, out, local)`` after every force evaluation, before the second half-kick"""
    m = torch.full((pos.shape[0],), MASS, dtype=pos.dtype)
    local = calc.distribute(pos, types, velocities=vel, masses=m)
    out = calc.compute(local)
    record(0, out, local)
    for step in range(1, steps + 1):
        local.arrays[D.VELOCITY_KEY] += 0.5 * DT * out[D.FORCE_KEY] / local.arrays["masses"][:, None]
        local.pos += DT * local.arrays[D.VELOCITY_KEY]
        out = calc.compute(local)  # may re-partition: read everything from `local` again
        record(step, out, local)
        local.arrays[D.VELOCITY_KEY] += 0.5 * DT * out[D.FORCE_KEY] / local.arrays["masses"][:, None]
    return local


def _np(t):
    return t.detach().double().cpu().numpy().copy()


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        _install()
        from test_halo_gloo_virial import _kwargs

        from allegro_b200.halo import DistributedCalculator

        model = _model(_kwargs("c2"))
        pos, cell, types, vel = md_frame()
        calc = DistributedCalculator(model, cell, R_MAX, SKIN, rank, world, device="cpu", transport="nccl", stress=True, heat_current=True)
        steps = []

        def record(step, out, local):
            frame = calc.gather(local)
            steps.append({"ids": _np(local.ids), "frame": None if frame is None else {k: _np(v) for k, v in frame.items()},
                          **{k: _np(v) for k, v in out.items()}})

        run_trajectory(calc, pos, types, vel, STEPS, record)
        stats = dict(rebuilds=calc.n_rebuilds, redone=calc.n_redone, left=calc.n_sent_left, right=calc.n_sent_right)
        # refusals: a cell other than the calculator's, before any exchange
        try:
            calc.compute(None, cell=cell * 1.01)
            stats["cell"] = "accepted"
        except ValueError as e:
            stats["cell"] = str(e)
        q.put((rank, steps, stats))
    finally:
        dist.destroy_process_group()


def _refusal_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        _install()
        from test_halo_gloo_virial import _kwargs

        from allegro_b200.halo import DistributedCalculator

        model = _model(_kwargs("c2"))
        pos, cell, types, vel = md_frame()
        got = {}
        try:  # slabs thinner than r_max + skin
            DistributedCalculator(model, cell, R_MAX, 2.5, rank, world, device="cpu", transport="nccl")
            got["thin"] = "accepted"
        except ValueError as e:
            got["thin"] = str(e)
        calc = DistributedCalculator(model, cell, R_MAX, SKIN, rank, world, device="cpu", transport="nccl")
        local = calc.distribute(pos, types, velocities=vel)
        calc.compute(local)
        if rank == 0:  # one atom two slabs to the right: the rebuild this triggers must refuse it on every rank
            local.pos[0, 0] += 2 * calc.width
        try:
            calc.compute(local)
            got["far"] = "accepted"
        except ValueError as e:
            got["far"] = str(e)
        q.put((rank, got))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, *args):
    from test_halo_gloo_virial import _free_port

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    res, deadline = [], time.time() + 900
    try:
        while len(res) < world:  # fail fast when a worker dies instead of waiting out the deadline
            try:
                res.append(q.get(timeout=2))
            except queue.Empty:
                dead = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
                assert not dead, f"worker exited with {dead}"
                assert time.time() < deadline, "timed out waiting for the workers"
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    return sorted(res, key=lambda r: r[0])


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def oracle_frame(frame, cell, types):
    """fp64 oracle on the gathered frame, exact r_max list: E, F, stress, virial, atomic energies, W and J"""
    from test_halo_gloo_virial import _kwargs
    from test_host_atomic_virial import oracle_w_j

    from oracle.model_ref import AllegroOracle

    pos = torch.from_numpy(frame["pos"])
    ei, sh = D.neighbor_list(pos, R_MAX, cell, (True, True, True))
    d = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell.double(), D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh}
    oracle = AllegroOracle(**_kwargs("c2"))
    ref = oracle(d)
    W, J, _ = oracle_w_j(oracle, d, torch.from_numpy(frame["velocities"]))
    return ref, W, J


@pytest.mark.parametrize("world", [2, 3])
def test_md_trajectory_matches_oracle_at_every_step(world):
    res = _spawn(_worker, world)
    _, cell, types, _ = md_frame()
    n = types.shape[0]
    for _, _, st in res:
        assert "fixed" in st["cell"], st["cell"]
    stats = {k: sum(r[2][k] for r in res) for k in ("left", "right")}
    rebuilds, redone = res[0][2]["rebuilds"], res[0][2]["redone"]
    assert all(r[2]["rebuilds"] == rebuilds and r[2]["redone"] == redone for r in res)  # every rank rebuilt together
    assert rebuilds >= 3 and redone >= 2, (rebuilds, redone)
    assert stats["left"] > 0 and stats["right"] > 0, stats  # migrations in both directions
    x_images = [torch.from_numpy(res[0][1][s]["frame"]["image"][:, 0]) for s in range(STEPS + 1)]
    assert any(bool((x_images[s] != x_images[0]).any()) for s in range(STEPS + 1))  # an atom crossed the periodic x boundary
    for s in range(STEPS + 1):
        frame = res[0][1][s]["frame"]
        assert frame["ids"].tolist() == list(range(n))
        ref, W_ref, J_ref = oracle_frame(frame, cell, types)
        F, Ea, W = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 1, dtype=torch.float64), torch.zeros(n, 3, 3, dtype=torch.float64)
        seen = torch.zeros(n, dtype=torch.long)
        for _, steps, _ in res:
            r = steps[s]
            ids = torch.from_numpy(r["ids"]).long()
            seen[ids] += 1
            F[ids], Ea[ids], W[ids] = torch.from_numpy(r[D.FORCE_KEY]), torch.from_numpy(r[D.PER_ATOM_ENERGY_KEY]), torch.from_numpy(r[D.ATOMIC_VIRIAL_KEY])
            assert _rel(r[D.TOTAL_ENERGY_KEY].reshape(-1), ref[D.TOTAL_ENERGY_KEY].reshape(-1)) < 1e-10, s
            assert _rel(r[D.STRESS_KEY], ref[D.STRESS_KEY]) < 1e-10 and _rel(r[D.VIRIAL_KEY], ref[D.VIRIAL_KEY]) < 1e-10, s
            assert _rel(r[D.HEAT_CURRENT_KEY][0], J_ref) < 1e-10, s
        assert bool((seen == 1).all()), s  # every atom owned exactly once
        assert _rel(F, ref[D.FORCE_KEY]) < 1e-10, s
        assert _rel(Ea, ref[D.PER_ATOM_ENERGY_KEY]) < 1e-10, s
        assert _rel(W, W_ref) < 1e-10, s


def test_md_refusals_raise_on_every_rank():
    res = _spawn(_refusal_worker, 3)
    for _, got in res:
        assert "r_max + skin" in got["thin"], got["thin"]
        assert "time step or the skin" in got["far"], got["far"]
