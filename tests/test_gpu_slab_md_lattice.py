"""The slab decomposition on triclinic cells on the GPU: ab2_slab_plan_count_lattice against its torch restatement
(tests/test_halo_gloo_lattice.py) bit for bit, and against ab2_slab_plan_count on diagonal cells; ``DistributedCalculator``
molecular dynamics and the static ``DistributedAllegro`` / ``GraphedDistributedAllegro`` on a rotated triclinic frame,
over the peer-memory mailboxes (ab2_p2p_push_rows_v) and over NCCL, against single-GPU ``energy_and_forces`` of the same
frame and cell.

``test_lattice_ranks_sharing_a_device`` puts two ranks on one device (gloo for set-up and migration, CUDA IPC within the
device for the mailboxes), so the whole protocol runs on a one-GPU box; ``test_lattice_matches_single_gpu`` needs one
device per rank (world 2, 4, 8; skipped when fewer devices exist)."""
import os
import queue
import time

import pytest
import torch

from test_gpu_slab_md import R_MAX, SKIN, TOL, _free_port, _np, _reference, _rel
from test_halo_gloo_lattice import _rotation, plan_atoms, plan_cells, slab_faces_lattice_spec, slab_wrap_classify_lattice_spec
from test_halo_gloo_md import STEPS, md_frame, plan_cases, run_trajectory

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("cell", range(6))
def test_lattice_plan_kernel_matches_restatement(dtype, world, cell):
    from allegro_b200 import _lib

    cname, rows = plan_cells()[cell]
    dt = getattr(torch, dtype)
    for name, pos, jump in plan_atoms(rows, world):
        jump = {None: float("inf"), "slab": 1.0 / world}[jump]
        for rank in range(world):
            p_k, p_s = pos.to("cuda", dt), pos.to("cuda", dt)
            i_k = torch.full((p_k.shape[0], 3), 3, dtype=torch.int32, device="cuda")
            i_s = i_k.clone()
            got = _lib.slab_wrap_classify_lattice(p_k, i_k, rows, rank, world, jump)
            want = slab_wrap_classify_lattice_spec(p_s, i_s, rows, rank, world, jump)
            for a, b in zip(got[:3], want[:3]):
                assert a.dtype == torch.int64 and torch.equal(a, b), (cname, name, rank)
            assert got[3] == want[3], (cname, name, rank)
            assert torch.equal(p_k, p_s) and torch.equal(i_k, i_s), (cname, name, rank)
            for a, b in zip(_lib.slab_faces_lattice(p_k, rows, rank, world, R_MAX + SKIN),
                            slab_faces_lattice_spec(p_s, rows, rank, world, R_MAX + SKIN)):
                assert torch.equal(a, b), (cname, name, rank)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("world", [2, 3])
def test_lattice_plan_kernel_on_diagonal_cells_matches_orthorhombic(dtype, world):
    """random atoms in and around a diagonal box, away from the faces by more than rounding: the same lists"""
    from allegro_b200 import _lib

    dt = getattr(torch, dtype)
    for case in (0, 3):  # random, negative coordinates
        name, pos, box, _ = plan_cases()[case]
        rows = torch.diag(torch.tensor(box, dtype=torch.float64))
        width = box[0] / world
        for rank in range(world):
            p_o, p_l = pos.to("cuda", dt), pos.to("cuda", dt)
            i_o = torch.zeros(p_o.shape[0], 3, dtype=torch.int32, device="cuda")
            i_l = i_o.clone()
            got_o = _lib.slab_wrap_classify(p_o, i_o, box, rank, world, width, width)
            got_l = _lib.slab_wrap_classify_lattice(p_l, i_l, rows, rank, world, 1.0 / world)
            for a, b in zip(got_o[:3], got_l[:3]):
                assert torch.equal(a, b), (name, rank)
            assert got_o[3] == got_l[3] and torch.equal(i_o, i_l), (name, rank)
            assert torch.allclose(p_o.double(), p_l.double(), rtol=0, atol=1e-5 if dtype == "float32" else 1e-12), (name, rank)
            for a, b in zip(_lib.slab_faces(p_o, box, rank, world, width, R_MAX + SKIN), _lib.slab_faces_lattice(p_l, rows, rank, world, R_MAX + SKIN)):
                assert torch.equal(a, b), (name, rank)


def test_lattice_plan_kernel_refuses_singular_cells_before_launch():
    from allegro_b200 import _lib

    pos = torch.rand(10, 3, device="cuda", dtype=torch.float64)
    for rows in ([[5.0, 0, 0], [0, 5.0, 0], [5.0, 5.0, 0]], [[5.0, 0, 0], [0, 5.0, 0], [5.0, 5.0, 1e-14]], [[5.0, 0, 0], [0, float("nan"), 0], [0, 0, 5.0]]):
        for p in (pos, pos[:0]):
            with pytest.raises(RuntimeError, match="cell"):
                _lib.slab_wrap_classify_lattice(p.clone(), torch.zeros(p.shape[0], 3, dtype=torch.int32, device="cuda"), rows, 0, 2)


# ---- distributed runs on a triclinic frame ----------------------------------------------------------------------------
def _reps(world):
    return (max(8, 4 * world), 5, 5)


def _frame(world, dtype):
    """the sheared c2 frame of tests/test_gpu_slab_md.py in rows (a, b + 2 a0, c) (a0 the cubic lattice constant along x:
    the same crystal, slanted faces, H_0 = 0.93 |a|), rotated so that no row is axis-aligned"""
    pos, cell, types, vel = md_frame(_reps(world), torch.float64, seed=3, world=world, spread=0.02)
    A, B, C = cell
    a0 = A / _reps(world)[0]
    R = _rotation()
    rows = torch.stack([A, B + 2 * a0, C]) @ R.T
    dt = getattr(torch, dtype)
    return (pos @ R.T).to(dt), rows.to(dt), types, (vel @ R.T).to(dt)


def _md(rank, world, dev, dtype, transport, model):
    """a trajectory; at every step the graph's outputs, those of the same step run eagerly, and the gathered frame"""
    from allegro_b200.halo import DistributedCalculator

    pos, cell, types, vel = _frame(world, dtype)
    calc = DistributedCalculator(model, cell, R_MAX, SKIN, rank, world, device=dev, transport=transport, stress=True, heat_current=True)
    assert not calc.geom.diagonal
    steps, diff = [], [0.0]

    def record(step, out, local):
        graphed = {k: v.clone() for k, v in out.items()}
        with torch.no_grad():  # the same step, eagerly (collective): between rebuilds a replay must give what it gives
            eager = calc._step(local.pos, local.arrays["velocities"])
        torch.cuda.synchronize()
        assert float(eager["extra"][0]) == 0.0
        diff[0] = max(diff[0], max(_rel(graphed[k], eager[k]) for k in graphed))
        frame = calc.gather(local)
        steps.append({"ids": _np(local.ids), "frame": None if frame is None else {k: _np(v) for k, v in frame.items()},
                      **{k: _np(v) for k, v in graphed.items()}})

    run_trajectory(calc, pos.to(dev), types.to(dev), vel.to(dev), STEPS, record)
    stats = dict(rebuilds=calc.n_rebuilds, redone=calc.n_redone, left=calc.n_sent_left, right=calc.n_sent_right, diff=diff[0],
                 graphed=calc._graphed is not None)
    if calc.p2p is not None:
        stats["err"], stats["grown"] = calc.p2p.error(), calc.p2p.n_grown
    calc.close()
    return steps, stats


def _static(rank, world, dev, dtype, transport, model):
    """eager evaluate of the first frame and 4 graph replays of it -> (owned ids, eager outputs, max |graph - eager|, error word)"""
    from allegro_b200.halo import DistributedAllegro, GraphedDistributedAllegro, P2PHalo, SlabDecomposition

    pos, cell, types, vel = _frame(world, dtype)
    dec = SlabDecomposition(pos, cell, types, R_MAX, rank, world, device=dev if transport == "p2p" else None)
    assert not dec.geom.diagonal
    pos_owned = dec.local_positions_from_global(pos)[: dec.n_owned].to(dev)
    vel_owned = vel[dec.owned].to(dev)
    dec.to(dev)
    p2p = P2PHalo(dec, dev, atomic_virial=True) if transport == "p2p" else None
    runner = DistributedAllegro(model, dec, p2p=p2p, stress=True, atomic_virial=True, heat_current=True)
    eager = {k: v.clone() for k, v in runner.evaluate(pos_owned, vel_owned).items()}
    graphed = GraphedDistributedAllegro(runner, pos_owned + 0.01, velocities=0.5 * vel_owned)
    diff = 0.0
    for _ in range(4):
        out = graphed(pos_owned, vel_owned)
        torch.cuda.synchronize()
        diff = max(diff, max(_rel(out[k], eager[k]) for k in eager))
    err = p2p.error() if p2p is not None else 0
    del graphed
    if p2p is not None:
        p2p.close()
    return dec.owned.cpu().numpy(), {k: _np(v) for k, v in eager.items()}, diff, err


def _worker(rank, world, port, q, shared):
    import torch.distributed as dist

    from allegro_b200 import halo, systems
    from allegro_b200.model import AllegroModel

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", 0 if shared else rank)
    torch.cuda.set_device(dev)
    if shared:  # NCCL refuses two ranks on one device; the P2P step makes no collective call
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        halo.MAILBOX_HEADROOM = 1.0  # every rebuild that needs more rows than the mailbox holds re-allocates it
        res = {}
        for dtype in ("float64", "float32"):
            model = AllegroModel(**systems.model_kwargs("c2", 42.0, dtype)).to(dev).model
            for transport in (("p2p",) if shared else ("nccl", "p2p")):
                res[("static", dtype, transport)] = _static(rank, world, dev, dtype, transport, model)
                res[("md", dtype, transport)] = _md(rank, world, dev, dtype, transport, model)
        q.put((rank, res))
        dist.barrier()
        torch.cuda.synchronize()
        q.close()
        q.join_thread()
        # live graphs with captured NCCL kernels block communicator teardown: leave without the destructors
        os._exit(0)
    except BaseException:
        dist.destroy_process_group()
        raise


def _collect(world, shared):
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, shared)) for r in range(world)]
    for p in procs:
        p.start()
    res, deadline = [], time.time() + 1200
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


def _gathered(outs, n):
    """per-rank (ids, outputs) -> F, E_atom, W in global order and how often each atom was owned"""
    from allegro_b200 import data as D

    F, Ea, W = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 1, dtype=torch.float64), torch.zeros(n, 3, 3, dtype=torch.float64)
    seen = torch.zeros(n, dtype=torch.long)
    for ids, r in outs:
        ids = torch.from_numpy(ids).long()
        seen[ids] += 1
        F[ids], Ea[ids], W[ids] = torch.from_numpy(r[D.FORCE_KEY]), torch.from_numpy(r[D.PER_ATOM_ENERGY_KEY]), torch.from_numpy(r[D.ATOMIC_VIRIAL_KEY])
    return F, Ea, W, seen


def _check_totals(outs, ref, tol, what):
    from allegro_b200 import data as D

    for _, r in outs:
        for k in (D.TOTAL_ENERGY_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.HEAT_CURRENT_KEY):
            got = torch.from_numpy(r[k]).reshape(ref[k].shape)
            assert _rel(got, ref[k]) < tol, (what, k, _rel(got, ref[k]))
    F, Ea, W, seen = _gathered(outs, ref[D.FORCE_KEY].shape[0])
    assert bool((seen == 1).all()), what  # every atom owned exactly once
    for k, v in ((D.FORCE_KEY, F), (D.PER_ATOM_ENERGY_KEY, Ea), (D.ATOMIC_VIRIAL_KEY, W)):
        assert _rel(v, ref[k]) < tol, (what, k, _rel(v, ref[k]))


def _check(res, transports):
    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel

    world = len(res)
    for dtype in ("float64", "float32"):
        model = AllegroModel(**systems.model_kwargs("c2", 42.0, dtype)).to("cuda:0").model
        pos, cell, types, vel = _frame(world, dtype)
        tol = TOL[dtype]
        for transport in transports:
            # static runner on the first frame, eager and graph-replayed
            st = [r[("static", dtype, transport)] for _, r in res]
            assert all(s[3] == 0 for s in st) and max(s[2] for s in st) <= tol, (dtype, transport, [s[2:] for s in st])
            frame = {"pos": pos.double().numpy(), "types": types.numpy(), "velocities": vel.double().numpy()}
            _check_totals([(s[0], s[1]) for s in st], _reference(model, frame, cell, dtype), tol, (dtype, transport, "static"))
            # the trajectory
            runs = [r[("md", dtype, transport)] for _, r in res]
            stats = [s for _, s in runs]
            assert all(s["rebuilds"] == stats[0]["rebuilds"] and s["redone"] == stats[0]["redone"] for s in stats)
            assert stats[0]["rebuilds"] >= 3 and stats[0]["redone"] >= 2, stats[0]
            assert sum(s["left"] for s in stats) > 0 and sum(s["right"] for s in stats) > 0, stats
            assert all(s["graphed"] for s in stats)
            assert max(s["diff"] for s in stats) <= tol, (dtype, transport, [s["diff"] for s in stats])  # graph replay == eager step
            if transport == "p2p":
                assert all(s["err"] == 0 for s in stats), stats
                assert sum(s["grown"] for s in stats) >= 1, stats  # a rebuild re-allocated the mailbox
            x0 = runs[0][0][0]["frame"]["image"][:, 0]
            assert any((runs[0][0][s]["frame"]["image"][:, 0] != x0).any() for s in range(STEPS + 1))  # crossed the face of row 0
            for s in range(STEPS + 1):
                ref = _reference(model, runs[0][0][s]["frame"], cell, dtype)
                _check_totals([(steps[s]["ids"], steps[s]) for steps, _ in runs], ref, tol, (dtype, transport, s))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_lattice_matches_single_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _check(_collect(world, shared=False), ("nccl", "p2p"))


def test_lattice_ranks_sharing_a_device():
    _check(_collect(2, shared=True), ("p2p",))
