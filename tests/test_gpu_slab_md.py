"""``DistributedCalculator`` on the GPU: the slab-plan kernels (ab2_slab_plan_count / fill) against their torch
restatement, and molecular dynamics over the peer-memory mailboxes and over NCCL, checked at every step against the
single-GPU ``energy_and_forces`` of the gathered frame on an exact r_max list.

``test_md_ranks_sharing_a_device`` puts two ranks on one device (gloo for set-up and migration, CUDA IPC within the
device for the mailboxes), so the whole protocol runs on a one-GPU box; ``test_md_matches_single_gpu`` needs one device
per rank (world 2, 4, 8; skipped when fewer devices exist)."""
import os
import queue
import time

import pytest
import torch

from test_halo_gloo_md import STEPS, md_frame, plan_cases, run_trajectory, slab_faces_spec, slab_wrap_classify_spec

pytestmark = pytest.mark.gpu

TOL = {"float64": 1e-9, "float32": 1e-4}
R_MAX, SKIN = 5.0, 0.5


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", range(6))
def test_plan_kernel_matches_restatement(dtype, world, case):
    from allegro_b200 import _lib

    name, pos, box, jump = plan_cases()[case]
    width = box[0] / world
    jump = {None: float("inf"), "width": width}[jump]
    dt = getattr(torch, dtype)
    for rank in range(world):
        p_k, p_s = pos.to("cuda", dt), pos.to("cuda", dt)
        i_k = torch.full((p_k.shape[0], 3), 3, dtype=torch.int32, device="cuda")
        i_s = i_k.clone()
        got = _lib.slab_wrap_classify(p_k, i_k, box, rank, world, width, jump)
        want = slab_wrap_classify_spec(p_s, i_s, box, rank, world, width, jump)
        for a, b in zip(got[:3], want[:3]):
            assert a.dtype == torch.int64 and torch.equal(a, b), (name, rank)
        assert got[3] == want[3], (name, rank)
        assert torch.equal(p_k, p_s) and torch.equal(i_k, i_s), (name, rank)
        for a, b in zip(_lib.slab_faces(p_k, box, rank, world, width, R_MAX + SKIN), slab_faces_spec(p_s, box, rank, world, width, R_MAX + SKIN)):
            assert torch.equal(a, b), (name, rank)


def _free_port():
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _reps(world):
    return (max(8, 4 * world), 5, 5)


def _frame(world, dtype):
    return md_frame(_reps(world), getattr(torch, dtype), seed=3, world=world, spread=0.02)


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _np(t):
    return t.detach().double().cpu().numpy().copy()


def _run(rank, world, dev, dtype, transport, model):
    """a trajectory; at every step the graph's outputs, those of the same step run eagerly, and the gathered frame"""
    from allegro_b200.halo import DistributedCalculator

    pos, cell, types, vel = _frame(world, dtype)
    calc = DistributedCalculator(model, cell, R_MAX, SKIN, rank, world, device=dev, transport=transport, stress=True, heat_current=True)
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
                res[(dtype, transport)] = _run(rank, world, dev, dtype, transport, model)
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


def _reference(model, frame, cell, dtype):
    from allegro_b200 import data as D

    dt = getattr(torch, dtype)
    pos = torch.from_numpy(frame["pos"]).to("cuda:0", dt)
    c = cell.to("cuda:0", dt)
    csr, shift = D.neighbor_csr(pos, R_MAX, c, (True, True, True))
    d = {D.POSITIONS_KEY: pos, D.CELL_KEY: c, D.ATOM_TYPE_KEY: torch.from_numpy(frame["types"]).to("cuda:0", torch.long),
         D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: shift, D.VELOCITY_KEY: torch.from_numpy(frame["velocities"]).to("cuda:0", dt)}
    out = model.energy_and_forces(d, stress=True, atomic_virial=True, heat_current=True)
    return {k: out[k].double().cpu() for k in (D.TOTAL_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.STRESS_KEY, D.VIRIAL_KEY,
                                                D.ATOMIC_VIRIAL_KEY, D.HEAT_CURRENT_KEY)}


def _check(res, transports):
    from allegro_b200 import data as D
    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel

    world = len(res)
    for dtype in ("float64", "float32"):
        model = AllegroModel(**systems.model_kwargs("c2", 42.0, dtype)).to("cuda:0").model
        _, cell, _, _ = _frame(world, dtype)
        tol = TOL[dtype]
        for transport in transports:
            runs = [r[(dtype, transport)] for _, r in res]
            st = [s for _, s in runs]
            assert all(s["rebuilds"] == st[0]["rebuilds"] and s["redone"] == st[0]["redone"] for s in st)
            assert st[0]["rebuilds"] >= 3 and st[0]["redone"] >= 2, st[0]
            assert sum(s["left"] for s in st) > 0 and sum(s["right"] for s in st) > 0, st
            assert all(s["graphed"] for s in st)
            assert max(s["diff"] for s in st) <= tol, (dtype, transport, [s["diff"] for s in st])  # graph replay == eager step
            if transport == "p2p":
                assert all(s["err"] == 0 for s in st), st
                assert sum(s["grown"] for s in st) >= 1, st  # a rebuild re-allocated the mailbox
            x0 = runs[0][0][0]["frame"]["image"][:, 0]
            assert any((runs[0][0][s]["frame"]["image"][:, 0] != x0).any() for s in range(STEPS + 1))  # periodic x crossing
            for s in range(STEPS + 1):
                frame = runs[0][0][s]["frame"]
                ref = _reference(model, frame, cell, dtype)
                n = ref[D.FORCE_KEY].shape[0]
                F, Ea, W = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 1, dtype=torch.float64), torch.zeros(n, 3, 3, dtype=torch.float64)
                seen = torch.zeros(n, dtype=torch.long)
                for steps, _ in runs:
                    r = steps[s]
                    ids = torch.from_numpy(r["ids"]).long()
                    seen[ids] += 1
                    F[ids], Ea[ids] = torch.from_numpy(r[D.FORCE_KEY]), torch.from_numpy(r[D.PER_ATOM_ENERGY_KEY])
                    W[ids] = torch.from_numpy(r[D.ATOMIC_VIRIAL_KEY])
                    for k in (D.TOTAL_ENERGY_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.HEAT_CURRENT_KEY):
                        got = torch.from_numpy(r[k]).reshape(ref[k].shape)
                        assert _rel(got, ref[k]) < tol, (dtype, transport, s, k, _rel(got, ref[k]))
                assert bool((seen == 1).all()), (dtype, transport, s)
                for k, v in ((D.FORCE_KEY, F), (D.PER_ATOM_ENERGY_KEY, Ea), (D.ATOMIC_VIRIAL_KEY, W)):
                    assert _rel(v, ref[k]) < tol, (dtype, transport, s, k, _rel(v, ref[k]))


@pytest.mark.parametrize("world", [2, 4, 8])
def test_md_matches_single_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _check(_collect(world, shared=False), ("nccl", "p2p"))


def test_md_ranks_sharing_a_device():
    _check(_collect(2, shared=True), ("p2p",))
