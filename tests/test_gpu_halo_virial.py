"""Stress, per-atom virial and heat current of the slab decomposition on the GPU: ``DistributedAllegro.evaluate`` with
the CUDA model on every rank == the single-GPU ``energy_and_forces(stress, atomic_virial, heat_current)`` of the whole
periodic frame, eager and replayed from a CUDA graph, over NCCL and over the peer-memory mailboxes (P2PHalo with the
extended layout: width-12 reverse rows and the vector all-reduce).

``test_virial_halo_matches_single_gpu`` needs one device per rank (skipped below 2 devices; world 4 and 8 run when
that many exist).  ``test_p2p_virial_ranks_sharing_a_device`` puts two ranks on one device (gloo for set-up, CUDA IPC
within the device for the mailboxes), so the new kernels also run on a one-GPU box."""
import os
import queue
import socket
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {"float64": 1e-9, "float32": 1e-4}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _reps(world):
    return (max(8, 4 * world), 5, 5)


def _frame(world):
    from allegro_b200 import systems

    pos, cell, types = systems.make_positions("c2", _reps(world))
    g = torch.Generator().manual_seed(3)
    pos = pos + 0.05 * torch.randn(pos.shape, generator=g, dtype=pos.dtype)
    vel = torch.randn(pos.shape, generator=g, dtype=torch.float64)
    return pos, cell, types, vel


def _np(d):
    return {k: v.detach().double().cpu().numpy().copy() for k, v in d.items()}


def _run(rank, world, dev, dtype, transport, model, pos, cell, types, vel):
    """eager evaluate + 6 graph replays (both mailbox parities) -> (eager dict, max |graph - eager|, p2p error word)"""
    from allegro_b200.halo import DistributedAllegro, GraphedDistributedAllegro, P2PHalo, SlabDecomposition

    p2p_mode = transport == "p2p"
    dec = SlabDecomposition(pos, cell, types, 5.0, rank, world, device=dev if p2p_mode else None)
    pos_owned = dec.local_positions_from_global(pos)[: dec.n_owned].to(dev, getattr(torch, dtype))
    vel_owned = vel[dec.owned].to(dev, getattr(torch, dtype))
    dec.to(dev)
    p2p = P2PHalo(dec, dev, atomic_virial=True) if p2p_mode else None
    runner = DistributedAllegro(model, dec, p2p=p2p, stress=True, atomic_virial=True, heat_current=True)
    eager = {k: v.clone() for k, v in runner.evaluate(pos_owned, vel_owned).items()}
    # captured on other inputs, replayed on these: the static buffers are refilled on every call
    graphed = GraphedDistributedAllegro(runner, pos_owned + 0.01, velocities=0.5 * vel_owned)
    diff = 0.0
    for _ in range(6):
        out = graphed(pos_owned, vel_owned)
        torch.cuda.synchronize()
        # relative: the model's own backward accumulates some fp64 sums with atomics, so a step is repeatable to rounding
        diff = max(diff, max(_rel(out[k], eager[k]) for k in eager))
    if p2p is not None:
        diff = (diff, _halo_replay_diff(p2p, dec, dev, getattr(torch, dtype)))
    err = p2p.error() if p2p is not None else 0
    return dec.owned.cpu().numpy(), _np(eager), diff, err


def _halo_replay_diff(p2p, dec, dev, dt):
    """The halo alone on fixed rows (forward, width-12 reverse, 13-value all-reduce): graph replays must give the eager
    bits -- fixed accumulation order, rank-ordered sums.  -> number of replays that differed."""
    g0 = torch.Generator().manual_seed(dec.rank)
    nl, n = dec.n_owned + dec.n_ghost, dec.n_owned
    g = torch.randn(nl, 3, generator=g0).to(dev, dt)
    W = torch.randn(nl, 3, 3, generator=g0).to(dev, dt)
    v = torch.randn(13, generator=g0, dtype=torch.float64).to(dev)
    pos = torch.randn(n, 3, generator=g0).to(dev, dt)

    def step():
        go, Wo = g[:n].clone(), W[:n].clone()
        p2p.forward(pos)
        p2p.reverse_w(g, W, go, Wo)
        return go, Wo, p2p.reduce(v).clone()

    ref = step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    bad = 0
    for _ in range(6):
        graph.replay()
        torch.cuda.synchronize()
        bad += not all(torch.equal(a, b) for a, b in zip(out, ref))
    return bad


def _worker(rank, world, port, q, shared):
    import torch.distributed as dist

    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", 0 if shared else rank)
    torch.cuda.set_device(dev)
    if shared:  # NCCL refuses two ranks on one device; set-up only needs gloo, the P2P step makes no collective call
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from allegro_b200.halo import P2PHalo, SlabDecomposition

        pos, cell, types, vel = _frame(world)
        res = {}
        for dtype in ("float64", "float32"):
            model = AllegroModel(**systems.model_kwargs("c2", 42.0, dtype)).to(dev).model
            for transport in (("p2p",) if shared else ("nccl", "p2p")):
                res[(dtype, transport)] = _run(rank, world, dev, dtype, transport, model, pos, cell, types, vel)
        # the mailbox layout must agree: a mismatch is refused on every rank at set-up, before anything is allocated
        dec = SlabDecomposition(pos, cell, types, 5.0, rank, world, device=dev).to(dev)
        try:
            P2PHalo(dec, dev, atomic_virial=(rank == 0))
            res["mismatch"] = "accepted"
        except ValueError as e:
            res["mismatch"] = str(e)
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
    res, deadline = [], time.time() + 600
    while len(res) < world:  # fail fast when a worker dies instead of waiting out the queue timeout
        try:
            res.append(q.get(timeout=2))
        except queue.Empty:
            dead = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
            assert not dead, f"worker exited with {dead}"
            assert time.time() < deadline, "timed out waiting for the workers"
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _reference(dtype, world):
    from allegro_b200 import data as D
    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel

    pos, cell, types, vel = _frame(world)
    ei, sh = D.neighbor_list(pos, 5.0, cell, (True, True, True))
    dt = getattr(torch, dtype)
    d = {D.POSITIONS_KEY: pos.to(dt), D.CELL_KEY: cell.to(dt), D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh,
         D.VELOCITY_KEY: vel.to(dt)}
    model = AllegroModel(**systems.model_kwargs("c2", 42.0, dtype)).to("cuda:0").model
    out = model.energy_and_forces({k: v.to("cuda:0") for k, v in d.items()}, stress=True, atomic_virial=True, heat_current=True)
    return {k: out[k].double().cpu() for k in (D.TOTAL_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.STRESS_KEY, D.VIRIAL_KEY,
                                                D.ATOMIC_VIRIAL_KEY, D.HEAT_CURRENT_KEY)}


def _check(res, transports):
    from allegro_b200 import data as D

    for _, r in res:
        assert "disagree" in r["mismatch"], r["mismatch"]
    for dtype in ("float64", "float32"):
        ref = _reference(dtype, len(res))
        n = ref[D.FORCE_KEY].shape[0]
        tol = TOL[dtype]
        gathered = {}
        for transport in transports:
            F, Ea, W = torch.zeros(n, 3, dtype=torch.float64), torch.zeros(n, 1, dtype=torch.float64), torch.zeros(n, 3, 3, dtype=torch.float64)
            seen = torch.zeros(n, dtype=torch.long)
            for _, r in res:
                owned, out, diff, err = r[(dtype, transport)]
                owned = torch.from_numpy(owned)
                assert err == 0
                if transport == "p2p":
                    diff, bad = diff
                    assert bad == 0, (dtype, bad)  # halo replay bitwise equal to halo eager
                assert diff <= tol, (dtype, transport, diff)
                seen[owned] += 1
                F[owned] = torch.from_numpy(out[D.FORCE_KEY])
                Ea[owned] = torch.from_numpy(out[D.PER_ATOM_ENERGY_KEY])
                W[owned] = torch.from_numpy(out[D.ATOMIC_VIRIAL_KEY])
                for k in (D.TOTAL_ENERGY_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.HEAT_CURRENT_KEY):
                    got = torch.from_numpy(out[k]).reshape(ref[k].shape)
                    assert _rel(got, ref[k]) < tol, (dtype, transport, k, _rel(got, ref[k]))
            assert bool((seen == 1).all())
            for k, v in ((D.FORCE_KEY, F), (D.PER_ATOM_ENERGY_KEY, Ea), (D.ATOMIC_VIRIAL_KEY, W)):
                assert _rel(v, ref[k]) < tol, (dtype, transport, k, _rel(v, ref[k]))
            gathered[transport] = (F, W)
        if dtype == "float64" and len(gathered) == 2:
            for a, b in zip(gathered["nccl"], gathered["p2p"]):
                assert _rel(a, b) < 1e-12


@pytest.mark.parametrize("world", [2, 4, 8])
def test_virial_halo_matches_single_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    _check(_collect(world, shared=False), ("nccl", "p2p"))


def test_p2p_virial_ranks_sharing_a_device():
    _check(_collect(2, shared=True), ("p2p",))
