"""The model on lists pruned to its per-edge-type cutoffs: the same energies, forces, stress, per-atom virials and heat
current as on the unpruned list (an edge beyond its own cutoff contributes an exact zero), for the fp32-grid Li/P/S
table, the reference's asymmetric H/C/O table with the spline embedding and a ZBL model; the MD calculators with
``prune_edges=True`` against exact-r_max evaluations at every step (one GPU, and two slab ranks sharing it)."""
import os
import queue
import time

import pytest
import torch

from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from oracle.model_ref import AllegroOracle

pytestmark = pytest.mark.gpu
DEV = "cuda"

GRID_TABLE = {"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}  # tests/test_gpu_fp32_grid.py, three_species
SMALL = dict(num_scalar_features=32, num_tensor_features=16, radial_chemical_embed_dim=32, scalar_embed_mlp_hidden_layers_width=32,
             allegro_mlp_hidden_layers_width=32, readout_mlp_hidden_layers_width=32)
OUTPUTS = (D.TOTAL_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.STRESS_KEY, D.VIRIAL_KEY, D.ATOMIC_VIRIAL_KEY, D.HEAT_CURRENT_KEY)


def _kwargs(kind):
    kw = systems.model_kwargs("c3", 40.0, "float64")
    kw.update(SMALL, per_type_energy_shifts=[0.5, -1.0, 0.25])
    if kind == "grid":
        kw.update(per_edge_type_cutoff=GRID_TABLE)
    elif kind == "zbl":
        kw.update(per_edge_type_cutoff=GRID_TABLE,
                  pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})
    elif kind == "spline":
        from golden_util import load_models

        ref = {r["name"]: r for r in load_models()}["spline_embed_per_edge_type_cutoff"]["kwargs"]
        kw = dict(ref)
        assert kw["per_edge_type_cutoff"]["C"]["H"] != kw["per_edge_type_cutoff"]["H"]  # asymmetric: H -> C 2.0, C -> H 4.0
    return kw


def _models(kind):
    kw = _kwargs(kind)
    oracle = AllegroOracle(**kw)
    out = {}
    for dt in ("float64", "float32"):
        m = AllegroModel(**dict(kw, model_dtype=dt))
        m.load_state_dict(oracle.state_dict())
        out[dt] = m.to(DEV).model
    return oracle, out, kw


def _frame(scale, dtype, seed=3):
    pos, cell, types = systems.make_positions("c3", scale)
    g = torch.Generator().manual_seed(seed)
    vel = 0.3 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
    return pos.to(DEV, dtype), cell.to(DEV, dtype), types.to(DEV), vel.to(DEV, dtype)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _eval(model, pos, cell, types, vel, csr, sv):
    d = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv, D.VELOCITY_KEY: vel}
    out = model.energy_and_forces(d, stress=True, atomic_virial=True, heat_current=True)
    return {k: out[k].clone() for k in OUTPUTS}


@pytest.mark.parametrize("kind", ["grid", "spline", "zbl"])
def test_pruned_list_gives_the_unpruned_outputs(kind):
    oracle, models, kw = _models(kind)
    r_max = kw["r_max"]
    tab = models["float64"].edge_norm.rmax_table
    for dt in ("float64", "float32") if kind == "grid" else ("float64",):
        pos, cell, types, vel = _frame(6, getattr(torch, dt))
        csr, sv = D.neighbor_csr(pos, r_max, cell, (True, True, True))
        pcsr, psv = D.prune_csr(csr, sv, pos, types, tab)
        assert 0 < pcsr.num_edges < csr.num_edges
        print(f"\n[prune-model] {kind} {dt}: edges {csr.num_edges} -> {pcsr.num_edges}")
        full = _eval(models[dt], pos, cell, types, vel, csr, sv)
        pruned = _eval(models[dt], pos, cell, types, vel, pcsr, psv)
        if dt == "float64":
            for k in OUTPUTS:
                assert _rel(pruned[k], full[k]) < 1e-12, (kind, k, _rel(pruned[k], full[k]))
        else:  # fp32 on the pruned list against the fp64 oracle on an exact r_max list
            ei, sh = D.neighbor_list(pos.double().cpu(), r_max, cell.double().cpu(), (True, True, True))
            ref = oracle({D.POSITIONS_KEY: pos.double().cpu(), D.CELL_KEY: cell.double().cpu(), D.ATOM_TYPE_KEY: types.cpu(),
                          D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh})
            assert _rel(pruned[D.PER_ATOM_ENERGY_KEY], ref[D.PER_ATOM_ENERGY_KEY]) < 1e-4
            assert _rel(pruned[D.FORCE_KEY], ref[D.FORCE_KEY]) < 1e-4
            assert _rel(pruned[D.FORCE_KEY], full[D.FORCE_KEY]) < 1e-4


def test_calculator_prune_edges_trajectory():
    from allegro_b200.calculator import AllegroCalculator

    _, models, kw = _models("grid")
    model, r_max = models["float64"], kw["r_max"]
    pos, cell, types, vel = _frame(6, torch.float64, seed=5)
    kwc = dict(skin=0.5, compute_stress=True, compute_heat_current=True)
    pruned, plain = AllegroCalculator(model, r_max, prune_edges=True, **kwc), AllegroCalculator(model, r_max, **kwc)
    g = torch.Generator(device=DEV).manual_seed(9)
    rebuilds = []
    for step in range(20):
        a = {k: v.clone() for k, v in pruned.compute(pos, cell, types, velocities=vel).items()}
        b = {k: v.clone() for k, v in plain.compute(pos, cell, types, velocities=vel).items()}
        rebuilds.append((pruned.n_rebuilds, plain.n_rebuilds))
        assert pruned.num_edges < plain.num_edges
        csr, sv = D.neighbor_csr(pos, r_max, cell, (True, True, True))
        ref = _eval(model, pos, cell, types, vel, csr, sv)
        for key, rk in (("energy", D.TOTAL_ENERGY_KEY), ("forces", D.FORCE_KEY), ("stress", D.STRESS_KEY),
                        ("atomic_virial", D.ATOMIC_VIRIAL_KEY), ("heat_current", D.HEAT_CURRENT_KEY)):
            assert _rel(a[key], ref[rk]) < 1e-12, (step, key, _rel(a[key], ref[rk]))
            assert _rel(b[key], ref[rk]) < 1e-12, (step, key)
        pos = pos + 0.06 * torch.randn(pos.shape, generator=g, device=DEV, dtype=pos.dtype)
    assert all(p == q for p, q in rebuilds), rebuilds
    assert rebuilds[-1][0] >= 3, rebuilds


# ---- two slab ranks sharing the device ----------------------------------------------------------------------------------
STEPS = 12


def _free_port():
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _md_frame():
    pos, cell, types = systems.make_positions("c3", (8, 5, 5))
    g = torch.Generator().manual_seed(21)
    vel = 0.3 * torch.randn(pos.shape, generator=g, dtype=torch.float64)
    return pos, cell, types, vel


def _worker(rank, world, port, q):
    import torch.distributed as dist

    from allegro_b200.halo import DistributedCalculator

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        _, models, kw = _models("grid")
        pos, cell, types, vel = _md_frame()
        calc = DistributedCalculator(models["float64"], cell, kw["r_max"], 0.5, rank, world, device=dev, prune_edges=True)
        assert calc.r_list == 6.5 and calc._cutoffs is not None
        local = calc.distribute(pos, types, velocities=vel)
        res = []
        for step in range(STEPS + 1):
            if step:
                local.pos += 0.1 * local.arrays["velocities"]
            out = calc.compute(local)
            frame = calc.gather(local)
            # numpy copies: tensors would travel as shared-memory handles that die with this process
            res.append({"ids": local.ids.cpu().numpy().copy(), "forces": out[D.FORCE_KEY].double().cpu().numpy().copy(),
                        "e": float(out[D.TOTAL_ENERGY_KEY].reshape(-1)[0]), "edges": calc.plan.n_edges,
                        "pos": None if frame is None else frame["pos"].numpy().copy()})
        q.put((rank, res, calc.n_rebuilds))
        calc.close()
        dist.barrier()
        torch.cuda.synchronize()
        q.close()
        q.join_thread()
        os._exit(0)
    except BaseException:
        dist.destroy_process_group()
        raise


def test_distributed_calculator_prune_edges_two_ranks_one_device():
    import torch.multiprocessing as mp

    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got, deadline = [], time.time() + 900
    try:
        while len(got) < world:
            try:
                got.append(q.get(timeout=2))
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
    got.sort(key=lambda r: r[0])
    assert got[0][2] == got[1][2] >= 2, [g[2] for g in got]
    _, models, kw = _models("grid")
    model, r_max = models["float64"], kw["r_max"]
    _, cell, types, _ = _md_frame()
    cell_d, types_d = cell.to(DEV), types.to(DEV)
    for s in range(STEPS + 1):
        pos = torch.from_numpy(got[0][1][s]["pos"]).to(DEV)
        csr, sv = D.neighbor_csr(pos, r_max, cell_d, (True, True, True))
        skin_csr, _ = D.neighbor_csr(pos, r_max + 0.5, cell_d, (True, True, True))
        d ={D.POSITIONS_KEY: pos, D.CELL_KEY: cell_d, D.ATOM_TYPE_KEY: types_d, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
        ref = model.energy_and_forces(d)
        F = torch.zeros(pos.shape[0], 3, dtype=torch.float64)
        for _, res, _ in got:
            F[torch.from_numpy(res[s]["ids"]).long()] = torch.from_numpy(res[s]["forces"])
        assert _rel(F, ref[D.FORCE_KEY]) < 1e-9, (s, _rel(F, ref[D.FORCE_KEY]))
        e = float(ref[D.TOTAL_ENERGY_KEY].reshape(-1)[0])
        assert abs(got[0][1][s]["e"] - e) < 1e-9 * float(ref[D.PER_ATOM_ENERGY_KEY].abs().sum()), s
        # pruned: fewer edges than the r_max + skin list holds
        assert sum(res[s]["edges"] for _, res, _ in got) < skin_csr.num_edges, s
