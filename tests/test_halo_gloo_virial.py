"""world_size-2/3 gloo tests (CPU) of the stress, per-atom virial and heat current of the slab decomposition:
``DistributedAllegro.evaluate`` with every flag combination == the fp64 oracle on the whole periodic frame.

Each rank runs the package's fused model on the CPU through ``_energy_and_forces``, with every kernel wrapper replaced by
its torch restatement (tests/kernel_spec.py and the batch / virial restatements of tests/test_host_frames.py and
tests/test_host_atomic_virial.py), so the host logic -- ghost rows of W folded onto their owners by the reverse halo, the
width-12 exchange, the fp64 vector all-reduce, J over owned rows only -- is what is checked here.  The peer-memory
transport and the kernels are checked on the GPU (tests/test_gpu_halo_virial.py)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from allegro_b200 import data as D
from allegro_b200 import systems

# (stress, atomic_virial, heat_current); heat_current implies atomic_virial
FLAGS = [(False, False, False), (True, False, False), (False, True, False), (False, False, True), (True, True, False), (True, False, True)]
SMALL = dict(num_scalar_features=8, num_tensor_features=4, radial_chemical_embed_dim=8, scalar_embed_mlp_hidden_layers_width=8,
             allegro_mlp_hidden_layers_width=8, readout_mlp_hidden_layers_width=8)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _kwargs(name):
    kw = systems.model_kwargs(name, 42.0, "float64")
    kw.update(SMALL, per_type_energy_shifts=[-0.7] * len(systems.CONFIGS[name]["type_names"]))
    return kw


def _frame(name, reps):
    """displaced positions (so that the virial is not that of a perfect lattice) and seeded velocities of the global frame"""
    pos, cell, types = systems.make_positions(name, reps)
    g = torch.Generator().manual_seed(11)
    pos = pos + 0.1 * torch.randn(pos.shape, generator=g, dtype=pos.dtype)
    vel = torch.randn(pos.shape, generator=g, dtype=torch.float64)
    return pos, cell, types, vel


class _CpuFused:
    """the fused model's host path on CPU tensors (the public energy_and_forces refuses them)"""

    def __init__(self, m):
        self.m = m

    def energy_and_forces(self, data, stress=False, atomic_virial=False, heat_current=False):
        return self.m._energy_and_forces(data, stress, atomic_virial, heat_current)


def _install_spec_kernels():
    import kernel_spec
    from test_host_atomic_virial import VIRIAL_SPEC
    from test_host_frames import BATCH_SPEC

    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        setattr(_lib, name, getattr(kernel_spec, name))
    for name, fn in list(BATCH_SPEC.items()) + list(VIRIAL_SPEC.items()):
        setattr(_lib, name, fn)
    FusedAllegroEnergy.core = lambda self: self._core_for(torch.device("cpu"))


def _np(t):
    return t.detach().double().numpy().copy()


def _worker(rank, world, port, name, reps, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.set_num_threads(2)
        _install_spec_kernels()
        from test_host_frames import _models

        from allegro_b200.halo import DistributedAllegro, SlabDecomposition
        from oracle.model_ref import AllegroEnergyOracle, AllegroOracle

        kw = _kwargs(name)
        _, fused = _models(kw, AllegroOracle(**kw).state_dict())
        model = _CpuFused(fused)
        pos, cell, types, vel = _frame(name, reps)
        dec = SlabDecomposition(pos, cell, types, systems.CONFIGS[name]["r_max"], rank, world)
        pos_owned = dec.local_positions_from_global(pos)[: dec.n_owned]
        vel_owned = vel[dec.owned]
        plain = DistributedAllegro(model, dec)(pos_owned)
        out = {"owned": dec.owned.numpy().copy()}
        for flags in FLAGS:
            s, a, h = flags
            runner = DistributedAllegro(model, dec, stress=s, atomic_virial=a, heat_current=h)
            # __call__ is the plain step whatever the flags
            assert all(torch.equal(x, y) for x, y in zip(runner(pos_owned), plain))
            r = runner.evaluate(pos_owned, vel_owned if h else None)
            out[flags] = {k: _np(v) for k, v in r.items()}
        # refusals, made on every rank before any exchange: nobody is left waiting, the next collective step still works
        heat = DistributedAllegro(model, dec, heat_current=True)
        refused = 0
        for bad in (None, vel_owned[:-1], vel_owned[:, :2]):
            try:
                heat.evaluate(pos_owned, bad)
            except ValueError as e:
                refused += "velocities" in str(e)
        try:
            DistributedAllegro(AllegroEnergyOracle(**kw), dec, stress=True)
        except NotImplementedError:
            refused += 1
        again = heat.evaluate(pos_owned, vel_owned)
        out["refused"] = refused
        out["again"] = bool(torch.equal(again[D.HEAT_CURRENT_KEY], torch.from_numpy(out[(False, False, True)][D.HEAT_CURRENT_KEY])))
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _reference(name, reps):
    """fp64 oracle on the whole periodic frame: E, F, stress, virial, and W, J by autograd with the edge vectors as the leaf"""
    from test_host_atomic_virial import oracle_w_j

    from oracle.model_ref import AllegroOracle

    pos, cell, types, vel = _frame(name, reps)
    ei, sh = D.neighbor_list(pos, systems.CONFIGS[name]["r_max"], cell, (True, True, True))
    d = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh}
    oracle = AllegroOracle(**_kwargs(name))
    ref = oracle(d)
    W, J, _ = oracle_w_j(oracle, d, vel)
    return ref, W, J


@pytest.mark.parametrize("world,name,reps", [(2, "c2", (6, 3, 3)), (3, "c2", (6, 3, 3)), (2, "c5", (6, 3, 3))])
def test_slab_virial_and_heat_current_match_periodic_oracle(world, name, reps):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, name, reps, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ref, W_ref, J_ref = _reference(name, reps)
    n = ref[D.POSITIONS_KEY].shape[0]
    seen = torch.zeros(n, dtype=torch.long)
    for _, out in res:
        seen[torch.from_numpy(out["owned"])] += 1
        assert out["refused"] == 4 and out["again"]
    assert bool((seen == 1).all())  # every atom owned exactly once
    for flags in FLAGS:
        s, a, h = flags
        F = torch.zeros(n, 3, dtype=torch.float64)
        Ea = torch.zeros(n, 1, dtype=torch.float64)
        W = torch.zeros(n, 3, 3, dtype=torch.float64)
        totals = []
        for _, out in res:
            owned = torch.from_numpy(out["owned"])
            r = out[flags]
            F[owned] = torch.from_numpy(r[D.FORCE_KEY])
            Ea[owned] = torch.from_numpy(r[D.PER_ATOM_ENERGY_KEY])
            if a or h:
                W[owned] = torch.from_numpy(r[D.ATOMIC_VIRIAL_KEY])
            totals.append(r)
            assert (D.STRESS_KEY in r) == s and (D.VIRIAL_KEY in r) == s
            assert (D.ATOMIC_VIRIAL_KEY in r) == (a or h) and (D.HEAT_CURRENT_KEY in r) == h
        for r in totals:  # every rank holds the same totals
            assert _rel(r[D.TOTAL_ENERGY_KEY].reshape(-1), ref[D.TOTAL_ENERGY_KEY].reshape(-1)) < 1e-10, flags
            if s:
                assert r[D.STRESS_KEY].shape == (1, 3, 3) and r[D.VIRIAL_KEY].shape == (1, 3, 3)
                assert _rel(r[D.VIRIAL_KEY], ref[D.VIRIAL_KEY]) < 1e-10, flags
                assert _rel(r[D.STRESS_KEY], ref[D.STRESS_KEY]) < 1e-10, flags
            if h:
                assert r[D.HEAT_CURRENT_KEY].shape == (1, 3)
                assert _rel(r[D.HEAT_CURRENT_KEY][0], J_ref) < 1e-10, flags
        assert _rel(Ea, ref[D.PER_ATOM_ENERGY_KEY]) < 1e-10, flags
        assert _rel(F, ref[D.FORCE_KEY]) < 1e-10, flags
        if a or h:
            assert _rel(W, W_ref) < 1e-10, flags
