"""Per-atom virials and the heat current on the HOST side, on a CPU-only box.

The two new kernels are restated below in torch (what include/allegro_b200.h says ab2_force_virial_scatter and
ab2_frame_heat_current compute) and monkeypatched over their wrappers together with tests/kernel_spec.py and the batch
restatements of tests/test_host_frames.py.  Every host path that can return ``atomic_virial`` / ``heat_current`` --
single frame, prepared CSR, both ghost formats, batches, a pair potential, frames without edges -- is compared with the
fp64 oracle, which gets W from autograd with the edge vectors as the leaf:

    W_ref[a] = - sum_{z : nbr[z] = a} vec[z] (x) dE/dvec[z],     J_ref = sum_a E_a v_a + W_ref[a] v_a

The kernels themselves are checked on the GPU (tests/test_gpu_atomic_virial.py).
"""
import pytest
import torch

import kernel_spec
from golden_util import load_models, unpack_state_dict
from test_host_frames import BATCH_SPEC, _mixed_frames, _models

MODELS = {r["name"]: r for r in load_models()}


# --------------------------------------------------------------------------- #
# restatements of the two kernels
# --------------------------------------------------------------------------- #
def force_virial_scatter(vec, gvec, csr, num_atoms_total):
    F = kernel_spec.force_scatter(gvec, csr, num_atoms_total)
    outer = vec.unsqueeze(2) * gvec.unsqueeze(1)
    W = torch.zeros(num_atoms_total, 3, 3, dtype=gvec.dtype).index_add_(0, csr.nbr.long(), -outer)
    return F, W


def frame_heat_current(e_atom, vel, W, frame_ptr):
    n = W.shape[0]
    v = vel.double()
    per = e_atom.reshape(n, 1).double() * v + (W.double() @ v.unsqueeze(2)).squeeze(2)
    fp = frame_ptr.long().tolist()
    return torch.stack([per[fp[b]:fp[b + 1]].sum(0) for b in range(len(fp) - 1)]).to(W.dtype)


VIRIAL_SPEC = {"force_virial_scatter": force_virial_scatter, "frame_heat_current": frame_heat_current}


@pytest.fixture()
def spec_kernels(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    for name, fn in list(BATCH_SPEC.items()) + list(VIRIAL_SPEC.items()):
        monkeypatch.setattr(_lib, name, fn)
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))


# --------------------------------------------------------------------------- #
# the fp64 oracle
# --------------------------------------------------------------------------- #
def oracle_w_j(oracle, d, vel=None):
    """(W_ref [n,3,3], J_ref [3] or None, E_atom [n]) of one frame from the oracle energy model with vec as the leaf."""
    from allegro_b200 import data as D

    pos = d[D.POSITIONS_KEY].double()
    ei = d[D.EDGE_INDEX_KEY]
    n = pos.shape[0]
    vec = pos[ei[1]] - pos[ei[0]]
    if D.EDGE_CELL_SHIFT_KEY in d and D.CELL_KEY in d:
        vec = vec + d[D.EDGE_CELL_SHIFT_KEY].double() @ d[D.CELL_KEY].view(3, 3).double()
    vec = vec.detach().requires_grad_(True)
    inp = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: d[D.ATOM_TYPE_KEY], D.EDGE_INDEX_KEY: ei, "edge_vectors": vec,
           "edge_lengths": vec.norm(dim=-1)}
    with torch.enable_grad():
        out = oracle.model(inp)
        e = out[D.PER_ATOM_ENERGY_KEY].reshape(-1)
        if vec.shape[0]:
            (g,) = torch.autograd.grad(e.sum(), vec)
        else:
            g = torch.zeros_like(vec)
    W = torch.zeros(n, 3, 3, dtype=torch.float64).index_add_(0, ei[1], -(vec.detach().unsqueeze(2) * g.unsqueeze(1)))
    J = None
    if vel is not None:
        v = vel.double()
        J = (e.detach().unsqueeze(1) * v).sum(0) + (W @ v.unsqueeze(2)).squeeze(2).sum(0)
    return W, J, e.detach()


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _vel(n, seed):
    return torch.randn(n, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _tol(kw):
    return 1e-10 if kw["model_dtype"] == "float64" else 5e-5


# --------------------------------------------------------------------------- #
# single frame: edge_index and prepared CSR
# --------------------------------------------------------------------------- #
CASES = ["c1_lmax1_L1", "c2_lmax2_L2", "c2_lmax2_L2_f32", "c5_lmax3_L3_5species", "cluster_open_unsorted", "isolated_atoms_ragged_rows",
         "no_edges_at_all", "spline_embed_reftest_cfg"]


def _prepared(d):
    """The same frame as a prebuilt CSR + shift vectors (the calculator's route)."""
    from allegro_b200 import data as D

    p = {k: v for k, v in d.items() if k not in (D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY)}
    csr = D.build_csr(d[D.EDGE_INDEX_KEY], d[D.POSITIONS_KEY].shape[0])
    p[D.CSR_KEY] = csr
    if D.EDGE_CELL_SHIFT_KEY in d:
        sh = d[D.EDGE_CELL_SHIFT_KEY] if csr.perm is None else d[D.EDGE_CELL_SHIFT_KEY][csr.perm]
        p[D.EDGE_SHIFT_VEC_KEY] = sh.double() @ d[D.CELL_KEY].view(3, 3).double()
    return p


@pytest.mark.parametrize("route", ["edge_index", "prepared"])
@pytest.mark.parametrize("name", CASES)
def test_single_frame_against_oracle(name, route, spec_kernels):
    from allegro_b200 import data as D

    rec = MODELS[name]
    kw = rec["kwargs"]
    oracle, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    d = dict(rec["data"])
    n = d[D.POSITIONS_KEY].shape[0]
    vel = _vel(n, len(name))
    W_ref, J_ref, _ = oracle_w_j(oracle, d, vel)
    inp = dict(d) if route == "edge_index" else _prepared(d)
    inp[D.VELOCITY_KEY] = vel
    stress = D.CELL_KEY in d
    out = model._energy_and_forces(inp, stress, False, True)
    plain = model._energy_and_forces(inp, stress)
    tol = _tol(kw)
    W = out[D.ATOMIC_VIRIAL_KEY]
    assert W.shape == (n, 3, 3) and out[D.HEAT_CURRENT_KEY].shape == (1, 3)
    assert _rel(W, W_ref) < tol, _rel(W, W_ref)
    assert _rel(out[D.HEAT_CURRENT_KEY][0], J_ref) < tol, (out[D.HEAT_CURRENT_KEY], J_ref)
    for k in (D.FORCE_KEY, D.PER_ATOM_ENERGY_KEY):
        assert torch.equal(out[k], plain[k]), k
    if stress:  # the symmetric part of the sum is the virial output
        Ws = W.double().sum(0)
        assert _rel(0.5 * (Ws + Ws.T), plain[D.VIRIAL_KEY][0]) < tol
    if d[D.EDGE_INDEX_KEY].shape[1] == 0:
        assert bool((W == 0).all())
        e = out[D.PER_ATOM_ENERGY_KEY].double()
        assert _rel(out[D.HEAT_CURRENT_KEY][0], (e * vel).sum(0)) < 1e-12
    # atomic_virial alone: the same W, no heat current, no velocities needed
    inp.pop(D.VELOCITY_KEY)
    only = model._energy_and_forces(inp, stress, True, False)
    assert torch.equal(only[D.ATOMIC_VIRIAL_KEY], W) and D.HEAT_CURRENT_KEY not in only


def test_pair_potential_against_oracle(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200 import systems
    from oracle.model_ref import AllegroOracle

    d = systems.make_system("c3", 2)
    kw = systems.model_kwargs("c3", d[D.EDGE_INDEX_KEY].shape[1] / 8, "float64")
    kw.update(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16, scalar_embed_mlp_hidden_layers_width=16,
              allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=16, per_type_energy_scales=[0.7, 1.3, 0.9],
              per_type_energy_shifts=[0.1, -0.2, 0.3],
              pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})
    oracle, model = _models(kw, AllegroOracle(**kw).state_dict())
    n = d[D.POSITIONS_KEY].shape[0]
    vel = _vel(n, 3)
    W_ref, J_ref, e_ref = oracle_w_j(oracle, d, vel)
    inp = dict(d)
    inp[D.VELOCITY_KEY] = vel
    out = model._energy_and_forces(inp, True, False, True)
    assert _rel(out[D.PER_ATOM_ENERGY_KEY].reshape(-1), e_ref) < 1e-10
    assert _rel(out[D.ATOMIC_VIRIAL_KEY], W_ref) < 1e-10
    assert _rel(out[D.HEAT_CURRENT_KEY][0], J_ref) < 1e-10


# --------------------------------------------------------------------------- #
# ghost formats against the periodic frame
# --------------------------------------------------------------------------- #
def _ghost_owners(d):
    """Owner of every appended ghost of data.to_ghost_format(d), in ghost order."""
    from allegro_b200 import data as D

    outside = d[D.EDGE_CELL_SHIFT_KEY].abs().sum(-1) != 0
    return d[D.EDGE_INDEX_KEY][1, outside]


@pytest.mark.parametrize("name", ["c2_lmax2_L2", "c5_lmax3_L3_5species"])
def test_ghost_formats_fold_onto_the_periodic_frame(name, spec_kernels):
    from allegro_b200 import data as D

    rec = MODELS[name]
    kw = rec["kwargs"]
    _, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    d = dict(rec["data"])
    n = d[D.POSITIONS_KEY].shape[0]
    vel = _vel(n, 9)
    per = dict(d)
    per[D.VELOCITY_KEY] = vel
    ref = model._energy_and_forces(per, False, False, True)
    g = D.to_ghost_format(d)
    g.pop("num_local_atoms")
    owners = _ghost_owners(d)
    n_all = g[D.POSITIONS_KEY].shape[0]
    assert n_all == n + owners.shape[0]
    vg = torch.cat([vel, vel[owners]])
    # (a) appended ghosts given as edge_index (every atom has a row; ghosts own no edge)
    ga = dict(g)
    ga[D.VELOCITY_KEY] = vg
    oa = model._energy_and_forces(ga, False, False, True)
    # (b) a prepared CSR with rows for the owned atoms only (the halo / pair-style layout)
    gb = {D.POSITIONS_KEY: g[D.POSITIONS_KEY], D.ATOM_TYPE_KEY: g[D.ATOM_TYPE_KEY], D.CSR_KEY: D.build_csr(g[D.EDGE_INDEX_KEY], n),
          D.VELOCITY_KEY: vg}
    ob = model._energy_and_forces(gb, False, False, True)
    for o in (oa, ob):
        W = o[D.ATOMIC_VIRIAL_KEY]
        assert W.shape == (n_all, 3, 3)
        folded = W[:n].clone().index_add_(0, owners, W[n:])
        assert _rel(folded, ref[D.ATOMIC_VIRIAL_KEY]) < 1e-10
    # with rows for the owned atoms only, the ghosts carry no energy: J is the periodic J
    assert ob[D.PER_ATOM_ENERGY_KEY].shape[0] == n
    assert _rel(ob[D.HEAT_CURRENT_KEY], ref[D.HEAT_CURRENT_KEY]) < 1e-10
    # appended ghosts are centres without edges (energy = the per-type shift): J sums over every row given
    e = oa[D.PER_ATOM_ENERGY_KEY].reshape(-1).double()
    ghost_term = (e[n:].unsqueeze(1) * vg[n:]).sum(0)
    assert _rel(oa[D.HEAT_CURRENT_KEY][0] - ghost_term, ref[D.HEAT_CURRENT_KEY][0]) < 1e-10


# --------------------------------------------------------------------------- #
# batches
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", ["c2_lmax2_L2", "c2_lmax2_L2_f32", "cluster_open_unsorted"])
def test_batch_equals_single_frames_and_oracle(name, spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate, split

    rec = MODELS[name]
    kw = rec["kwargs"]
    oracle, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    frames = _mixed_frames(rec["data"], kw["r_max"], len(kw["type_names"]), seed=7)
    for i, f in enumerate(frames):
        f[D.VELOCITY_KEY] = _vel(f[D.POSITIONS_KEY].shape[0], 100 + i)
    batch = collate(frames)
    assert D.VELOCITY_KEY in batch
    out = model._energy_and_forces_frames(batch, False, False, True)
    B = len(frames)
    assert out[D.HEAT_CURRENT_KEY].shape == (B, 3)
    tol = _tol(kw)
    fp = batch[D.NUM_NODES_KEY].cumsum(0).tolist()
    fp = [0] + fp
    for b, f in enumerate(frames):
        one = model._energy_and_forces(f, False, False, True)
        Wb = out[D.ATOMIC_VIRIAL_KEY][fp[b]:fp[b + 1]]
        assert _rel(Wb, one[D.ATOMIC_VIRIAL_KEY]) < tol, b
        assert _rel(out[D.HEAT_CURRENT_KEY][b], one[D.HEAT_CURRENT_KEY][0]) < tol, b
        W_ref, J_ref, _ = oracle_w_j(oracle, f, f[D.VELOCITY_KEY])
        assert _rel(Wb, W_ref) < tol, b
        scale = float(J_ref.abs().max()) or 1.0
        assert float((out[D.HEAT_CURRENT_KEY][b].double() - J_ref).abs().max()) / scale < tol, b
    for b, p in enumerate(split(out)):  # split hands every frame its rows and its [1,3] heat current
        assert torch.equal(p[D.HEAT_CURRENT_KEY], out[D.HEAT_CURRENT_KEY][b:b + 1])
        assert torch.equal(p[D.ATOMIC_VIRIAL_KEY], out[D.ATOMIC_VIRIAL_KEY][fp[b]:fp[b + 1]])
        assert torch.equal(p[D.VELOCITY_KEY], frames[b][D.VELOCITY_KEY])


# --------------------------------------------------------------------------- #
# validation and the opt-out
# --------------------------------------------------------------------------- #
def _c2():
    from allegro_b200 import data as D

    rec = MODELS["c2_lmax2_L2"]
    _, model = _models(rec["kwargs"], unpack_state_dict(rec["state_dict"]))
    d = dict(rec["data"])
    return model, d, d[D.POSITIONS_KEY].shape[0]


def test_heat_current_needs_velocities_of_every_atom(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, d, n = _c2()
    with pytest.raises(ValueError, match="velocities"):
        model._energy_and_forces(d, False, False, True)
    for bad in (torch.zeros(n - 1, 3, dtype=torch.float64), torch.zeros(n, 2, dtype=torch.float64), torch.zeros(3 * n, dtype=torch.float64)):
        dd = dict(d)
        dd[D.VELOCITY_KEY] = bad
        with pytest.raises(ValueError, match="velocities"):
            model._energy_and_forces(dd, False, False, True)
    batch = collate([d, d])
    with pytest.raises(ValueError, match="velocities"):
        model._energy_and_forces_frames(batch, False, False, True)
    batch[D.VELOCITY_KEY] = torch.zeros(n, 3, dtype=torch.float64)
    with pytest.raises(ValueError, match="velocities"):
        model._energy_and_forces_frames(batch, False, False, True)


def test_autograd_branch_refuses_the_new_outputs(spec_kernels):
    from allegro_b200.model.allegro_models import ForceStressOutput

    model, d, n = _c2()
    wrapped = ForceStressOutput(model)
    assert wrapped.compute_atomic_virial is False and wrapped.compute_heat_current is False
    wrapped.use_autograd = True
    for attr in ("compute_atomic_virial", "compute_heat_current"):
        setattr(wrapped, attr, True)
        with pytest.raises(NotImplementedError):
            wrapped(d)
        setattr(wrapped, attr, False)


def test_without_flags_the_output_keys_are_unchanged(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, d, n = _c2()
    dv = dict(d)
    dv[D.VELOCITY_KEY] = _vel(n, 1)  # velocities alone switch nothing on
    expected = set(dv) | {D.EDGE_FEATURES_KEY, D.EDGE_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.TOTAL_ENERGY_KEY, D.FORCE_KEY}
    assert set(model._energy_and_forces(dv, False)) == expected
    assert set(model._energy_and_forces(dv, True)) == expected | {D.STRESS_KEY, D.VIRIAL_KEY}
    batch = collate([d, d])
    out = model._energy_and_forces_frames(batch, False)
    assert D.ATOMIC_VIRIAL_KEY not in out and D.HEAT_CURRENT_KEY not in out
