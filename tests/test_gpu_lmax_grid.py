"""Models at l_max 4 and l_max 0, the two ends of the range the kernels are instantiated for (AB2_MAX_LMAX), on the GPU
against the fp64 oracle.

At l_max 4 every tensor product runs the shape-generic kernels of tp.cu (tables of 1158 and 2052 entries, d up to 49), the
environment adjoint runs env_bwd_kernel<..., 4> and the latent MLPs write S + 5U columns; at l_max 0 the tables are 1 x 1 x 1
and the SH adjoint is zero.  fp64 models are held to 1e-9 on atomic energies, total energy, forces, stress and per-atom
virials (the latter from oracle autograd with the edge vectors as the leaf), on the c2 architecture at 3^3 (108 atoms) and
on the golden open cluster with isolated atoms and the frame without edges.  Further: a batch of frames, a CUDA-graph
replay of the MD calculator, the reference-generated vectors of tests/golden/ref_models_lmax.*.pt, and a check that the
l = 4 channels carry enough of the forces for the comparisons to see them.
"""
import pytest
import torch

from allegro_b200 import data as D
from allegro_b200 import systems
from golden_util import load_models, load_sharded, unpack_state_dict
from test_gpu_model import _check, _pair, _to_dev

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-9

GRID = {
    "lmax4_L1": dict(l_max=4, num_layers=1),
    "lmax4_L1_noparity": dict(l_max=4, num_layers=1, parity=False),
    "lmax4_L2": dict(l_max=4, num_layers=2),
    "lmax4_L2_noparity": dict(l_max=4, num_layers=2, parity=False),
    "lmax4_L3": dict(l_max=4, num_layers=3),
    "lmax4_L3_noparity": dict(l_max=4, num_layers=3, parity=False),
    "lmax4_L2_no_coupling": dict(l_max=4, num_layers=2, tp_path_channel_coupling=False),
    "lmax0_L1": dict(l_max=0, num_layers=1),
    "lmax0_L2": dict(l_max=0, num_layers=2),
}
# the golden open-boundary frames (centres without edges in the middle of the index range; no edge at all) on these
GOLDEN_FRAMES = ("isolated_atoms_ragged_rows", "no_edges_at_all")
ON_GOLDEN_FRAMES = ("lmax4_L2", "lmax4_L3", "lmax0_L2")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0) if a.numel() else 0.0


def _oracle_forces_and_virials(oracle, d):
    """(forces [n,3], per-atom virials [n,3,3], virial [3,3]) from one oracle pass with the edge vectors as the autograd leaf:
    F = -dE/dr, W_j = -sum over edges z with neighbour j of vec_z (x) dE/dvec_z, virial = sum_j W_j."""
    pos = d[D.POSITIONS_KEY].double()
    ei = d[D.EDGE_INDEX_KEY]
    n = pos.shape[0]
    vec = pos[ei[1]] - pos[ei[0]]
    if D.EDGE_CELL_SHIFT_KEY in d and D.CELL_KEY in d:
        vec = vec + d[D.EDGE_CELL_SHIFT_KEY].double() @ d[D.CELL_KEY].view(3, 3).double()
    vec = vec.detach().requires_grad_(True)
    inp = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: d[D.ATOM_TYPE_KEY], D.EDGE_INDEX_KEY: ei, "edge_vectors": vec, "edge_lengths": vec.norm(dim=-1)}
    with torch.enable_grad():
        e = oracle.model(inp)[D.PER_ATOM_ENERGY_KEY].reshape(-1)
        g = torch.autograd.grad(e.sum(), vec)[0] if vec.shape[0] else torch.zeros_like(vec)
    F = torch.zeros(n, 3, dtype=torch.float64).index_add_(0, ei[0], g).index_add_(0, ei[1], -g)
    W = torch.zeros(n, 3, 3, dtype=torch.float64).index_add_(0, ei[1], -(vec.detach().unsqueeze(2) * g.unsqueeze(1)))
    return F, W, W.sum(0)


def _golden_frame_pair(name, over):
    """fp64 oracle and model of the c2 architecture with `over` on the frame of a golden case (two species, open, r_max 3.5)."""
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    d = dict({r["name"]: r for r in load_models()}[name]["data"])
    kw = systems.model_kwargs("c2", 9.0, "float64")
    kw.update(type_names=["X", "Y"], r_max=3.5, per_type_energy_shifts=[0.5, -1.0], **over)
    oracle = AllegroOracle(**kw)
    model = AllegroModel(**kw)
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to(DEV), d


def _check_all(oracle, model, d):
    """_check (atomic and total energy, forces) plus stress and per-atom virials against the oracle; returns the errors."""
    ee, ef = _check(oracle, model, d, TOL, TOL)
    F_ref, W_ref, vir_ref = _oracle_forces_and_virials(oracle, d)
    stress = D.CELL_KEY in d
    out = model.model.energy_and_forces(_to_dev(d), stress=stress, atomic_virial=True)
    n = F_ref.shape[0]
    assert _rel(out[D.FORCE_KEY][:n], F_ref) < TOL  # the leaf-vector oracle agrees with the oracle's own forces
    ew = _rel(out[D.ATOMIC_VIRIAL_KEY][:n], W_ref)
    assert ew < TOL, f"per-atom virial rel err {ew}"
    es = 0.0
    if stress:
        volume = float(torch.linalg.det(d[D.CELL_KEY].view(3, 3).double()).abs())
        es = _rel(out[D.VIRIAL_KEY][0], vir_ref)
        assert es < TOL, f"virial rel err {es}"
        assert _rel(out[D.STRESS_KEY][0], -vir_ref / volume) < TOL
    return ee, ef, ew, es


def _cases():
    out = [pytest.param(c, "c2_3", id=f"{c}-c2_3") for c in GRID]
    out += [pytest.param(c, f, id=f"{c}-{f}") for c in ON_GOLDEN_FRAMES for f in GOLDEN_FRAMES]
    return out


@pytest.mark.parametrize("case,frame", _cases())
def test_fp64_against_oracle(case, frame):
    if frame == "c2_3":
        oracle, model, d = _pair("c2", 3, "float64", **GRID[case])
    else:
        oracle, model, d = _golden_frame_pair(frame, GRID[case])
    ee, ef, ew, es = _check_all(oracle, model, d)
    print(f"\n{case} {frame} (E = {d[D.EDGE_INDEX_KEY].shape[1]}): E {ee:.1e} F {ef:.1e} W {ew:.1e} virial {es:.1e}")


@pytest.mark.parametrize("case", ["lmax4_L2", "lmax4_L3"])
def test_lmax4_channels_carry_the_forces(case):
    """A comparison that cannot see the l = 4 channels would pass on a kernel that drops them.  With the l = 4 columns of the
    two-body env weights zeroed (MakeWeightedChannels layout [u][l]) the forces move by far more than the fp64 bar, and the
    CUDA model follows the oracle to the bar with and without them."""
    oracle, model, d = _pair("c2", 3, "float64", **GRID[case])
    F0 = model(_to_dev(d))[D.FORCE_KEY].double().cpu()
    sd = oracle.state_dict()
    w = sd["model.tensor_embed.env_embed_linear.weights.0"]
    w.view(w.shape[0], -1, 5)[:, :, 4] = 0
    oracle.load_state_dict(sd)
    model.load_state_dict(sd)
    _check(oracle, model, d, TOL, TOL)
    moved = _rel(model(_to_dev(d))[D.FORCE_KEY], F0)
    print(f"\n{case}: forces move by {moved:.2e} of max |F| without the l = 4 env weights")
    assert moved > 100 * TOL


def test_lmax4_batch_of_frames():
    """energy_and_forces_frames at l_max 4: periodic FCC frames (one sheared into a triclinic cell), an open cluster and a
    one-atom frame without edges, each against the oracle on the batch's own neighbour rows."""
    from allegro_b200.batch import collate, split
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle
    from test_gpu_frames import _model_frames

    kw = systems.model_kwargs("c2", 40.0, "float64")
    kw.update(GRID["lmax4_L2"])
    oracle = AllegroOracle(**kw)
    model = AllegroModel(**kw)
    model.load_state_dict(oracle.state_dict())
    model = model.to(DEV)
    frames = _model_frames("c2", 1, torch.Generator().manual_seed(43), False)
    batch = collate([{k: v.to(DEV) for k, v in f.items()} for f in frames], kw["r_max"])
    out = model.energy_and_forces_frames(batch)
    n_edges = []
    for b, (f, fin, fo) in enumerate(zip(frames, split(batch), split(out))):
        csr, sv = fin[D.CSR_KEY], fin[D.EDGE_SHIFT_VEC_KEY].double().cpu()
        ref_in = {D.POSITIONS_KEY: f[D.POSITIONS_KEY], D.ATOM_TYPE_KEY: f[D.ATOM_TYPE_KEY],
                  D.EDGE_INDEX_KEY: torch.stack([csr.ctr.long(), csr.nbr.long()]).cpu()}
        if D.CELL_KEY in f:
            ref_in[D.CELL_KEY] = f[D.CELL_KEY]
            ref_in[D.EDGE_CELL_SHIFT_KEY] = torch.round(sv @ torch.linalg.inv(f[D.CELL_KEY]))
        ref = oracle(ref_in)
        n_edges.append(csr.num_edges)
        for k in (D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY):
            assert _rel(fo[k], ref[k]) < TOL, (b, k, _rel(fo[k], ref[k]))
        e_scale = float(ref[D.PER_ATOM_ENERGY_KEY].abs().sum())
        assert abs(float(fo[D.TOTAL_ENERGY_KEY]) - float(ref[D.TOTAL_ENERGY_KEY])) <= TOL * e_scale, b
    assert n_edges[-1] == 0 and min(n_edges[:-1]) > 0


def test_lmax4_calculator_graph_replay_matches_eager():
    """The MD calculator at l_max 4: CUDA-graph replay against eager evaluation along a short random walk.  The generic
    tensor-product backward adds gamma and gY gradients with atomics, so the two agree to rounding, not bitwise."""
    from allegro_b200.calculator import AllegroCalculator

    _, model, d = _pair("c2", 3, "float64", **GRID["lmax4_L2"])
    pos, cell, types = d[D.POSITIONS_KEY], d[D.CELL_KEY].to(DEV), d[D.ATOM_TYPE_KEY].to(DEV)
    calcs = [AllegroCalculator(model, 5.0, skin=0.6, use_graph=ug) for ug in (True, False)]
    assert calcs[0].use_graph and not calcs[1].use_graph
    g = torch.Generator().manual_seed(5)
    p = pos.clone()
    for step in range(4):
        graph, eager = (c.compute(p.to(DEV), cell, types) for c in calcs)
        for k in ("forces", "atomic_energy"):
            assert _rel(graph[k], eager[k]) < 1e-12, (step, k, _rel(graph[k], eager[k]))
        p = p + 0.1 * torch.randn(p.shape, generator=g, dtype=p.dtype)
    assert calcs[0].n_evaluations == 4


LMAX_GOLDEN = {r["name"]: r for r in load_sharded("ref_models_lmax")}


@pytest.mark.parametrize("name", list(LMAX_GOLDEN))
def test_cuda_model_reproduces_reference(name):
    """The reference builder's own l_max 0 and 4 models (tests/golden/make_lmax_vectors.py): energies and forces to 1e-9."""
    from allegro_b200.model import AllegroModel

    rec = LMAX_GOLDEN[name]
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    out = model.to(DEV)(_to_dev(rec["data"]))
    assert _rel(out[D.PER_ATOM_ENERGY_KEY], rec["atomic_energy"]) < TOL
    assert _rel(out[D.FORCE_KEY], rec["forces"]) < TOL
    assert _rel(out[D.EDGE_ENERGY_KEY], rec["edge_energy"]) < TOL
    assert abs(float(out[D.TOTAL_ENERGY_KEY]) - float(rec["total_energy"])) < TOL * float(rec["atomic_energy"].abs().sum())
