"""GPU parity tests of the whole path: AllegroModel (fused CUDA pipeline) vs the fp64 CPU oracle
on the same seeded inputs and weights: atomic energies, total energy and forces.

Bar (BASELINE.json north_star): 1e-5 relative for fp64 kernels, 1e-3 for bf16; forces
relative to max|F|.  fp32 is held to 1e-4 (the reference's compile tolerance is 5e-5,
tests/model/test_allegro.py:72-74).
"""
import copy

import pytest
import torch

from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from oracle.model_ref import AllegroOracle

pytestmark = pytest.mark.gpu
DEV = "cuda"

SMALL = dict(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16,
             scalar_embed_mlp_hidden_layers_width=16, allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=8)


def _to_dev(d):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _pair(name, scale, dtype, **over):
    d = systems.make_system(name, scale)
    kw = systems.model_kwargs(name, d[D.EDGE_INDEX_KEY].shape[1] / d[D.POSITIONS_KEY].shape[0], "float64")
    kw.update(over)
    oracle = AllegroOracle(**kw)
    kwm = dict(kw)
    kwm["model_dtype"] = dtype
    model = AllegroModel(**kwm)
    sd = {k: v for k, v in oracle.state_dict().items()}
    model.load_state_dict(sd)
    return oracle, model.to(DEV), d


def _check(oracle, model, d, tol_e, tol_f):
    ref = oracle(d)
    out = model(_to_dev(d))
    e_ref, e = ref[D.PER_ATOM_ENERGY_KEY], out[D.PER_ATOM_ENERGY_KEY].double().cpu()
    f_ref, f = ref[D.FORCE_KEY], out[D.FORCE_KEY].double().cpu()
    n = e_ref.shape[0]
    err_e = (e[:n] - e_ref).abs().max().item() / e_ref.abs().max().item()
    # a frame without edges has no forces at all: then the error is absolute
    err_f = (f[:n] - f_ref).abs().max().item() / (f_ref.abs().max().item() or 1.0)
    # total energy on the scale of what is summed (per-atom energies of mixed sign can cancel in the total)
    err_t = abs(out[D.TOTAL_ENERGY_KEY].double().cpu().item() - ref[D.TOTAL_ENERGY_KEY].item()) / float(e_ref.abs().sum())
    assert err_e < tol_e, f"atomic energy rel err {err_e}"
    assert err_t < tol_e, f"total energy rel err {err_t}"
    assert err_f < tol_f, f"force rel err {err_f}"
    return err_e, err_f


@pytest.mark.parametrize("dtype,tol", [("float64", 1e-9), ("float32", 1e-4)])
def test_c1_si_bulk(dtype, tol):
    """configs[0]: 64-atom Si, l_max=1, 1 layer, 32 features (reference-size plumbing case)."""
    oracle, model, d = _pair("c1", None, dtype)
    _check(oracle, model, d, tol, tol)


@pytest.mark.parametrize("dtype,tol", [("float64", 1e-9), ("float32", 1e-4)])
def test_c2_shape_small(dtype, tol):
    """configs[1] architecture (l_max=2, 2 layers, S=64, U=32) on a 3^3 FCC supercell."""
    oracle, model, d = _pair("c2", 3, dtype)
    _check(oracle, model, d, tol, tol)


def test_c2_shape_generic_kernels_fp32():
    """Same as above with the shape-generic kernels forced (A/B against the fast paths)."""
    from allegro_b200 import _lib

    _lib.set_option("tp_fast", 0)
    _lib.set_option("linear_tc", 0)
    try:
        oracle, model, d = _pair("c2", 3, "float32")
        _check(oracle, model, d, 1e-4, 1e-4)
    finally:
        _lib.set_option("tp_fast", 1)
        _lib.set_option("linear_tc", 1)


def test_autograd_path_matches_direct_path():
    """ForceStressOutput via torch.autograd through the custom Function == the autograd-free
    energy_and_forces pass (both are product paths; the second is the default)."""
    oracle, model, d = _pair("c2", 3, "float64")
    dd = _to_dev(d)
    direct = model(dd)
    model.use_autograd = True
    try:
        _check(oracle, model, d, 1e-9, 1e-9)
        auto = model(dd)
    finally:
        model.use_autograd = False
    assert (direct[D.FORCE_KEY] - auto[D.FORCE_KEY]).abs().max() < 1e-10
    assert (direct[D.PER_ATOM_ENERGY_KEY] - auto[D.PER_ATOM_ENERGY_KEY]).abs().max() < 1e-10


def test_c2_bf16():
    oracle, model, d = _pair("c2", 3, "bfloat16")
    ee, ef = _check(oracle, model, d, 2e-2, 5e-2)
    print("bf16 generic path: rel err E", ee, "F", ef)


def test_c5_lmax3_three_layers_fp64():
    """configs[4] architecture (l_max=3, 3 layers, 5 species) with reduced widths."""
    oracle, model, d = _pair("c5", 2, "float64", **SMALL)
    _check(oracle, model, d, 1e-9, 1e-9)


def test_c3_three_species_fp32():
    oracle, model, d = _pair("c3", 4, "float32", **SMALL)
    _check(oracle, model, d, 1e-4, 1e-4)


@pytest.mark.parametrize("over", [
    dict(tp_path_channel_coupling=False),
    dict(allegro_mlp_hidden_layers_depth=2, scalar_embed_mlp_hidden_layers_depth=2),
    dict(allegro_mlp_nonlinearity=None),
    dict(num_layers=3, l_max=1),
    dict(per_type_energy_scales=[2.5], per_type_energy_shifts=[-1.25]),
])
def test_architecture_grid_fp64(over):
    """tests/model/test_allegro.py:76-117 grid restated: coupling {T,F}, deeper MLPs, linear
    latents, more layers, scale/shift."""
    o = dict(SMALL)
    o.update(over)
    oracle, model, d = _pair("c2", 3, "float64", **o)
    _check(oracle, model, d, 1e-9, 1e-9)


def test_per_edge_type_cutoff_fp64():
    o = dict(SMALL)
    o["per_edge_type_cutoff"] = {"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}
    oracle, model, d = _pair("c3", 4, "float64", **o)
    _check(oracle, model, d, 1e-9, 1e-9)


def test_unsorted_edges_and_edge_outputs():
    oracle, model, d = _pair("c1", None, "float64")
    perm = torch.randperm(d[D.EDGE_INDEX_KEY].shape[1], generator=torch.Generator().manual_seed(0))
    d2 = dict(d)
    d2[D.EDGE_INDEX_KEY] = d[D.EDGE_INDEX_KEY][:, perm].contiguous()
    d2[D.EDGE_CELL_SHIFT_KEY] = d[D.EDGE_CELL_SHIFT_KEY][perm].contiguous()
    _check(oracle, model, d2, 1e-9, 1e-9)
    ref = oracle(d2)
    out = model(_to_dev(d2))
    assert (out[D.EDGE_FEATURES_KEY].cpu() - ref[D.EDGE_FEATURES_KEY]).abs().max() < 1e-9
    assert (out[D.EDGE_ENERGY_KEY].cpu() - ref[D.EDGE_ENERGY_KEY]).abs().max() < 1e-9


def test_ghost_atom_format():
    """pair_allegro data contract (allegro/_compile.py:17-65): ghosts appended, neighbour index >= N_local."""
    oracle, model, d = _pair("c1", None, "float64")
    g = D.to_ghost_format(d)
    n = int(g.pop("num_local_atoms"))
    ref = oracle(d)
    out = model(_to_dev(g))
    assert (out[D.PER_ATOM_ENERGY_KEY][:n].cpu() - ref[D.PER_ATOM_ENERGY_KEY]).abs().max() < 1e-9
    assert out[D.PER_ATOM_ENERGY_KEY][n:].abs().max() == 0  # ghosts own no edges


def test_equivariance_and_fd_forces_on_gpu():
    """Size-independent properties through the CUDA path: rotation equivariance, zero net
    force, forces = -dE/dpos by central differences."""
    from oracle.o3_ref import random_rotation

    _, model, d = _pair("c2", 3, "float64")
    dd = _to_dev(d)
    out = model(dd)
    Rm = (-random_rotation(2)).to(DEV)
    d2 = dict(dd)
    d2[D.POSITIONS_KEY] = dd[D.POSITIONS_KEY] @ Rm.T
    d2[D.CELL_KEY] = dd[D.CELL_KEY] @ Rm.T
    out2 = model(d2)
    assert (out[D.PER_ATOM_ENERGY_KEY] - out2[D.PER_ATOM_ENERGY_KEY]).abs().max() < 1e-9
    assert (out[D.FORCE_KEY] @ Rm.T - out2[D.FORCE_KEY]).abs().max() < 1e-9
    assert out[D.FORCE_KEY].sum(0).abs().max() < 1e-9
    h = 1e-5
    for atom, ax in [(3, 0), (50, 2)]:
        dp, dm = dict(dd), dict(dd)
        pp, pm = dd[D.POSITIONS_KEY].clone(), dd[D.POSITIONS_KEY].clone()
        pp[atom, ax] += h
        pm[atom, ax] -= h
        dp[D.POSITIONS_KEY], dm[D.POSITIONS_KEY] = pp, pm
        fd = -(model(dp)[D.TOTAL_ENERGY_KEY] - model(dm)[D.TOTAL_ENERGY_KEY]).item() / (2 * h)
        assert fd == pytest.approx(out[D.FORCE_KEY][atom, ax].item(), abs=1e-6)


def test_cpu_input_raises():
    _, model, d = _pair("c1", None, "float32")
    with pytest.raises(RuntimeError):
        model(d)
