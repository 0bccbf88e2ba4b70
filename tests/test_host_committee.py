"""``committee.Committee`` on a CPU-only box: its refusals, the list radii of committees for ``prune_edges``, and its
statistics layer run with the kernels replaced by their torch restatement (tests/committee_spec.py) and with members that
return the fp64 oracle's outputs, against numpy statistics of those outputs.  The restatement's own properties (one
member gives zero deviation; the member order changes nothing beyond an ulp) are checked here too; the kernels are held
to it bit for bit on the GPU (tests/test_gpu_committee.py)."""
import numpy as np
import pytest
import torch

import committee_spec
from allegro_b200 import calculator as C
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.batch import collate, split
from allegro_b200.committee import Committee

TYPES = ["Li", "P", "S"]
GRID_TABLE = {"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}  # tests/test_gpu_prune_model.py
TINY = dict(num_scalar_features=8, num_tensor_features=4, radial_chemical_embed_dim=8, scalar_embed_mlp_hidden_layers_width=8,
            allegro_mlp_hidden_layers_width=8, readout_mlp_hidden_layers_width=8)


class SpecCommittee(Committee):
    _kernels = committee_spec


class OracleMember(torch.nn.Module):
    """A fused member's entry points on the CPU, answered by the fp64 oracle (one frame at a time for a batch)."""

    def __init__(self, **kw):
        super().__init__()
        from oracle.model_ref import AllegroOracle

        self.oracle = AllegroOracle(**kw)
        self.type_names, self.r_max = list(kw["type_names"]), float(kw["r_max"])

    def energy_and_forces(self, data, stress=False):
        d = {k: v for k, v in data.items() if k in (D.POSITIONS_KEY, D.ATOM_TYPE_KEY, D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY, D.CELL_KEY)}
        if D.CELL_KEY in d and not bool(d[D.CELL_KEY].any()):
            d.pop(D.CELL_KEY)  # a molecule of a batch: collate's zero cell
        out = self.oracle(d)
        if not stress:
            out.pop(D.STRESS_KEY, None), out.pop(D.VIRIAL_KEY, None)
        return out

    def energy_and_forces_frames(self, data, stress=False):
        outs = [self.energy_and_forces(f, stress) for f in split(data)]
        res = {k: torch.cat([o[k] for o in outs], 0) for k in (D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.TOTAL_ENERGY_KEY)}
        if stress:
            res[D.STRESS_KEY] = torch.cat([o[D.STRESS_KEY] for o in outs], 0)
            res[D.VIRIAL_KEY] = torch.cat([o[D.VIRIAL_KEY] for o in outs], 0)
        return res


class _Unreached(torch.nn.Module):
    def __init__(self, r_max=5.0, names=TYPES):
        super().__init__()
        self.type_names, self.r_max = list(names), r_max

    def energy_and_forces(self, data, stress=False):
        raise AssertionError("a member was reached")

    energy_and_forces_frames = energy_and_forces


def oracle_kwargs(seed, **over):
    kw = systems.model_kwargs("c3", 20.0, "float64", seed=seed)
    kw.update(TINY)
    kw.update(over)
    return kw


def reference_stats(outs, sizes):
    """numpy statistics of member outputs (dicts of tensors; atoms of frames back to back, ``sizes`` atoms per frame)."""
    def st(key):
        return np.stack([o[key].detach().double().cpu().numpy() for o in outs])

    E, Ea, F = st(D.TOTAL_ENERGY_KEY).reshape(len(outs), -1), st(D.PER_ATOM_ENERGY_KEY), st(D.FORCE_KEY)
    Fm = F.mean(0)
    sigma = np.sqrt(((F - Fm) ** 2).sum(-1).mean(0))
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    ext = np.zeros((len(sizes), 3))
    for b in range(len(sizes)):
        s = sigma[ptr[b]:ptr[b + 1]]
        if s.size:
            ext[b] = s.max(), s.min(), s.mean()
    ref = {D.TOTAL_ENERGY_KEY: E.mean(0).reshape(-1, 1), D.ENERGY_STD_KEY: E.std(0).reshape(-1, 1), D.COMMITTEE_ENERGY_KEY: E,
           D.PER_ATOM_ENERGY_KEY: Ea.mean(0), D.ATOMIC_ENERGY_STD_KEY: Ea.std(0), D.FORCE_KEY: Fm, D.FORCE_DEVIATION_KEY: sigma,
           D.MAX_FORCE_DEVIATION_KEY: ext[:, 0], D.MIN_FORCE_DEVIATION_KEY: ext[:, 1], D.MEAN_FORCE_DEVIATION_KEY: ext[:, 2]}
    if all(D.STRESS_KEY in o for o in outs):
        V = st(D.VIRIAL_KEY)
        ref[D.STRESS_KEY], ref[D.VIRIAL_KEY], ref[D.VIRIAL_STD_KEY] = st(D.STRESS_KEY).mean(0), V.mean(0), V.std(0)
    return ref


def assert_stats(out, ref, tol, scale_of=None):
    """every key of ``ref`` in ``out`` within ``tol`` of the largest |value| of its group (forces / energies / virial)"""
    groups = {D.FORCE_KEY: (D.FORCE_KEY, D.FORCE_DEVIATION_KEY, D.MAX_FORCE_DEVIATION_KEY, D.MIN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY),
              D.PER_ATOM_ENERGY_KEY: (D.PER_ATOM_ENERGY_KEY, D.ATOMIC_ENERGY_STD_KEY),
              D.COMMITTEE_ENERGY_KEY: (D.TOTAL_ENERGY_KEY, D.ENERGY_STD_KEY, D.COMMITTEE_ENERGY_KEY),
              D.VIRIAL_KEY: (D.VIRIAL_KEY, D.VIRIAL_STD_KEY), D.STRESS_KEY: (D.STRESS_KEY,)}
    for head, keys in groups.items():
        if head not in ref:
            continue
        den = max(float(np.abs(ref[head]).max()) if ref[head].size else 0.0, 1e-300)
        for k in keys:
            got = out[k].detach().double().cpu().numpy()
            assert got.shape == ref[k].shape, (k, got.shape, ref[k].shape)
            err = float(np.abs(got - ref[k]).max()) / den if got.size else 0.0
            assert err < tol, (k, err)


# --------------------------------------------------------------------------- #
# refusals
# --------------------------------------------------------------------------- #
def test_construction_refusals():
    with pytest.raises(ValueError, match="at least one"):
        Committee([])
    with pytest.raises(ValueError, match="at most 16"):
        Committee([_Unreached() for _ in range(17)])
    Committee([_Unreached() for _ in range(16)])
    with pytest.raises(ValueError, match="type_names"):
        Committee([_Unreached(), _Unreached(names=["Li", "S", "P"])])
    other = _Unreached()
    other.w = torch.nn.Parameter(torch.zeros(1, device="meta"))
    here = _Unreached()
    here.w = torch.nn.Parameter(torch.zeros(1))
    with pytest.raises(ValueError, match="different devices"):
        Committee([here, other])
    lin = torch.nn.Linear(2, 2)
    lin.type_names, lin.r_max = TYPES, 5.0
    with pytest.raises(TypeError, match="fused"):
        Committee([_Unreached(), lin])
    c = Committee([_Unreached(4.0), _Unreached(6.5)])
    assert c.r_max == 6.5 and not hasattr(c, "model") and len(c.members) == 2


def _csr(n_rows, radius):
    z = torch.zeros(0, dtype=torch.int32)
    return D.EdgeCSR(n_rows, z, z, torch.zeros(n_rows + 1, dtype=torch.int32), None, 0, radius)


@pytest.mark.parametrize("entry", ["energy_and_forces", "energy_and_forces_frames"])
def test_evaluation_refusals(entry):
    c = Committee([_Unreached(4.0), _Unreached(6.0)])
    pos = torch.zeros(5, 3, dtype=torch.float64)
    data = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: torch.zeros(5, dtype=torch.long), D.BATCH_KEY: torch.zeros(5, dtype=torch.long)}
    f = getattr(c, entry)
    with pytest.raises(NotImplementedError):
        f(data, atomic_virial=True)
    with pytest.raises(NotImplementedError):
        f(data, heat_current=True)
    with pytest.raises(ValueError, match="ghost"):
        f(dict(data, **{D.CSR_KEY: _csr(3, 6.5)}))
    with pytest.raises(ValueError, match="below the committee's r_max"):
        f(dict(data, **{D.CSR_KEY: _csr(5, 5.9)}))
    for radius in (None, 6.0):  # no recorded radius (a pruned list), or one at r_max: the members are reached
        with pytest.raises(AssertionError, match="reached"):
            f(dict(data, **{D.CSR_KEY: _csr(5, radius)}))


# --------------------------------------------------------------------------- #
# list radii of a committee
# --------------------------------------------------------------------------- #
def test_prune_table_of_committees():
    from allegro_b200.model import AllegroModel

    grid = AllegroModel(**oracle_kwargs(1, per_edge_type_cutoff=GRID_TABLE))
    other = AllegroModel(**oracle_kwargs(2, per_edge_type_cutoff={"Li": 4.5, "P": 3.0, "S": {"Li": 6.5, "P": 3.0, "S": 3.0}}, r_max=6.5))
    plain5 = AllegroModel(**oracle_kwargs(3, r_max=5.0))
    plain6 = AllegroModel(**oracle_kwargs(4))
    skin = 0.5
    tg, to = C.prune_table(grid, skin), C.prune_table(other, skin)
    assert tg is not None and to is not None
    assert C.prune_table(Committee([plain5, plain6]), skin) is None
    assert torch.equal(C.prune_table(Committee([grid]), skin), tg)
    assert torch.equal(C.prune_table(Committee([grid, other]), skin), torch.maximum(tg, to))
    mixed = C.prune_table(Committee([grid, plain5.model]), skin)
    assert torch.equal(mixed, torch.maximum(tg, torch.full_like(tg, 5.0 + skin)))
    assert float(mixed.min()) == 5.5 and float(mixed.max()) == 6.5
    # AllegroCalculator searches the list at the largest entry
    calc = C.AllegroCalculator(Committee([grid, plain5]), 6.0, skin, prune_edges=True)
    assert calc.r_list == 6.5 and torch.equal(calc._cutoffs, mixed)


# --------------------------------------------------------------------------- #
# the statistics layer with the restated kernels and oracle members
# --------------------------------------------------------------------------- #
def _members():
    return [OracleMember(**oracle_kwargs(11)), OracleMember(**oracle_kwargs(12)),
            OracleMember(**oracle_kwargs(13, l_max=1, num_layers=1, r_max=5.0, per_type_energy_shifts=[0.1, -0.2, 0.3]))]


def _frame(reps, seed, dtype=torch.float64):
    pos, cell, types = systems.make_positions("c3", reps, seed=seed)
    ei, sh = D.neighbor_list(pos, 6.0, cell, (True, True, True))
    return {D.POSITIONS_KEY: pos.to(dtype), D.CELL_KEY: cell.to(dtype), D.ATOM_TYPE_KEY: types, D.EDGE_INDEX_KEY: ei, D.EDGE_CELL_SHIFT_KEY: sh}


def test_single_frame_statistics():
    members = _members()
    c = SpecCommittee(members)
    d = _frame(2, 5)
    n = d[D.POSITIONS_KEY].shape[0]
    for stress in (False, True):
        out = c.energy_and_forces(d, stress=stress)
        outs = [m.energy_and_forces(d, stress) for m in members]
        ref = reference_stats(outs, [n])
        assert (D.VIRIAL_STD_KEY in out) == stress and (D.STRESS_KEY in out) == stress
        assert D.EDGE_ENERGY_KEY not in out and D.EDGE_FEATURES_KEY not in out
        shapes = {D.TOTAL_ENERGY_KEY: (1, 1), D.ENERGY_STD_KEY: (1, 1), D.COMMITTEE_ENERGY_KEY: (3, 1), D.ATOMIC_ENERGY_STD_KEY: (n, 1),
                  D.FORCE_DEVIATION_KEY: (n,), D.MAX_FORCE_DEVIATION_KEY: (1,), D.FORCE_KEY: (n, 3)}
        for k, s in shapes.items():
            assert tuple(out[k].shape) == s, (k, out[k].shape)
        assert_stats(out, ref, 1e-12)
        assert float(out[D.FORCE_DEVIATION_KEY].max()) > 0


def test_batch_statistics():
    members = _members()
    c = SpecCommittee(members)
    frames = [_frame(2, 5), _frame((2, 1, 2), 6), _frame((1, 2, 2), 7)]
    b = collate(frames)
    sizes = [f[D.POSITIONS_KEY].shape[0] for f in frames]
    out = c.energy_and_forces_frames(b, stress=True)
    outs = [m.energy_and_forces_frames(b, True) for m in members]
    ref = reference_stats(outs, sizes)
    assert tuple(out[D.VIRIAL_STD_KEY].shape) == (3, 3, 3) and tuple(out[D.COMMITTEE_ENERGY_KEY].shape) == (3, 3)
    assert tuple(out[D.MEAN_FORCE_DEVIATION_KEY].shape) == (3,) and tuple(out[D.ENERGY_STD_KEY].shape) == (3, 1)
    assert_stats(out, ref, 1e-12)
    # frame by frame: the single-frame committee gives the batch's rows
    a0 = 0
    for bi, f in enumerate(frames):
        one = c.energy_and_forces(f, stress=True)
        a1 = a0 + sizes[bi]
        assert torch.allclose(one[D.FORCE_DEVIATION_KEY], out[D.FORCE_DEVIATION_KEY][a0:a1], rtol=1e-12, atol=0)
        assert torch.allclose(one[D.MAX_FORCE_DEVIATION_KEY], out[D.MAX_FORCE_DEVIATION_KEY][bi:bi + 1], rtol=1e-12, atol=0)
        assert torch.allclose(one[D.VIRIAL_STD_KEY], out[D.VIRIAL_STD_KEY][bi:bi + 1], rtol=1e-10, atol=1e-14)
        a0 = a1


# --------------------------------------------------------------------------- #
# properties of the restatement
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_spec_one_member_and_member_order(dtype):
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(1000, 3, generator=g, dtype=torch.float64).to(dtype) * (1 + k) for k in range(5)]
    for G in (1, 3):
        mean, dev = committee_spec.committee_moments(xs[:1], G)
        assert torch.equal(mean, xs[0]) and bool((dev == 0).all())
        m1, d1 = committee_spec.committee_moments(xs, G)
        m2, d2 = committee_spec.committee_moments(xs[::-1], G)
        m3, d3 = committee_spec.committee_moments([xs[k] for k in (2, 0, 4, 1, 3)], G)
        eps = torch.finfo(dtype).eps
        # fp32: the fp64 sums differ far below the output's ulp, so the rounded results are within one ulp of each other;
        # fp64: the reordered sums of K terms are within K ulps of the largest term
        big = torch.stack([x.abs().reshape(-1, G) for x in xs]).amax(dim=(0, 2))
        for a, b in ((m1, m2), (m1, m3), (d1, d2), (d1, d3)):
            a, b = a.reshape(big.shape[0], -1), b.reshape(big.shape[0], -1)
            if dtype == torch.float32:
                bound = eps * torch.maximum(a.abs(), b.abs())
            else:
                bound = len(xs) * eps * big.view(-1, 1).expand_as(a)
            assert bool(((a - b).abs() <= bound).all())
        ref = torch.stack([x.double().reshape(-1, G) for x in xs])
        assert torch.allclose(d1.double(), (ref - ref.mean(0)).pow(2).sum(-1).mean(0).sqrt(), rtol=4 * eps, atol=0)
    with pytest.raises(RuntimeError):
        committee_spec.committee_moments([xs[0]] * 17, 1)
