"""Committees of models on the GPU (allegro_b200.committee).

1. The statistics kernels against their torch restatement (tests/committee_spec.py): ab2_committee_moments bitwise at
   K = 1, 2, 3, 16, G = 1, 3, fp32 and fp64, up to 10^6 elements; ab2_frame_extrema on a ragged batch with empty frames,
   frames at the chunk edges and a 120 000-atom frame (max / min exact, mean to rounding); launches are reproducible.
2. A committee of one member gives the member's own outputs bitwise and zero deviations.
3. A mixed committee (two seeds of one small architecture, and an l_max = 1 model of other widths with a ZBL pair term and
   a smaller r_max) on a periodic frame and on batches with molecules, triclinic cells and an empty frame: bitwise the
   restatement applied to the outputs the members gave the committee, and the fp64 oracle's statistics to 1e-9 (fp64) /
   1e-4 (fp32).
4. A frame's statistics do not depend on the batch.
5. AllegroCalculator and BatchedCalculator run a committee from one graph, with the statistics' launch count of DESIGN.
6. A list built below a member's r_max is refused."""
import pytest
import torch

import committee_spec
from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.batch import collate
from allegro_b200.committee import STAT_LAUNCHES, STAT_LAUNCHES_STRESS, Committee
from test_host_committee import assert_stats, reference_stats

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]
R_MAX = 6.0
SMALL = dict(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16,
             scalar_embed_mlp_hidden_layers_width=16, allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=8)
OTHER = dict(l_max=1, r_max=5.0, num_scalar_features=32, num_tensor_features=16, radial_chemical_embed_dim=32,
             scalar_embed_mlp_hidden_layers_width=32, allegro_mlp_hidden_layers_width=32, readout_mlp_hidden_layers_width=16,
             per_type_energy_scales=[0.7, 1.3, 0.9], per_type_energy_shifts=[0.1, -0.2, 0.3],
             pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})
MEAN_KEYS = (D.TOTAL_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.STRESS_KEY, D.VIRIAL_KEY)
DEV_KEYS = (D.ENERGY_STD_KEY, D.ATOMIC_ENERGY_STD_KEY, D.FORCE_DEVIATION_KEY, D.VIRIAL_STD_KEY, D.MAX_FORCE_DEVIATION_KEY,
            D.MIN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0) if a.numel() else 0.0


# --------------------------------------------------------------------------- #
# 1. the kernels
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_committee_moments_kernel(dtype):
    g = torch.Generator().manual_seed(1)
    for K in (1, 2, 3, 16):
        for G in (1, 3):
            for m in (0, 1, 255, 256, 4099, 1_000_000 // G):
                base = torch.randn(m, G, generator=g, dtype=torch.float64)
                xs = [(base + 0.1 * (k + 1) * torch.randn(m, G, generator=g, dtype=torch.float64)).to(dtype) for k in range(K)]
                xd = [x.to(DEV) for x in xs]
                mean, dev = _lib.committee_moments(xd, G)
                assert mean.shape == (m, G) and dev.shape == (m,) and mean.dtype == dtype and dev.dtype == dtype
                rm, rd = committee_spec.committee_moments(xs, G)
                assert torch.equal(mean.cpu(), rm) and torch.equal(dev.cpu(), rd), (K, G, m)
                mean2, dev2 = _lib.committee_moments(xd, G)
                assert torch.equal(mean, mean2) and torch.equal(dev, dev2)
                if K == 1:
                    assert torch.equal(mean, xd[0]) and bool((dev == 0).all())
    x = torch.zeros(10, 3, dtype=dtype, device=DEV)
    with pytest.raises(RuntimeError, match="members"):
        _lib.committee_moments([x] * 17, 3)
    with pytest.raises(RuntimeError):
        _lib.committee_moments([x, x.double() if dtype == torch.float32 else x.float()], 3)


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_frame_extrema_kernel(dtype):
    g = torch.Generator().manual_seed(5)  # the ragged batch of test_gpu_atomic_virial.test_frame_heat_current_kernel
    sizes = torch.tensor([0, 0] + [7] * 2000 + [0] + [int(torch.randint(1, 40, (1,), generator=g)) for _ in range(300)]
                         + [120_000] + [0, 2047, 2048, 2049, 1])
    B, n = sizes.shape[0], int(sizes.sum())
    ptr = torch.cat([torch.zeros(1, dtype=torch.long), sizes.cumsum(0)])
    x = (torch.randn(n, generator=g, dtype=torch.float64).abs() + 0.01).to(dtype)
    fp = ptr.to(DEV, torch.int32)
    out = _lib.frame_extrema(x.to(DEV), fp)
    assert out.shape == (B, 3) and out.dtype == dtype
    assert torch.equal(out, _lib.frame_extrema(x.to(DEV), fp))
    ref = committee_spec.frame_extrema(x, ptr)
    got = out.cpu()
    assert torch.equal(got[:, :2], ref[:, :2])
    seg = torch.repeat_interleave(torch.arange(B), sizes)
    mean64 = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, x.double()) / sizes.clamp(min=1).double()
    if dtype == torch.float64:
        assert bool(((got[:, 2] - mean64).abs() <= 1e-12 * mean64.abs()).all())
    else:  # rounded once from fp64: within half an fp32 ulp of the fp64 mean
        assert bool(((got[:, 2].double() - mean64).abs() <= 0.5 * torch.finfo(torch.float32).eps * mean64.abs() * 1.0001).all())
    assert bool((got[sizes == 0] == 0).all())
    big = int((sizes == 120_000).nonzero()[0, 0])
    for b in (big, 5, B - 2):
        p0, p1 = int(ptr[b]), int(ptr[b + 1])
        alone = _lib.frame_extrema(x[p0:p1].to(DEV), torch.tensor([0, p1 - p0], dtype=torch.int32, device=DEV))
        assert torch.equal(alone[0], out[b])


# --------------------------------------------------------------------------- #
# members and frames
# --------------------------------------------------------------------------- #
class Recorder(torch.nn.Module):
    """a member that keeps the outputs it gave the committee: the fp64 tensor-product backward accumulates with atomics
    (DESIGN §8), so an fp64 member's forces are not bitwise the same from one call to the next, and the committee's
    statistics are held to the outputs it actually received"""

    def __init__(self, member):
        super().__init__()
        self.inner = getattr(member, "model", member)
        self.type_names, self.r_max = self.inner.type_names, self.inner.r_max
        self.last = None

    def energy_and_forces(self, data, stress=False):
        self.last = self.inner.energy_and_forces(data, stress=stress)
        return self.last

    def energy_and_forces_frames(self, data, stress=False):
        self.last = self.inner.energy_and_forces_frames(data, stress=stress)
        return self.last


def _kwargs(seed, **over):
    kw = systems.model_kwargs("c3", 20.0, "float64", seed=seed)
    kw.update(SMALL)
    kw.update(over)
    return kw


def _members(dtype):
    """three members (AllegroModel on the device) and their fp64 oracles"""
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    members, oracles = [], []
    for kw in (_kwargs(31), _kwargs(32), _kwargs(33, **OTHER)):
        oracle = AllegroOracle(**kw)
        m = AllegroModel(**dict(kw, model_dtype="float64" if dtype == torch.float64 else "float32"))
        m.load_state_dict(oracle.state_dict())
        members.append(m.to(DEV))
        oracles.append(oracle)
    return members, oracles


def _periodic(reps=4, seed=1234, shear=False):
    pos, cell, types = systems.make_positions("c3", reps, seed=seed)
    if shear:
        new = cell.clone()
        new[1, 0], new[2, 0], new[2, 1] = 0.3 * cell[0, 0], -0.2 * cell[0, 0], 0.25 * cell[1, 1]
        pos = pos @ torch.linalg.inv(cell) @ new
        cell = new
    return {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types}


def _molecule():
    pos, _, types = systems.make_positions("c3", 2, seed=9)
    return {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: types}


def _empty():
    return {D.POSITIONS_KEY: torch.zeros(0, 3, dtype=torch.float64), D.ATOM_TYPE_KEY: torch.zeros(0, dtype=torch.long)}


def _on(frame, dtype):
    return {k: (v.to(DEV, dtype) if v.is_floating_point() else v.to(DEV)) for k, v in frame.items()}


def _prepared(frame, dtype, radius=R_MAX):
    d = _on(frame, dtype)
    cell = d.get(D.CELL_KEY)
    csr, sv = D.neighbor_csr(d[D.POSITIONS_KEY], radius, cell, (cell is not None,) * 3)
    d[D.CSR_KEY], d[D.EDGE_SHIFT_VEC_KEY] = csr, sv
    return d


def _oracle_outs(oracles, frame, stress):
    d = dict(frame)
    cell = d.get(D.CELL_KEY)
    d[D.EDGE_INDEX_KEY], d[D.EDGE_CELL_SHIFT_KEY] = D.neighbor_list(d[D.POSITIONS_KEY], R_MAX, cell, (cell is not None,) * 3)
    outs = [o(d) for o in oracles]
    if not stress:
        for o in outs:
            o.pop(D.STRESS_KEY, None), o.pop(D.VIRIAL_KEY, None)
    return outs


def _frame_of(out, b, a0, a1):
    """the committee fields of frame b (atoms [a0, a1)) of a batch, in single-frame shapes"""
    res = {}
    for k in (D.TOTAL_ENERGY_KEY, D.ENERGY_STD_KEY, D.MAX_FORCE_DEVIATION_KEY, D.MIN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY,
              D.STRESS_KEY, D.VIRIAL_KEY, D.VIRIAL_STD_KEY):
        if k in out:
            res[k] = out[k][b:b + 1]
    for k in (D.PER_ATOM_ENERGY_KEY, D.ATOMIC_ENERGY_STD_KEY, D.FORCE_KEY, D.FORCE_DEVIATION_KEY):
        res[k] = out[k][a0:a1]
    res[D.COMMITTEE_ENERGY_KEY] = out[D.COMMITTEE_ENERGY_KEY][:, b:b + 1]
    return res


def _spec_of(outs, dtype, frame_ptr):
    """the restated statistics of member outputs"""
    def f(key):
        return [o[key].to(dtype).cpu() for o in outs]

    res = {}
    res[D.TOTAL_ENERGY_KEY], std = committee_spec.committee_moments(f(D.TOTAL_ENERGY_KEY), 1)
    res[D.ENERGY_STD_KEY] = std.view(-1, 1)
    res[D.PER_ATOM_ENERGY_KEY], std = committee_spec.committee_moments(f(D.PER_ATOM_ENERGY_KEY), 1)
    res[D.ATOMIC_ENERGY_STD_KEY] = std.view(-1, 1)
    res[D.FORCE_KEY], res[D.FORCE_DEVIATION_KEY] = committee_spec.committee_moments(f(D.FORCE_KEY), 3)
    ext = committee_spec.frame_extrema(res[D.FORCE_DEVIATION_KEY], frame_ptr.cpu())
    res[D.MAX_FORCE_DEVIATION_KEY], res[D.MIN_FORCE_DEVIATION_KEY], res[D.MEAN_FORCE_DEVIATION_KEY] = ext[:, 0], ext[:, 1], ext[:, 2]
    if all(D.STRESS_KEY in o for o in outs):
        res[D.STRESS_KEY], _ = committee_spec.committee_moments(f(D.STRESS_KEY), 1)
        res[D.VIRIAL_KEY], std = committee_spec.committee_moments(f(D.VIRIAL_KEY), 1)
        res[D.VIRIAL_STD_KEY] = std.view(-1, 3, 3)
    return res


def _against_spec(out, outs, dtype, frame_ptr):
    spec = _spec_of(outs, dtype, frame_ptr)
    for k, v in spec.items():
        got = out[k].cpu()
        assert got.dtype == dtype and got.shape == v.shape, (k, got.dtype, got.shape, v.shape)
        if k == D.MEAN_FORCE_DEVIATION_KEY:
            assert _rel(got, v) < (1e-12 if dtype == torch.float64 else 1e-6), k
        else:
            assert torch.equal(got, v), (k, _rel(got, v))
    assert torch.equal(out[D.COMMITTEE_ENERGY_KEY].cpu(), torch.stack([o[D.TOTAL_ENERGY_KEY].to(dtype).reshape(-1).cpu() for o in outs]))


# --------------------------------------------------------------------------- #
# 2. one member
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_one_member_is_the_member(dtype):
    members, _ = _members(dtype)
    m = Recorder(members[0])
    c = Committee([m])
    d = _prepared(_periodic(), dtype)
    b = collate([_on(_periodic(3), dtype), _on(_molecule(), dtype), _on(_empty(), dtype), _on(_periodic(3, seed=7, shear=True), dtype)], R_MAX)
    bs = collate([_on(_periodic(3), dtype), _on(_periodic(3, seed=7, shear=True), dtype)], R_MAX)
    for call in (lambda: c.energy_and_forces(d, stress=True), lambda: c.energy_and_forces_frames(b),
                 lambda: c.energy_and_forces_frames(bs, stress=True)):
        out = call()
        own = m.last
        for k in MEAN_KEYS:
            if k in own:
                assert torch.equal(out[k], own[k].to(dtype)), k
        for k in DEV_KEYS:
            if k in out:
                assert bool((out[k] == 0).all()), k
        assert D.STRESS_KEY not in own or D.VIRIAL_STD_KEY in out


# --------------------------------------------------------------------------- #
# 3. a mixed committee: the restatement and the fp64 oracle
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_mixed_committee(dtype):
    members, oracles = _members(dtype)
    rec = [Recorder(m) for m in members]
    c = Committee(rec)
    assert c.r_max == R_MAX
    tol = 1e-9 if dtype == torch.float64 else 1e-4
    # one periodic frame
    frame = _periodic()
    d = _prepared(frame, dtype)
    n = frame[D.POSITIONS_KEY].shape[0]
    out = c.energy_and_forces(d, stress=True)
    outs = [r.last for r in rec]
    _against_spec(out, outs, dtype, torch.tensor([0, n], dtype=torch.int32))
    ref = reference_stats(_oracle_outs(oracles, frame, True), [n])
    assert_stats(out, ref, tol)
    assert float(out[D.MAX_FORCE_DEVIATION_KEY]) > 0 and float(out[D.ENERGY_STD_KEY]) > 0
    # batches: molecules, triclinic cells, an empty frame (no stress); periodic frames only (stress)
    for frames, stress in (([_periodic(3), _molecule(), _empty(), _periodic(3, seed=7, shear=True), _molecule()], False),
                           ([_periodic(3, seed=8), _periodic(3, seed=7, shear=True)], True)):
        b = collate([_on(f, dtype) for f in frames], R_MAX)
        out = c.energy_and_forces_frames(b, stress=stress)
        outs = [r.last for r in rec]
        sizes = [f[D.POSITIONS_KEY].shape[0] for f in frames]
        fp = torch.tensor([0] + sizes).cumsum(0).to(torch.int32)
        _against_spec(out, outs, dtype, fp)
        for bi, f in enumerate(frames):
            a0, a1 = int(fp[bi]), int(fp[bi + 1])
            got = _frame_of(out, bi, a0, a1)
            if a1 == a0:
                for k in (D.TOTAL_ENERGY_KEY, D.ENERGY_STD_KEY, D.MAX_FORCE_DEVIATION_KEY, D.MIN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY):
                    assert bool((got[k] == 0).all()), k
                continue
            assert_stats(got, reference_stats(_oracle_outs(oracles, f, stress), [a1 - a0]), tol)


# --------------------------------------------------------------------------- #
# 4. batch independence of the statistics
# --------------------------------------------------------------------------- #
def test_statistics_do_not_depend_on_the_batch():
    dtype = torch.float32
    members, _ = _members(dtype)
    rec = [Recorder(m) for m in members]
    c = Committee(rec)
    frames = [_periodic(3), _molecule(), _empty(), _periodic(3, seed=7, shear=True)]
    b = collate([_on(f, dtype) for f in frames], R_MAX)
    out = c.energy_and_forces_frames(b)
    outs = [r.last for r in rec]
    sizes = [f[D.POSITIONS_KEY].shape[0] for f in frames]
    fp = [0]
    for s in sizes:
        fp.append(fp[-1] + s)
    for bi in (0, 1, 3):
        a0, a1 = fp[bi], fp[bi + 1]
        e = [o[D.TOTAL_ENERGY_KEY][bi:bi + 1].contiguous() for o in outs]
        ea = [o[D.PER_ATOM_ENERGY_KEY][a0:a1].contiguous() for o in outs]
        f = [o[D.FORCE_KEY][a0:a1].contiguous() for o in outs]
        te, es = _lib.committee_moments(e, 1)
        ae, aes = _lib.committee_moments(ea, 1)
        fm, sig = _lib.committee_moments(f, 3)
        ext = _lib.frame_extrema(sig, torch.tensor([0, a1 - a0], dtype=torch.int32, device=DEV))
        got = _frame_of(out, bi, a0, a1)
        assert torch.equal(got[D.TOTAL_ENERGY_KEY], te) and torch.equal(got[D.ENERGY_STD_KEY], es.view(-1, 1))
        assert torch.equal(got[D.PER_ATOM_ENERGY_KEY], ae) and torch.equal(got[D.ATOMIC_ENERGY_STD_KEY], aes.view(-1, 1))
        assert torch.equal(got[D.FORCE_KEY], fm) and torch.equal(got[D.FORCE_DEVIATION_KEY], sig)
        assert torch.equal(got[D.MAX_FORCE_DEVIATION_KEY], ext[:, 0]) and torch.equal(got[D.MIN_FORCE_DEVIATION_KEY], ext[:, 1])
        assert torch.equal(got[D.MEAN_FORCE_DEVIATION_KEY], ext[:, 2])


# --------------------------------------------------------------------------- #
# 5. calculators
# --------------------------------------------------------------------------- #
CALC_KEYS = (("energy", D.TOTAL_ENERGY_KEY), ("forces", D.FORCE_KEY), ("stress", D.STRESS_KEY), (D.ENERGY_STD_KEY, D.ENERGY_STD_KEY),
             (D.FORCE_DEVIATION_KEY, D.FORCE_DEVIATION_KEY), (D.MAX_FORCE_DEVIATION_KEY, D.MAX_FORCE_DEVIATION_KEY),
             (D.MEAN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY), (D.VIRIAL_STD_KEY, D.VIRIAL_STD_KEY),
             (D.ATOMIC_ENERGY_STD_KEY, D.ATOMIC_ENERGY_STD_KEY))


def _members_launches(members, data, **kw):
    from allegro_b200.graph import GraphedEnergyForces

    return sum(GraphedEnergyForces(m, data, **kw).launches_per_replay for m in members)


def test_allegro_calculator_trajectory():
    from allegro_b200.calculator import AllegroCalculator

    dtype = torch.float64
    members, _ = _members(dtype)
    c = Committee(members)
    frame = _on(_periodic(), dtype)
    pos, cell, types = frame[D.POSITIONS_KEY], frame[D.CELL_KEY], frame[D.ATOM_TYPE_KEY]
    calc = AllegroCalculator(c, R_MAX, skin=0.5, compute_stress=True)
    g = torch.Generator(device=DEV).manual_seed(9)
    for step in range(12):
        res = {k: v.clone() for k, v in calc.compute(pos, cell, types).items()}
        if step == 0:
            stat = calc._graphed.launches_per_replay - _members_launches(members, calc._graphed.data, stress=True)
            assert stat == STAT_LAUNCHES + STAT_LAUNCHES_STRESS, stat
        ref = c.energy_and_forces(_prepared(frame | {D.POSITIONS_KEY: pos}, dtype), stress=True)
        for key, rk in CALC_KEYS:
            assert _rel(res[key], ref[rk]) < 1e-10, (step, key, _rel(res[key], ref[rk]))
        pos = pos + 0.06 * torch.randn(pos.shape, generator=g, device=DEV, dtype=dtype)
    assert calc.n_rebuilds >= 3


def test_batched_calculator():
    from allegro_b200.calculator import SLOT_REBUILD_LAUNCHES, BatchedCalculator

    dtype = torch.float64
    members, _ = _members(dtype)
    c = Committee(members)
    frames = [_on(f, dtype) for f in (_periodic(3), _molecule(), _empty(), _periodic(3, seed=7, shear=True))]
    calc = BatchedCalculator(c, frames, R_MAX, skin=0.5)
    graphed = calc._graphed
    members_launches = _members_launches(members, graphed.data, frames=True)
    assert graphed.launches_per_replay - members_launches - SLOT_REBUILD_LAUNCHES == STAT_LAUNCHES
    sizes = [f[D.POSITIONS_KEY].shape[0] for f in frames]
    fp = [0]
    for s in sizes:
        fp.append(fp[-1] + s)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames], 0)
    g = torch.Generator(device=DEV).manual_seed(4)
    for step in range(6):
        res = {k: v.clone() for k, v in calc.compute(pos).items()}
        for bi, f in enumerate(frames):
            a0, a1 = fp[bi], fp[bi + 1]
            if a1 == a0:
                continue
            one = c.energy_and_forces(_prepared(f | {D.POSITIONS_KEY: pos[a0:a1]}, dtype))
            assert _rel(res["energy"][bi:bi + 1], one[D.TOTAL_ENERGY_KEY]) < 1e-10
            assert _rel(res["forces"][a0:a1], one[D.FORCE_KEY]) < 1e-10
            assert _rel(res[D.FORCE_DEVIATION_KEY][a0:a1], one[D.FORCE_DEVIATION_KEY]) < 1e-10
            assert _rel(res[D.ENERGY_STD_KEY][bi:bi + 1], one[D.ENERGY_STD_KEY]) < 1e-10
            for k in (D.MAX_FORCE_DEVIATION_KEY, D.MIN_FORCE_DEVIATION_KEY, D.MEAN_FORCE_DEVIATION_KEY):
                assert _rel(res[k][bi:bi + 1], one[k]) < 1e-10, (step, bi, k)
        pos = pos + 0.02 * torch.randn(pos.shape, generator=g, device=DEV, dtype=dtype)
    assert calc.n_captures == 1 and calc.n_overflows == 0 and calc.n_evaluations == 6


def test_calculator_prune_edges():
    from allegro_b200.calculator import AllegroCalculator
    from allegro_b200.model import AllegroModel

    grid = AllegroModel(**_kwargs(41, per_edge_type_cutoff={"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}, model_dtype="float64"))
    plain = AllegroModel(**_kwargs(42, r_max=5.0, model_dtype="float64"))
    c = Committee([grid.to(DEV), plain.to(DEV)])
    frame = _on(_periodic(), torch.float64)
    pos, cell, types = frame[D.POSITIONS_KEY], frame[D.CELL_KEY], frame[D.ATOM_TYPE_KEY]
    pruned, full = AllegroCalculator(c, R_MAX, skin=0.5, prune_edges=True), AllegroCalculator(c, R_MAX, skin=0.5)
    g = torch.Generator(device=DEV).manual_seed(2)
    for step in range(5):
        a = {k: v.clone() for k, v in pruned.compute(pos, cell, types).items()}
        b = {k: v.clone() for k, v in full.compute(pos, cell, types).items()}
        assert pruned.num_edges < full.num_edges
        for key, _ in CALC_KEYS:
            if key in b:
                assert _rel(a[key], b[key]) < 1e-12, (step, key)
        pos = pos + 0.05 * torch.randn(pos.shape, generator=g, device=DEV, dtype=pos.dtype)


# --------------------------------------------------------------------------- #
# 6. a list below a member's r_max
# --------------------------------------------------------------------------- #
def test_short_list_is_refused():
    members, _ = _members(torch.float64)
    c = Committee(members)
    d = _prepared(_periodic(), torch.float64, radius=5.5)
    with pytest.raises(ValueError, match="below the committee's r_max"):
        c.energy_and_forces(d)
    b = collate([_on(_periodic(3), torch.float64)], 5.5)
    with pytest.raises(ValueError, match="below the committee's r_max"):
        c.energy_and_forces_frames(b)
