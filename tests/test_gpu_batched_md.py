"""``calculator.BatchedCalculator`` on the GPU: the fixed-slot Verlet lists the ab2_slots_* kernels build inside the
replayed graph, and the energies, forces and stresses evaluated on them.

1. Layout, bitwise: after the first build and after chosen frames move past skin / 2, row_ptr / ctr / nbr / shift /
   col_ptr / col_perm equal the restated layout (tests/slot_spec.py) of ``data.neighbor_csr_frames`` at r_list, and the
   slots of frames that did not move are byte-identical to before; on the mixed small frames, and on a dense 4096-atom
   frame (rows and columns over 256 edges) next to one-atom, empty, 64-atom and triclinic 1176-atom frames.
2. Outputs: frame by frame those of ``collate`` + ``energy_and_forces_frames`` on the exact-r_max list; a frame alone in
   a one-frame calculator gives its in-batch results (bitwise in fp32).
3. A hot velocity-Verlet trajectory: forces at every step match a fresh exact-list evaluation, every frame rebuilds
   exactly when an AllegroCalculator of that frame alone rebuilds, and the graph is captured once.
4. A frame compressed past its slot (a small cluster, or the 4096-atom frame): right forces, one re-capture, the other
   frames unchanged.
5. Launches per replay: the model's plus the rebuild's five."""
import math

import pytest
import torch

import nlist_lattice_cases as LC
import slot_spec
from allegro_b200 import _lib
from allegro_b200 import calculator as C
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.batch import collate
from allegro_b200.model import AllegroModel

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]
SKIN = 0.5


def _model(dtype, name="c1"):
    kw = systems.model_kwargs(name, 16.0, "float64" if dtype == torch.float64 else "float32")
    return AllegroModel(**kw).to(DEV), kw["r_max"], len(kw["type_names"])


def _f(pos, cell=None, pbc=None, ntypes=1, g=None):
    f = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: torch.randint(0, ntypes, (pos.shape[0],), generator=g)}
    if cell is not None:
        f[D.CELL_KEY] = cell
        f[D.PBC_KEY] = torch.tensor(pbc if pbc is not None else (True,) * 3)
    return f


def _cluster(g, n=21, r_min=2.0, half=5.0):
    pts = []
    while len(pts) < n:
        p = (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * half
        if all(float((p - q).norm()) > r_min for q in pts):
            pts.append(p)
    return torch.stack(pts)


def _kind(kind, g, r_max, ntypes):
    if kind == "si":
        pos, cell = systems._lattice(systems._DIAMOND, 5.431, (2, 2, 2), 0.1, g)
        return _f(pos, cell, None, ntypes, g)
    if kind == "fcc_sheared":
        pos, cell = systems._lattice(systems._FCC, 3.615, (2, 2, 2), 0.05, g)
        shear = torch.tensor([[1.0, 0.0, 0.0], [0.18, 1.0, 0.0], [-0.12, 0.1, 1.0]], dtype=torch.float64)
        return _f(pos @ shear, cell @ shear, None, ntypes, g)
    if kind == "hcp":
        pos, cell = LC.hcp(reps=(2, 2, 2), seed=int(torch.randint(0, 1000, (1,), generator=g)))
        return _f(pos, cell, None, ntypes, g)
    if kind == "short_axis":  # periodic axis 0.6 r_max long: several images of every atom, self-image edges
        cell = torch.diag(torch.tensor([1.7 * r_max, 0.6 * r_max, 1.5 * r_max], dtype=torch.float64))
        return _f(torch.rand(10, 3, generator=g, dtype=torch.float64) @ cell, cell, None, ntypes, g)
    if kind == "zero_row_sheet":  # ASE's 2-D cell: periodic in x, y, zero third row
        cell = torch.tensor([[7.0, 0.0, 0.0], [2.0, 6.5, 0.0], [0.0, 0.0, 0.0]], dtype=torch.float64)
        pos = torch.rand(12, 3, generator=g, dtype=torch.float64) * torch.tensor([1.0, 1.0, 0.0], dtype=torch.float64)
        pos = pos @ cell + torch.rand(12, 3, generator=g, dtype=torch.float64) * torch.tensor([0.0, 0.0, 3.0], dtype=torch.float64)
        return _f(pos, cell, (True, True, False), ntypes, g)
    if kind == "cluster":
        return _f(_cluster(g), None, None, ntypes, g)
    if kind == "one_atom":
        return _f(torch.zeros(1, 3, dtype=torch.float64), None, None, ntypes, g)
    if kind == "empty":
        return _f(torch.zeros(0, 3, dtype=torch.float64), None, None, ntypes, g)
    if kind == "dense4096":  # the largest frame, ~340 neighbours per atom: rows and columns longer than 256 edges
        side = (4096 / (340.0 / (4.0 / 3.0 * math.pi * (r_max + SKIN) ** 3))) ** (1.0 / 3.0)
        cell = torch.diag(torch.tensor([side, side, side], dtype=torch.float64))
        return _f(torch.rand(4096, 3, generator=g, dtype=torch.float64) @ cell, cell, None, ntypes, g)
    if kind == "tri1176":  # triclinic, more than 1024 atoms: every thread of the place CTA holds atoms
        pos, cell = systems._lattice(systems._FCC, 3.615, (7, 7, 6), 0.05, g)
        shear = torch.tensor([[1.0, 0.0, 0.0], [0.21, 1.0, 0.0], [-0.15, 0.12, 1.0]], dtype=torch.float64)
        return _f(pos @ shear, cell @ shear, None, ntypes, g)
    raise KeyError(kind)


MIXED = ("si", "fcc_sheared", "hcp", "short_axis", "zero_row_sheet", "cluster", "one_atom", "empty")
# the frame-size limit next to the smallest frames
LARGE = ("dense4096", "one_atom", "empty", "si", "tri1176")


def _frames(kinds, dtype, r_max, ntypes, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in kinds:
        f = _kind(k, g, r_max, ntypes)
        out.append({key: (v.to(DEV, dtype) if v.is_floating_point() else v.to(DEV)) if key != D.PBC_KEY else v for key, v in f.items()})
    return out


def _bytes(t):
    """the bytes of a tensor, flat: a slice [lo * w, hi * w) is entries [lo, hi) of its first dimension, w bytes each"""
    return t.detach().contiguous().view(torch.uint8).reshape(-1).cpu()


def _state(calc):
    csr = calc.csr
    cp, cperm = csr.transposed(calc.num_atoms)
    return csr.row_ptr, csr.ctr, csr.nbr, calc.shift, cp, cperm


def _spec_state(calc, pos):
    fp = torch.tensor(calc._fp_host)
    cell = calc._base.get(D.CELL_KEY)
    pbc = calc._base[D.PBC_KEY].cpu() if cell is not None else torch.zeros(calc.num_frames, 3, dtype=torch.bool)
    csr, sh = D.neighbor_csr_frames(pos, fp, cell, pbc, calc.r_list)
    return slot_spec.layout(csr.row_ptr, csr.nbr, sh, calc._fp_host, calc.slot_ptr.cpu().tolist(), calc.pad), csr


def _check_layout(calc, pos):
    ref, csr = _spec_state(calc, pos)
    for what, got, want in zip(("row_ptr", "ctr", "nbr", "shift", "col_ptr", "col_perm"), _state(calc), ref):
        assert torch.equal(_bytes(got), _bytes(want)), what
    assert calc.real_edges() == csr.num_edges


# (dtype, frames, frames moved together at each step); the large batch moves its 4096-atom frame alone, then a small one
LAYOUT_CASES = ([pytest.param(dt, MIXED, ([0, 3, 5],), id=i) for dt, i in zip(DTYPES, DTYPE_IDS)]
                + [pytest.param(dt, LARGE, ([0], [3]), id="large-" + i) for dt, i in zip(DTYPES, DTYPE_IDS)])


@pytest.mark.parametrize("dtype,kinds,moves", LAYOUT_CASES)
def test_slots_equal_the_spec_and_untouched_frames_keep_their_bytes(dtype, kinds, moves):
    model, r_max, nt = _model(dtype)
    frames = _frames(kinds, dtype, r_max, nt, seed=1)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    _check_layout(calc, pos)
    assert calc.frame_rebuilds() == [1] * len(frames)
    calc.compute(pos)
    fp, sp = calc._fp_host, calc.slot_ptr.cpu().tolist()
    want = [1] * len(frames)
    for moved in moves:  # one atom of each frame past skin / 2
        before = [_bytes(t) for t in _state(calc)]
        for b in moved:
            pos[fp[b]] += torch.tensor([0.3, -0.1, 0.05], dtype=dtype, device=DEV)
            want[b] += 1
        calc.compute(pos)
        torch.cuda.synchronize()
        _check_layout(calc, pos)
        assert calc.frame_rebuilds() == want
        after = [_bytes(t) for t in _state(calc)]
        for b in range(len(frames)):
            if b in moved:
                continue
            for k, (x, y) in enumerate(zip(before, after)):
                per_atom = k in (0, 4)
                lo, hi = (fp[b], fp[b + 1]) if per_atom else (sp[b], sp[b + 1])
                w = x.numel() // ((fp[-1] + 1) if per_atom else sp[-1])
                assert torch.equal(x[lo * w:hi * w], y[lo * w:hi * w]), (b, k)
    assert calc.n_captures == 1


def _exact(model, frames, pos, r_max, stress=False):
    fs, a = [], 0
    for f in frames:
        n = f[D.POSITIONS_KEY].shape[0]
        g = dict(f)
        g[D.POSITIONS_KEY] = pos[a:a + n]
        fs.append(g)
        a += n
    return model.model.energy_and_forces_frames(collate(fs, r_max), stress=stress)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    if b.numel() == 0:
        return 0.0
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _per_frame(res, ref, fp, tol, stress):
    for b in range(len(fp) - 1):
        assert _rel(res["energy"][b], ref[D.TOTAL_ENERGY_KEY][b]) < tol, b
        assert _rel(res["forces"][fp[b]:fp[b + 1]], ref[D.FORCE_KEY][fp[b]:fp[b + 1]]) < tol, b
        if stress:
            assert _rel(res["stress"][b], ref[D.STRESS_KEY][b]) < tol, b


@pytest.mark.parametrize("stress", [False, True], ids=["mixed", "periodic_stress"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_outputs_equal_exact_lists_and_single_frame_calculators(dtype, stress):
    model, r_max, nt = _model(dtype)
    kinds = ("si", "fcc_sheared", "hcp", "short_axis") if stress else MIXED
    frames = _frames(kinds, dtype, r_max, nt, seed=2)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN, compute_stress=stress)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    g = torch.Generator().manual_seed(3)
    pos = pos + (0.1 * torch.randn(pos.shape, generator=g, dtype=torch.float64)).to(DEV, dtype)  # inside the skin
    tol = 1e-9 if dtype == torch.float64 else 1e-4
    res = {k: v.clone() for k, v in calc.compute(pos).items()}
    fp = calc._fp_host
    _per_frame(res, _exact(model, frames, pos, r_max, stress), fp, tol, stress)
    for b, f in enumerate(frames):
        if f[D.POSITIONS_KEY].shape[0] == 0:
            continue
        one = C.BatchedCalculator(model, [f], r_max, skin=SKIN, compute_stress=stress).compute(pos[fp[b]:fp[b + 1]].clone())
        for k in ("energy", "forces", "atomic_energy") + (("stress",) if stress else ()):
            got = one[k]
            want = res[k][b:b + 1] if k in ("energy", "stress") else res[k][fp[b]:fp[b + 1]]
            if dtype == torch.float32:
                assert torch.equal(got, want), (b, k)
            else:
                assert _rel(got, want) < 1e-13, (b, k)


def test_hot_trajectory_rebuilds_like_single_frame_calculators():
    dtype = torch.float64
    model, r_max, nt = _model(dtype)
    kinds = ("si", "fcc_sheared", "hcp", "short_axis", "cluster", "one_atom") * 5 + ("si", "cluster")
    frames = _frames(kinds, dtype, r_max, nt, seed=4)
    B = len(frames)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    singles = [C.AllegroCalculator(model, r_max, skin=SKIN, use_graph=False,
                                   pbc=tuple(bool(x) for x in f[D.PBC_KEY]) if D.PBC_KEY in f else (False,) * 3) for f in frames]
    fp = calc._fp_host
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    g = torch.Generator().manual_seed(5)
    # per-frame temperatures from 300 K to 3000 K: the frames cross skin / 2 at different steps
    mass, dt, kB = 28.0, 1.0, 8.617333e-5
    temps = torch.linspace(300.0, 3000.0, B, dtype=torch.float64)
    per_atom_T = torch.cat([temps[b].repeat(fp[b + 1] - fp[b]) for b in range(B)])
    acc_unit = 9.64853e-3  # eV / (A amu) -> A / fs^2
    vel = (torch.randn(pos.shape, generator=g, dtype=torch.float64) * (kB * per_atom_T / mass * acc_unit).sqrt().unsqueeze(1)).to(DEV)
    forces = calc.compute(pos)["forces"].clone()
    for b, s in enumerate(singles):
        s.compute(pos[fp[b]:fp[b + 1]], frames[b].get(D.CELL_KEY), frames[b][D.ATOM_TYPE_KEY].to(DEV))
    steps_with_rebuild = set()
    for step in range(40):
        vel = vel + 0.5 * dt * forces / mass * acc_unit
        pos = pos + dt * vel
        before = calc.frame_rebuilds()
        res = calc.compute(pos)
        forces = res["forces"].clone()
        after = calc.frame_rebuilds()
        if after != before:
            steps_with_rebuild.add(step)
        ref = _exact(model, frames, pos, r_max)
        assert _rel(forces, ref[D.FORCE_KEY]) < 1e-9, step
        assert _rel(res["energy"], ref[D.TOTAL_ENERGY_KEY]) < 1e-9, step
        for b, s in enumerate(singles):
            s.compute(pos[fp[b]:fp[b + 1]], frames[b].get(D.CELL_KEY))
        assert after == [s.n_rebuilds for s in singles], step
        vel = vel + 0.5 * dt * forces / mass * acc_unit
    final = calc.frame_rebuilds()
    assert len(steps_with_rebuild) >= 5 and len(set(final)) >= 3, (sorted(steps_with_rebuild), final)
    assert calc.n_captures == 1 and calc.n_overflows == 0


# (dtype, frames, the frame compressed, by how much): the cluster to 0.3 of its size, or the periodic 4096-atom frame to
# 0.7 (the gap the compression opens at the cell's faces leaves its list less than 0.7^-3 times longer)
OVERFLOW_CASES = ([pytest.param(dt, MIXED, "cluster", 0.3, id=i) for dt, i in zip(DTYPES, DTYPE_IDS)]
                  + [pytest.param(torch.float32, LARGE, "dense4096", 0.7, id="large-fp32")])


@pytest.mark.parametrize("dtype,kinds,squeezed,factor", OVERFLOW_CASES)
def test_overflow_recaptures_once_and_never_returns_a_stale_force(dtype, kinds, squeezed, factor):
    model, r_max, nt = _model(dtype)
    frames = _frames(kinds, dtype, r_max, nt, seed=6)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    fp, B = calc._fp_host, len(frames)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    first = {k: v.clone() for k, v in calc.compute(pos).items()}
    cap0 = list(calc.capacity)
    c = kinds.index(squeezed)
    p = pos[fp[c]:fp[c + 1]]
    pos[fp[c]:fp[c + 1]] = p.mean(0) + factor * (p - p.mean(0))
    res = calc.compute(pos)
    assert calc.n_overflows == 1 and calc.n_captures == 2 and calc.capacity[c] > cap0[c]
    tol = 1e-9 if dtype == torch.float64 else 1e-4
    ref = _exact(model, frames, pos, r_max)
    _per_frame(res, ref, fp, tol, False)
    for b in range(B):
        if b != c:
            assert _rel(res["forces"][fp[b]:fp[b + 1]], first["forces"][fp[b]:fp[b + 1]]) < tol, b
            assert _rel(res["energy"][b], first["energy"][b]) < tol, b
    _check_layout(calc, pos)
    calc.compute(pos)
    assert calc.n_captures == 2


def test_launches_per_replay_are_the_models_plus_the_rebuilds():
    model, r_max, nt = _model(torch.float32)
    frames = _frames(MIXED, torch.float32, r_max, nt, seed=7)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    n0 = _lib.PROF.launches
    model.model.energy_and_forces_frames(calc._data)
    torch.cuda.synchronize()
    assert calc._graphed.launches_per_replay == (_lib.PROF.launches - n0) + C.SLOT_REBUILD_LAUNCHES
