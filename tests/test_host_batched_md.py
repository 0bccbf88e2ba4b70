"""``calculator.BatchedCalculator`` on a CPU-only box: the fixed-slot layout of its Verlet lists, its host logic with the
rebuild kernels swapped for their torch restatement (tests/slot_spec.py), and its refusals.

* The restated count / place / fill / transpose of a fully flagged batch give, bitwise, ``data.neighbor_csr_frames``'
  rows plus the padding rule (``slot_spec.layout``), on the nlist_cases / nlist_lattice_cases geometries.
* With the restatement in place of the kernels (and of the model's kernels, tests/kernel_spec.py), the calculator's
  energies and forces equal those of a fresh exact-r_max list at every step: after a frame moves past skin / 2 (only that
  frame rebuilds), after small moves (nothing rebuilds), and after a frame outgrows its slot (every slot is re-sized once).
* Every refusal is raised before any kernel is reached.
The kernels themselves are held to the same layout on the GPU (tests/test_gpu_batched_md.py)."""
import bisect
import math

import pytest
import torch

import nlist_cases
import nlist_lattice_cases
import slot_cases
import slot_spec
from golden_util import unpack_state_dict
from test_host_frames import MODELS, _models, _mixed_frames, spec_kernels  # noqa: F401  (spec_kernels is a fixture)
from test_host_frames import nl_frames as spec_nl_frames
from allegro_b200 import _lib
from allegro_b200 import calculator as C
from allegro_b200 import data as D
from allegro_b200.batch import collate, split

DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]
SPEC_MAX_ATOMS = 600  # the torch search holds [n, n, images, 3]: larger frames are left to the GPU test


class _NoKernels:
    """stands in for the rebuild kernels: reaching one fails the test"""

    def __getattr__(self, name):
        raise AssertionError(f"{name} was reached")


class SpecCalculator(C.BatchedCalculator):
    _kernels = slot_spec
    _device = False


class NoLaunchCalculator(C.BatchedCalculator):
    _kernels = _NoKernels()
    _device = False


class _HostModel:
    """the fused model's batch entry point on CPU tensors (its kernels restated by the spec_kernels fixture)"""

    def __init__(self, model):
        self.m = model

    def energy_and_forces_frames(self, data, stress=False):
        return self.m._energy_and_forces_frames(data, stress)


class _Unused:
    def energy_and_forces_frames(self, data, stress=False):
        raise AssertionError("the model was reached")


@pytest.fixture()
def no_device(monkeypatch):
    """_lib.nl_frames restated; any ab2_* entry point reached fails the test"""
    monkeypatch.setattr(_lib, "load", lambda: _NoKernels())
    monkeypatch.setattr(_lib, "nl_frames", spec_nl_frames)


# --------------------------------------------------------------------------- #
# the layout
# --------------------------------------------------------------------------- #
def _geometries():
    out = []
    for c in nlist_cases.cases(False):
        if c.n_centres is None and c.pos.shape[0] <= SPEC_MAX_ATOMS:
            out.append((c.name, c.pos, c.cell if any(c.pbc) else None, c.pbc, c.r_max))
    for c in nlist_lattice_cases.cases(False):
        if c.pos.shape[0] <= SPEC_MAX_ATOMS:
            out.append((c.name, c.pos, c.cell, c.pbc, c.r_max))
    return out


GEOMS = _geometries()


def _cluster(n, radius, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n, 3, generator=g, dtype=torch.float64)
    return v / v.norm(dim=-1, keepdim=True) * radius * torch.rand(n, 1, generator=g, dtype=torch.float64) ** (1 / 3)


def _frame(pos, cell, pbc, dtype, types=None):
    f = {D.POSITIONS_KEY: pos.to(dtype), D.ATOM_TYPE_KEY: torch.zeros(pos.shape[0], dtype=torch.long) if types is None else types}
    if cell is not None:
        f[D.CELL_KEY], f[D.PBC_KEY] = cell.to(dtype), torch.tensor(pbc)
    return f


def _spec_build(frames, r_list, capacity_of):
    """a fully flagged build with the restated kernels -> (frame_ptr, slot_ptr, row_ptr, ctr, nbr, shift, col_ptr, col_perm)"""
    b = collate([{k: v for k, v in f.items()} for f in frames], r_list)
    pos, n, B = b[D.POSITIONS_KEY], b[D.POSITIONS_KEY].shape[0], len(frames)
    fp = torch.tensor([0] + [f[D.POSITIONS_KEY].shape[0] for f in frames]).cumsum(0).to(torch.int32)
    pbc = torch.stack([torch.as_tensor(f.get(D.PBC_KEY, torch.tensor([D.CELL_KEY in f] * 3))).reshape(3) for f in frames])
    cell = b.get(D.CELL_KEY)
    rows, nimg = D.frames_geometry(cell, pbc, r_list, pos.dtype)
    inv = torch.stack([torch.linalg.inv(r) if bool(p.any()) else torch.zeros(3, 3, dtype=torch.float64) for r, p in zip(rows, pbc)])
    geom = (fp, rows.to(pos.dtype), inv.to(pos.dtype), pbc.to(torch.int32), nimg.to(torch.int32))
    flag = torch.ones(B, dtype=torch.int32)
    counts = torch.zeros(n, dtype=torch.int32)
    slot_spec.slots_count(pos, *geom, r_list, flag, counts)
    per_frame = [int(counts[int(fp[i]):int(fp[i + 1])].sum()) for i in range(B)]
    cap = [capacity_of(c) if int(fp[i + 1]) > int(fp[i]) else 0 for i, c in enumerate(per_frame)]
    slot = torch.tensor([0] + cap).cumsum(0).to(torch.int32)
    E = int(slot[-1])
    row_ptr = torch.zeros(n + 1, dtype=torch.int32)
    row_ptr[n] = E
    col_ptr = row_ptr.clone()
    ctr, nbr, col_perm = (torch.full((E,), -1, dtype=torch.int32) for _ in range(3))
    shift = torch.full((E, 3), float("nan"), dtype=pos.dtype)
    overflow, rebuilds, pos_ref = torch.zeros(1, dtype=torch.int32), torch.zeros(B, dtype=torch.int32), torch.zeros_like(pos)
    slot_spec.slots_place(fp, slot, counts, flag, row_ptr, overflow, rebuilds)
    slot_spec.slots_fill(pos, *geom, r_list, flag, row_ptr, 2 * r_list, ctr, nbr, shift, pos_ref)
    slot_spec.slots_transpose(fp, slot, nbr, flag, col_ptr, col_perm, 4096)
    assert int(overflow[0]) == 0 and rebuilds.tolist() == [1] * B and flag.tolist() == [0] * B
    assert torch.equal(pos_ref, pos)
    return b, fp, slot, (row_ptr, ctr, nbr, shift, col_ptr, col_perm), per_frame


def _bitwise(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("name,pos,cell,pbc,r", GEOMS, ids=[g[0] for g in GEOMS])
def test_spec_slots_are_the_frames_list_plus_padding(name, pos, cell, pbc, r, dtype, no_device):
    frames = [_frame(pos, cell, pbc, dtype), _frame(_cluster(9, 1.2 * r, 3), None, (False,) * 3, dtype),
              _frame(torch.zeros(1, 3, dtype=torch.float64), None, (False,) * 3, dtype)]
    b, fp, slot, got, per_frame = _spec_build(frames, r, lambda c: int(math.ceil(C.SLOT_HEADROOM * c)) + C.SLOT_MIN_EDGES)
    csr, shift = b[D.CSR_KEY], b[D.EDGE_SHIFT_VEC_KEY]
    ref = slot_spec.layout(csr.row_ptr, csr.nbr, shift, fp.tolist(), slot.tolist(), 2 * r)
    for what, x, y in zip(("row_ptr", "ctr", "nbr", "shift", "col_ptr", "col_perm"), got, ref):
        assert _bitwise(x, y), what
    row_ptr = got[0]
    for i in range(len(frames)):
        assert int(row_ptr[int(fp[i])]) == int(slot[i]) and int(row_ptr[int(fp[i + 1])]) == int(slot[i + 1])
        assert per_frame[i] == int(csr.row_ptr[int(fp[i + 1])] - csr.row_ptr[int(fp[i])])
    # the transposed list is EdgeCSR.transposed of the padded list
    padded = D.EdgeCSR(row_ptr.shape[0] - 1, got[1], got[2], row_ptr, None, 0)
    cp, cperm = padded.transposed(row_ptr.shape[0] - 1)
    assert torch.equal(cp, got[4]) and torch.equal(cperm, got[5])
    # padding: self-edges 2 r long, and every real edge is within r
    pad = (got[2] == got[1]) & (got[3][:, 0] == torch.tensor(2 * r, dtype=torch.float64).to(dtype)) & (got[3][:, 1:] == 0).all(1)
    assert int(pad.sum()) == int(slot[-1]) - csr.num_edges


def test_slack_is_spread_over_the_atoms():
    assert slot_spec.pad_counts([5, 0, 2], 3, 7 + 8) == [5 + 3, 0 + 3, 2 + 2]
    assert slot_spec.pad_counts([1], 1, 17) == [17]
    assert slot_spec.pad_counts([0, 0, 0, 0], 4, 2) == [1, 1, 0, 0]


# --------------------------------------------------------------------------- #
# the restated place / transpose / check on the synthetic branch cases (tests/slot_cases.py) the GPU kernels are held to
# bitwise: here the restatement itself is held to the contract, written out a second way
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("mode", list(slot_cases.PLACE_SLACK))
def test_spec_place_follows_the_contract(mode):
    c = slot_cases.place_case(mode)
    flag0, rebuilds0 = c["frame_flag"].clone(), c["rebuilds"].clone()
    slot_spec.slots_place(c["frame_ptr"], c["slot_ptr"], c["counts"], c["frame_flag"], c["row_ptr"], c["overflow"], c["rebuilds"])
    fp, sp, counts, row_ptr = c["frame_ptr"].tolist(), c["slot_ptr"].tolist(), c["counts"].tolist(), c["row_ptr"].tolist()
    over = 0
    for b, nb in enumerate(c["sizes"]):
        a0, a1, cap = fp[b], fp[b + 1], sp[b + 1] - sp[b]
        count = sum(counts[a0:a1])
        if int(flag0[b]) != 1:
            assert int(c["frame_flag"][b]) == int(flag0[b]) and int(c["rebuilds"][b]) == int(rebuilds0[b])
            assert row_ptr[a0:a1] == [slot_cases.SENTINEL] * nb, b
            continue
        if count > cap:
            over += 1
            assert int(c["frame_flag"][b]) == 2 and int(c["rebuilds"][b]) == int(rebuilds0[b])
            assert row_ptr[a0:a1] == [slot_cases.SENTINEL] * nb, b
            continue
        assert int(c["frame_flag"][b]) == 1 and int(c["rebuilds"][b]) == int(rebuilds0[b]) + 1
        if nb == 0:
            continue
        # row l holds counts[l] real edges and k // n_b (+ 1 for the first k % n_b atoms) padding edges
        k = cap - count
        ends = row_ptr[a0 + 1:a1] + [sp[b + 1]]
        lens = [e - s for s, e in zip(row_ptr[a0:a1], ends)]
        assert row_ptr[a0] == sp[b] and sum(lens) == cap
        assert lens == [counts[a0 + l] + k // nb + (1 if l < k % nb else 0) for l in range(nb)], b
    assert int(c["overflow"][0]) == over
    assert (over > 0) == (mode == "one_over")


@pytest.mark.parametrize("pattern", slot_cases.TRANSPOSE_PATTERNS)
def test_spec_transpose_is_the_stable_column_sort(pattern):
    c = slot_cases.transpose_case(pattern)
    flag0 = c["frame_flag"].clone()
    slot_spec.slots_transpose(c["frame_ptr"], c["slot_ptr"], c["nbr"], c["frame_flag"], c["col_ptr"], c["col_perm"], c["max_frame_atoms"])
    assert c["frame_flag"].tolist() == [0] * len(c["sizes"])
    fp, sp = c["frame_ptr"].tolist(), c["slot_ptr"].tolist()
    nbr = c["nbr"].tolist()
    for b, nb in enumerate(c["sizes"]):
        s0, s1 = sp[b], sp[b + 1]
        perm, cp = c["col_perm"][s0:s1].tolist(), c["col_ptr"][fp[b]:fp[b + 1]].tolist()
        if int(flag0[b]) != 1:
            assert perm == [slot_cases.SENTINEL] * (s1 - s0) and cp == [slot_cases.SENTINEL] * nb, b
            continue
        # edge ids grouped by neighbour, ascending inside a group; col_ptr[j] = s0 + edges on columns before j
        want = sorted(range(s0, s1), key=lambda z: (nbr[z], z))
        assert perm == want, b
        cols = [nbr[z] for z in want]
        assert cp == [s0 + bisect.bisect_left(cols, fp[b] + j) for j in range(nb)], b


@pytest.mark.parametrize("skin", [0.5, 0.3, 1.0 / 3.0])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_spec_check_flags_only_beyond_half_the_skin(dtype, skin):
    pos, pos_ref, fp, half, want = slot_cases.check_case(dtype, skin)
    # the cases are what they claim: exact single-axis displacements, h and the next value above it
    h = torch.tensor(half, dtype=torch.float64).to(dtype)
    d = (pos - pos_ref).abs().max(dim=1).values
    assert torch.equal(((pos - pos_ref).abs() > 0).sum(1), torch.ones(pos.shape[0], dtype=torch.int64))
    assert torch.equal(d > h, torch.tensor(want[:-1], dtype=torch.bool))
    assert bool((d[torch.tensor(want[:-1]) == 0] <= h).all())
    flag = torch.zeros(fp.shape[0] - 1, dtype=torch.int32)
    slot_spec.slots_check(pos, pos_ref, fp, half, flag)
    assert flag.tolist() == want


# --------------------------------------------------------------------------- #
# the calculator's host logic, kernels restated
# --------------------------------------------------------------------------- #
def _exact(model, frames, pos, r_max, stress=False):
    fs = []
    a = 0
    for f in frames:
        n = f[D.POSITIONS_KEY].shape[0]
        g = dict(f)
        g[D.POSITIONS_KEY] = pos[a:a + n]
        fs.append(g)
        a += n
    return model._energy_and_forces_frames(collate(fs, r_max), stress)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    den = float(b.abs().max()) if b.numel() else 0.0
    return float((a - b).abs().max()) / (den if den > 0 else 1.0) if b.numel() else 0.0


def _agree(res, ref, tol, stress=False):
    assert _rel(res["energy"], ref[D.TOTAL_ENERGY_KEY]) < tol
    assert _rel(res["forces"], ref[D.FORCE_KEY]) < tol
    assert _rel(res["atomic_energy"], ref[D.PER_ATOM_ENERGY_KEY]) < tol
    if stress:
        assert _rel(res["stress"], ref[D.STRESS_KEY]) < tol and _rel(res["virial"], ref[D.VIRIAL_KEY]) < tol


def _md_frames(rec, r_max, ntypes, periodic_only):
    frames = [{k: v for k, v in f.items() if k not in (D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY)}
              for f in _mixed_frames(rec["data"], r_max, ntypes, seed=5, periodic_only=periodic_only)]
    if not periodic_only:
        g = torch.Generator().manual_seed(9)
        frames.append({D.POSITIONS_KEY: _cluster(14, 1.5 * r_max, 4), D.ATOM_TYPE_KEY: torch.randint(0, ntypes, (14,), generator=g)})
    return frames


@pytest.mark.parametrize("stress", [False, True], ids=["energy-forces", "stress"])
def test_host_logic_follows_exact_lists(stress, spec_kernels):
    rec = MODELS["c1_lmax1_L1"]
    kw = rec["kwargs"]
    _, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    r_max, skin, tol = kw["r_max"], 0.5, 1e-10
    frames = _md_frames(rec, r_max, len(kw["type_names"]), periodic_only=stress)
    calc = SpecCalculator(_HostModel(model), frames, r_max, skin=skin, compute_stress=stress)
    B = len(frames)
    fp = calc._fp_host
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    assert calc.frame_rebuilds() == [1] * B and calc.num_edges == sum(calc.capacity)
    _agree(calc.compute(pos), _exact(model, frames, pos, r_max, stress), tol, stress)
    assert calc.frame_rebuilds() == [1] * B
    # frame 1 moves one atom past skin / 2: only frame 1 rebuilds
    pos[fp[1]] += torch.tensor([0.3, 0.0, 0.0], dtype=pos.dtype)
    _agree(calc.compute(pos), _exact(model, frames, pos, r_max, stress), tol, stress)
    assert calc.frame_rebuilds() == [1, 2] + [1] * (B - 2)
    # every atom moves by less than skin / 2: nothing rebuilds, the skin keeps the result exact
    g = torch.Generator().manual_seed(1)
    d = torch.randn(pos.shape, generator=g, dtype=pos.dtype)
    pos = pos + 0.2 * d / d.norm(dim=-1, keepdim=True)
    _agree(calc.compute(pos), _exact(model, frames, pos, r_max, stress), tol, stress)
    assert calc.frame_rebuilds() == [1, 2] + [1] * (B - 2)
    assert calc.n_overflows == 0 and calc.n_captures == 0


def test_host_logic_resizes_on_overflow(spec_kernels):
    rec = MODELS["c1_lmax1_L1"]
    kw = rec["kwargs"]
    _, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    r_max = kw["r_max"]
    frames = _md_frames(rec, r_max, len(kw["type_names"]), periodic_only=False)
    calc = SpecCalculator(_HostModel(model), frames, r_max, skin=0.5)
    fp, B = calc._fp_host, len(frames)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    cap0, E0 = list(calc.capacity), calc.num_edges
    # the cluster (last frame) is compressed to 0.3 of its size: its list outgrows its slot
    c = pos[fp[B - 1]:fp[B]]
    pos[fp[B - 1]:fp[B]] = c.mean(0) + 0.3 * (c - c.mean(0))
    _agree(calc.compute(pos), _exact(model, frames, pos, r_max), 1e-10)
    assert calc.n_overflows == 1 and calc.capacity[-1] > cap0[-1] and calc.num_edges > E0
    assert calc.frame_rebuilds() == [2] * (B - 1) + [2]  # every slot rebuilt once more by the full build
    _agree(calc.compute(pos), _exact(model, frames, pos, r_max), 1e-10)
    assert calc.n_overflows == 1


# --------------------------------------------------------------------------- #
# refusals, before any kernel
# --------------------------------------------------------------------------- #
def _small(dtype=torch.float64):
    cell = torch.eye(3, dtype=torch.float64) * 6.0
    return [_frame(torch.rand(5, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64) * 6.0, cell, (True,) * 3, dtype),
            _frame(_cluster(4, 3.0, 1), None, (False,) * 3, dtype)]


def _refusals():
    r = 5.0
    out = []
    big = _frame(torch.rand(D.FRAMES_MAX_ATOMS + 1, 3, dtype=torch.float64) * 40.0, None, (False,) * 3, torch.float64)
    out.append(("frame-too-large", [big] + _small(), {}, "at most"))
    for what, c in (("nan-cell", torch.tensor([[6.0, 0, 0], [0, float("nan"), 0], [0, 0, 6.0]], dtype=torch.float64)),
                    ("coplanar-cell", torch.tensor([[5.0, 0, 0], [0, 5.0, 0], [5.0, 5.0, 1e-30]], dtype=torch.float64)),
                    ("image-budget", torch.eye(3, dtype=torch.float64) * (0.002 * r))):
        f = _frame(torch.zeros(2, 3, dtype=torch.float64), c, (True,) * 3, torch.float64)
        out.append((what, _small() + [f], {}, "frame 2 "))
    out.append(("stress-without-cell", _small(), {"compute_stress": True}, "non-singular cell"))
    out.append(("no-frame", [], {}, "at least one frame"))
    out.append(("no-atom", [_frame(torch.zeros(0, 3, dtype=torch.float64), None, (False,) * 3, torch.float64)], {}, "at least one atom"))
    bad_types = _small()
    bad_types[0][D.ATOM_TYPE_KEY] = torch.zeros(2, dtype=torch.long)
    out.append(("types-length", bad_types, {}, "atom_types"))
    out.append(("mixed-dtypes", [_small()[0], _small(torch.float32)[1]], {}, "one dtype"))
    out.append(("negative-skin", _small(), {"skin": -0.1}, "skin"))
    return out


REFUSALS = _refusals()


@pytest.mark.parametrize("name,frames,kw,match", REFUSALS, ids=[x[0] for x in REFUSALS])
def test_refused_before_any_kernel(name, frames, kw, match, no_device):
    with pytest.raises(ValueError, match=match):
        NoLaunchCalculator(_Unused(), frames, 5.0, **kw)


def test_cpu_tensors_are_refused(no_device):
    with pytest.raises(ValueError, match="CUDA"):
        C.BatchedCalculator(_Unused(), _small(), 5.0)


def test_model_without_the_batch_path_is_refused(no_device):
    with pytest.raises(TypeError, match="energy_and_forces_frames"):
        NoLaunchCalculator(object(), _small(), 5.0)


def test_compute_refuses_wrong_positions(spec_kernels):
    rec = MODELS["c1_lmax1_L1"]
    kw = rec["kwargs"]
    _, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    frames = _small()
    calc = SpecCalculator(_HostModel(model), frames, kw["r_max"])
    calc._kernels = _NoKernels()
    n = calc.num_atoms
    for bad in (torch.zeros(n - 1, 3, dtype=torch.float64), torch.zeros(n, 2, dtype=torch.float64), torch.zeros(n, 3, dtype=torch.float32),
                torch.zeros(3 * n, dtype=torch.float64), None):
        with pytest.raises(ValueError, match="pos must be"):
            calc.compute(bad)
    assert calc.n_evaluations == 0
