"""Batches of frames on the GPU: the frames neighbour list (ab2_nl_frames_*), the per-frame reductions (ab2_frame_sum /
ab2_frame_virial) and ``energy_and_forces_frames`` frame by frame against the single-frame path and the oracle."""

import pytest
import torch

from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.batch import collate, split

pytestmark = pytest.mark.gpu
DEV = "cuda"


# --------------------------------------------------------------------------- #
# seeded frames
# --------------------------------------------------------------------------- #
def _clear_of_cutoff(pos, cell, pbc, r_max, margin=1e-4):
    """No pair distance within ``margin`` of r_max (fp64): which side of the cutoff a pair falls on is then the same for
    every correctly rounded evaluation in fp32 or fp64, and the lists can be compared row for row."""
    lo = D.neighbor_list(pos, r_max - margin, cell, pbc, method="brute")[0].shape[1]
    hi = D.neighbor_list(pos, r_max + margin, cell, pbc, method="brute")[0].shape[1]
    return lo == hi


def _geometry(kind, g, r_max, n=None):
    """(pos fp64, cell or None, pbc) of one frame of the given kind."""
    n = n if n is not None else int(torch.randint(2, 24, (1,), generator=g))
    if kind == "triclinic":
        cell = torch.tensor([[1.3, 0.0, 0.0], [0.7, 1.1, 0.0], [-0.45, 0.5, 1.2]], dtype=torch.float64) * r_max
        cell = cell * (1 + 0.2 * torch.rand(3, 1, generator=g, dtype=torch.float64))
        pbc = (True, True, True)
    elif kind == "narrow":  # narrower than r_max along y: three images on each side
        cell = torch.diag(torch.tensor([1.6, 0.37, 1.4], dtype=torch.float64)) * r_max
        pbc = (True, True, True)
    elif kind == "mixed_pbc":
        cell = torch.tensor([[1.5, 0.2, 0.0], [0.0, 1.2, 0.0], [0.3, 0.0, 1.8]], dtype=torch.float64) * r_max
        pbc = (True, False, True)
    elif kind == "molecule":
        return torch.rand(n, 3, generator=g, dtype=torch.float64) * 1.5 * r_max, None, (False,) * 3
    elif kind == "isolated":  # no neighbours at all
        return torch.arange(n, dtype=torch.float64).unsqueeze(1).repeat(1, 3) * 1.1 * r_max, None, (False,) * 3
    else:
        raise KeyError(kind)
    pos = torch.rand(n, 3, generator=g, dtype=torch.float64) @ cell
    shifts = torch.randint(-4, 5, (n, 3), generator=g).double()  # raw coordinates several cells outside the home cell
    shifts[:, [not p for p in pbc]] = 0
    return pos + shifts @ cell, cell, pbc


KINDS = ("triclinic", "narrow", "mixed_pbc", "molecule", "isolated")


def _frames(kinds, g, r_max, sizes=None):
    out = []
    for i, kind in enumerate(kinds):
        while True:
            f = _geometry(kind, g, r_max, None if sizes is None else sizes[i])
            if _clear_of_cutoff(*f, r_max):
                break
        out.append(f)
    return out


def _pack(frames, dtype):
    pos = torch.cat([f[0] for f in frames]).to(DEV, dtype)
    fp = torch.tensor([0] + [f[0].shape[0] for f in frames]).cumsum(0)
    cell = torch.stack([f[1] if f[1] is not None else torch.zeros(3, 3, dtype=torch.float64) for f in frames]).to(DEV, dtype)
    pbc = torch.tensor([f[2] for f in frames], device=DEV)
    return pos, fp, cell, pbc


def _amax(t):
    return float(t.max()) if t.numel() else 0.0


def _check_rows(frames, dtype, r_max):
    pos, fp, cell, pbc = _pack(frames, dtype)
    csr, sv = D.neighbor_csr_frames(pos, fp, cell, pbc, r_max)
    assert sv.dtype == dtype and int(csr.row_ptr[-1]) == csr.num_edges
    ctr, nbr, sv, rp = csr.ctr.long().cpu(), csr.nbr.long().cpu(), sv.double().cpu(), csr.row_ptr.long().cpu()
    n_edges = 0
    for b, (p, c, pb) in enumerate(frames):
        ei, sh = D.neighbor_list(p.to(dtype), r_max, None if c is None else c.to(dtype), pb, method="brute")
        e0, e1 = int(rp[fp[b]]), int(rp[fp[b + 1]])
        assert e1 - e0 == ei.shape[1], (b, e1 - e0, ei.shape[1])
        assert torch.equal(ctr[e0:e1] - fp[b], ei[0]) and torch.equal(nbr[e0:e1] - fp[b], ei[1]), b
        if c is not None:
            img = sv[e0:e1] @ torch.linalg.inv(c)
            assert _amax((img - torch.round(img)).abs()) < 1e-3
            assert torch.equal(torch.round(img), sh.double()), b
            # r = pos[nbr] + shift - pos[ctr] on the raw positions stays inside the cutoff
            v = p[ei[1]] + sv[e0:e1] - p[ei[0]]
            assert _amax(v.norm(dim=-1)) < r_max * (1 + 1e-5)
        else:
            assert bool((sv[e0:e1] == 0).all())
        n_edges += e1 - e0
    return n_edges


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_frames_list_equals_brute_force_row_for_row(dtype):
    g = torch.Generator().manual_seed(21)
    kinds = KINDS * 3
    frames = _frames(kinds, g, 4.0)
    frames.insert(4, _frames(["molecule"], g, 4.0, sizes=[1])[0])              # one atom, no cell
    frames.insert(0, _frames(["triclinic"], g, 4.0, sizes=[1])[0])             # one atom in a periodic cell: self images
    assert _check_rows(frames, dtype, 4.0) > 0


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_frames_list_on_a_thousand_frames(dtype):
    g = torch.Generator().manual_seed(22)
    kinds = [KINDS[int(k)] for k in torch.randint(0, len(KINDS), (1000,), generator=g)]
    frames = _frames(kinds, g, 3.5)
    assert _check_rows(frames, dtype, 3.5) > 10000


def test_frames_list_does_not_depend_on_the_other_frames():
    g = torch.Generator().manual_seed(23)
    frames = _frames(KINDS, g, 4.0)
    pos, fp, cell, pbc = _pack(frames, torch.float64)
    csr, sv = D.neighbor_csr_frames(pos, fp, cell, pbc, 4.0)
    pos1, fp1, cell1, pbc1 = _pack(frames[:1], torch.float64)
    csr1, sv1 = D.neighbor_csr_frames(pos1, fp1, cell1, pbc1, 4.0)
    e1 = csr1.num_edges
    assert torch.equal(csr.nbr[:e1], csr1.nbr) and torch.equal(sv[:e1], sv1)


# --------------------------------------------------------------------------- #
# per-frame reductions
# --------------------------------------------------------------------------- #
def _ragged_sizes(g):
    """empty frames, thousands of 10-element frames and one c2-sized frame (461 k) inside the batch"""
    sizes = [0, 0] + [10] * 3000 + [0] + [int(torch.randint(1, 40, (1,), generator=g)) for _ in range(500)] + [461_000] + [10] * 1000 + [0, 2047, 2048, 2049]
    return torch.tensor(sizes)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_frame_sum_and_virial_against_fp64(dtype):
    g = torch.Generator(device="cpu").manual_seed(31)
    sizes = _ragged_sizes(g)
    B = sizes.shape[0]
    total = int(sizes.sum())
    ptr = torch.cat([torch.zeros(1, dtype=torch.long), sizes.cumsum(0)])
    # frame_sum: one value per "atom"
    x = (torch.randn(total, generator=g, dtype=torch.float64) + 0.3).to(dtype)
    fp = ptr.to(DEV, torch.int32)
    xd = x.to(DEV)
    s1 = _lib.frame_sum(xd, fp)
    s2 = _lib.frame_sum(xd, fp)
    assert torch.equal(s1, s2)
    seg = torch.repeat_interleave(torch.arange(B), sizes)
    ref = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, x.double())
    scale = torch.zeros(B, dtype=torch.float64).index_add_(0, seg, x.double().abs())
    tol = 1e-13 if dtype == torch.float64 else 1e-7
    assert bool(((s1.double().cpu() - ref).abs() <= tol * scale.clamp(min=1e-300)).all())
    assert bool((s1.cpu()[sizes == 0] == 0).all()) and not bool(torch.signbit(s1.cpu()[sizes == 0]).any())
    # frame_virial: one "atom" per frame, frame b's edges = sizes[b]
    vec = torch.randn(total, 3, generator=g, dtype=torch.float64).to(dtype)
    gvec = torch.randn(total, 3, generator=g, dtype=torch.float64).to(dtype)
    frame_ptr = torch.arange(B + 1, dtype=torch.int32, device=DEV)
    row_ptr = ptr.to(DEV, torch.int32)
    W1 = _lib.frame_virial(vec.to(DEV), gvec.to(DEV), frame_ptr, row_ptr)
    W2 = _lib.frame_virial(vec.to(DEV), gvec.to(DEV), frame_ptr, row_ptr)
    assert W1.shape == (B, 3, 3) and W1.dtype == dtype and torch.equal(W1, W2)
    outer = (vec.double().unsqueeze(2) * gvec.double().unsqueeze(1)).reshape(total, 9)
    refW = torch.zeros(B, 9, dtype=torch.float64).index_add_(0, seg, outer)
    scaleW = torch.zeros(B, 9, dtype=torch.float64).index_add_(0, seg, outer.abs())
    assert bool(((W1.double().cpu().reshape(B, 9) - refW).abs() <= tol * scaleW.clamp(min=1e-300)).all())
    assert bool((W1.cpu()[sizes == 0] == 0).all())
    # a frame's result does not depend on the rest of the batch: the big frame and a small one alone
    big = int((sizes == 461_000).nonzero()[0, 0])
    for b in (big, 5):
        p0, p1 = int(ptr[b]), int(ptr[b + 1])
        alone = _lib.frame_sum(xd[p0:p1].contiguous(), torch.tensor([0, p1 - p0], dtype=torch.int32, device=DEV))
        assert torch.equal(alone[0], s1[b])
        Wa = _lib.frame_virial(vec[p0:p1].to(DEV), gvec[p0:p1].to(DEV), torch.tensor([0, 1], dtype=torch.int32, device=DEV),
                               torch.tensor([0, p1 - p0], dtype=torch.int32, device=DEV))
        assert torch.equal(Wa[0], W1[b])


# --------------------------------------------------------------------------- #
# the model, frame by frame
# --------------------------------------------------------------------------- #
def _shear_fcc(g, a=3.615):
    pos, cell = systems._lattice(systems._FCC, a, (2, 2, 2), 0.05, g)
    shear = torch.tensor([[1.0, 0.0, 0.0], [0.18, 1.0, 0.0], [-0.12, 0.1, 1.0]], dtype=torch.float64)
    return pos @ shear, cell @ shear


def _cluster(g, n=21, r_min=2.0):
    pts = []
    while len(pts) < n:
        p = (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 5.0
        if all(float((p - q).norm()) > r_min for q in pts):
            pts.append(p)
    return torch.stack(pts)


def _model_frames(name, ntypes, g, periodic_only):
    """Seeded frames from the systems.py primitives for model ``name`` (no neighbour lists)."""
    frames = []

    def add(pos, cell=None):
        f = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: torch.randint(0, ntypes, (pos.shape[0],), generator=g)}
        if cell is not None:
            f[D.CELL_KEY] = cell
        frames.append(f)

    if name == "c1":
        pos, cell = systems._lattice(systems._DIAMOND, 5.431, (2, 2, 2), 0.1, g)
        add(pos, cell)
        add(pos + 2.0 * cell[1] - cell[2] + 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64), cell)
    else:
        pos, cell = systems._lattice(systems._FCC, 3.615 if name == "c2" else 2.9, (2, 2, 2), 0.05, g)
        add(pos, cell)
        add(*_shear_fcc(g, 3.615 if name == "c2" else 2.9))
        add(pos + 0.05 * torch.randn(pos.shape, generator=g, dtype=torch.float64) + cell[0], cell)
    if not periodic_only:
        add(_cluster(g))
        add(torch.tensor([[0.0, 0.0, 0.0]], dtype=torch.float64))
    return frames


def _model(name, dtype):
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    if name == "zbl":
        kw = systems.model_kwargs("c3", 20.0, "float64")
        kw.update(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16, scalar_embed_mlp_hidden_layers_width=16,
                  allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=16, r_max=4.5,
                  per_type_energy_scales=[0.7, 1.3, 0.9], per_type_energy_shifts=[0.1, -0.2, 0.3],
                  pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})
    else:
        kw = systems.model_kwargs(name, 40.0 if name == "c2" else 16.0, "float64")
    oracle = AllegroOracle(**kw)
    kwm = dict(kw)
    kwm["model_dtype"] = dtype
    model = AllegroModel(**kwm)
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to(DEV), kw


def _amax(t):
    return float(t.max()) if t.numel() else 0.0


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    den = float(b.abs().max()) if b.numel() else 0.0
    return _amax((a - b).abs()) / (den if den > 0 else 1.0)


MODELS = [("c2", "float32"), ("c2", "float64"), ("c1", "float64"), ("c1", "float32"), ("zbl", "float64"), ("zbl", "float32")]


@pytest.mark.parametrize("periodic_only", [True, False], ids=["periodic_stress", "mixed"])
@pytest.mark.parametrize("name,dtype", MODELS, ids=[f"{n}-{d}" for n, d in MODELS])
def test_batch_equals_single_frames_and_oracle(name, dtype, periodic_only):
    oracle, model, kw = _model(name, dtype)
    r_max = kw["r_max"]
    g = torch.Generator().manual_seed(41)
    frames = _model_frames(name, len(kw["type_names"]), g, periodic_only)
    stress = periodic_only
    batch = collate([{k: v.to(DEV) for k, v in f.items()} for f in frames], r_max)
    out = model.energy_and_forces_frames(batch, stress=stress)
    assert out[D.TOTAL_ENERGY_KEY].shape == (len(frames), 1)
    fp64 = dtype == "float64"
    mismatched = []
    for b, (f, fin, fo) in enumerate(zip(frames, split(batch), split(out))):
        # the single-frame path on the same rows (offsets removed): the same edge order
        one = model.model.energy_and_forces(fin, stress=stress)
        for k in (D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.EDGE_ENERGY_KEY, D.EDGE_FEATURES_KEY):
            if k == D.FORCE_KEY and fp64:
                # fp64 models run the shape-generic tensor-product backward (tp_bwd_kernel, tp.cu), which adds gGamma and gY
                # with fp64 atomicAdd: the forces of ONE frame evaluated twice differ in the last bits, so batch and single
                # frame cannot agree bitwise either.  Every other output is bitwise (fp32 forces included).
                if _rel(fo[k], one[k]) > 1e-13:
                    mismatched.append((b, k, _rel(fo[k], one[k])))
            elif not torch.equal(fo[k], one[k]):
                mismatched.append((b, k, _rel(fo[k], one[k])))
        for k in (D.TOTAL_ENERGY_KEY,) + ((D.STRESS_KEY, D.VIRIAL_KEY) if stress else ()):
            assert _rel(fo[k], one[k]) <= (1e-12 if fp64 else 1e-6), (b, k, _rel(fo[k], one[k]))
        # the oracle on the same list
        csr, sv = fin[D.CSR_KEY], fin[D.EDGE_SHIFT_VEC_KEY].double().cpu()
        ref_in = {D.POSITIONS_KEY: f[D.POSITIONS_KEY], D.ATOM_TYPE_KEY: f[D.ATOM_TYPE_KEY],
                  D.EDGE_INDEX_KEY: torch.stack([csr.ctr.long(), csr.nbr.long()]).cpu()}
        if D.CELL_KEY in f:
            ref_in[D.CELL_KEY] = f[D.CELL_KEY]
            ref_in[D.EDGE_CELL_SHIFT_KEY] = torch.round(sv @ torch.linalg.inv(f[D.CELL_KEY]))
        ref = oracle(ref_in)
        tol = 1e-9 if fp64 else 1e-4
        for k in (D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY) + ((D.STRESS_KEY,) if stress else ()):
            assert _rel(fo[k], ref[k]) < tol, (b, k, _rel(fo[k], ref[k]))
        e_scale = float(ref[D.PER_ATOM_ENERGY_KEY].abs().sum())
        assert abs(float(fo[D.TOTAL_ENERGY_KEY]) - float(ref[D.TOTAL_ENERGY_KEY])) <= tol * max(e_scale, 1e-30), b
    assert not mismatched, f"batch and single-frame outputs differ: {mismatched}"


@pytest.mark.parametrize("name,dtype", [("c2", "float32"), ("c2", "float64"), ("zbl", "float64")])
def test_prepared_and_edge_index_routes_agree(name, dtype):
    oracle, model, kw = _model(name, dtype)
    g = torch.Generator().manual_seed(42)
    frames = [{k: v.to(DEV) for k, v in f.items()} for f in _model_frames(name, len(kw["type_names"]), g, True)]
    prepared = collate(frames, kw["r_max"])
    with_ei = []
    for f, o in zip(frames, split(prepared)):
        csr, sv = o[D.CSR_KEY], o[D.EDGE_SHIFT_VEC_KEY]
        h = dict(f)
        h[D.EDGE_INDEX_KEY] = torch.stack([csr.ctr.long(), csr.nbr.long()])
        h[D.EDGE_CELL_SHIFT_KEY] = torch.round(sv.double() @ torch.linalg.inv(f[D.CELL_KEY].double())).to(sv.dtype)
        with_ei.append(h)
    a = model.energy_and_forces_frames(prepared, stress=True)
    b = model.energy_and_forces_frames(collate(with_ei), stress=True)
    tol = 1e-12 if dtype == "float64" else 1e-5
    for k in (D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.EDGE_ENERGY_KEY, D.TOTAL_ENERGY_KEY, D.STRESS_KEY):
        assert _rel(a[k], b[k]) < tol, (k, _rel(a[k], b[k]))
    # the cached per-list data is reused on a second call with the same dict
    c = model.energy_and_forces_frames(prepared, stress=True)
    assert torch.equal(c[D.PER_ATOM_ENERGY_KEY], a[D.PER_ATOM_ENERGY_KEY])
    assert _rel(c[D.FORCE_KEY], a[D.FORCE_KEY]) <= (1e-13 if dtype == "float64" else 0.0)  # fp64: see the note above


def test_empty_and_edgeless_batches():
    oracle, model, kw = _model("c2", "float64")
    frames = [{D.POSITIONS_KEY: torch.tensor([[0.0, 0, 0], [9.0, 0, 0]], device=DEV, dtype=torch.float64),
               D.ATOM_TYPE_KEY: torch.zeros(2, dtype=torch.long, device=DEV)},
              {D.POSITIONS_KEY: torch.zeros(1, 3, device=DEV, dtype=torch.float64), D.ATOM_TYPE_KEY: torch.zeros(1, dtype=torch.long, device=DEV)}]
    batch = collate(frames, kw["r_max"])
    assert batch[D.CSR_KEY].num_edges == 0
    out = model.energy_and_forces_frames(batch)
    assert out[D.TOTAL_ENERGY_KEY].shape == (2, 1) and bool((out[D.FORCE_KEY] == 0).all())
