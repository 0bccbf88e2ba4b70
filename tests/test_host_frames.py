"""Batches of frames on the HOST side, on a CPU-only box: ``energy_and_forces_frames``, ``batch.collate`` / ``split`` and
``data.neighbor_csr_frames``.

The three batch kernels are restated below in torch (what include/allegro_b200.h says ab2_nl_frames_*, ab2_frame_sum and
ab2_frame_virial compute) and monkeypatched over their wrappers together with tests/kernel_spec.py, as in
tests/test_host_pipeline.py.  A batch mixing the reference cases' frames with rotated and translated copies, a frame
without edges, a one-atom frame and a small triclinic cell must give, frame by frame, what the single-frame host path and
the oracle give.  The kernels themselves are checked on the GPU (tests/test_gpu_frames.py).
"""
import math

import pytest
import torch

import kernel_spec
from golden_util import load_models, unpack_state_dict

MODELS = {r["name"]: r for r in load_models()}


# --------------------------------------------------------------------------- #
# restatements of the batch kernels
# --------------------------------------------------------------------------- #
def nl_frames(pos, frame_ptr, cell, inv_cell, pbc, r_max):
    rows, nbrs, shifts = [], [], []
    fp = frame_ptr.long().tolist()
    n = pos.shape[0]
    for b in range(len(fp) - 1):
        a0, a1 = fp[b], fp[b + 1]
        p, c, iv, per = pos[a0:a1], cell[b], inv_cell[b], pbc[b].bool()
        if bool(per.any()):
            img0 = torch.where(per, torch.floor(p @ iv), torch.zeros_like(p)).long()
            w = p - img0.to(p.dtype) @ c
            c64 = c.double()
            heights = [abs(float(torch.det(c64))) / float(torch.linalg.cross(c64[(a + 1) % 3], c64[(a + 2) % 3]).norm()) for a in range(3)]
            reps = [int(math.ceil(r_max / h)) if bool(per[a]) else 0 for a, h in enumerate(heights)]
        else:
            img0, w, reps = torch.zeros(p.shape, dtype=torch.long), p, [0, 0, 0]
        rng = [torch.arange(-r, r + 1) for r in reps]
        S = torch.stack(torch.meshgrid(*rng, indexing="ij"), -1).reshape(-1, 3)        # images in (x, y, z) lexicographic order
        d = w.unsqueeze(0).unsqueeze(2) + (S.to(p.dtype) @ c).view(1, 1, -1, 3) - w.unsqueeze(1).unsqueeze(2)   # [i, j, s, 3]
        mask = d.norm(dim=-1) < r_max
        k0 = int(((S == 0).all(-1)).nonzero()[0, 0])
        mask[torch.arange(a1 - a0), torch.arange(a1 - a0), k0] = False
        ijs = mask.nonzero()                                                            # ordered by (i, j, s)
        raw = S[ijs[:, 2]] - img0[ijs[:, 1]] + img0[ijs[:, 0]]
        rows.append(ijs[:, 0] + a0)
        nbrs.append(ijs[:, 1] + a0)
        shifts.append(raw.to(p.dtype) @ c)
    ctr = torch.cat(rows)
    row_ptr = torch.zeros(n + 1, dtype=torch.int32)
    row_ptr[1:] = torch.cumsum(torch.bincount(ctr, minlength=n), 0).to(torch.int32)
    return row_ptr, torch.cat(nbrs).to(torch.int32), torch.cat(shifts).to(pos.dtype).contiguous()


def frame_sum(x, frame_ptr):
    fp = frame_ptr.long().tolist()
    return torch.stack([x[fp[b]:fp[b + 1]].double().sum() for b in range(len(fp) - 1)]).to(x.dtype)


def frame_virial(vec, gvec, frame_ptr, row_ptr):
    e = row_ptr.long()[frame_ptr.long()].tolist()
    return torch.stack([vec[e[b]:e[b + 1]].double().T @ gvec[e[b]:e[b + 1]].double() for b in range(len(e) - 1)]).to(vec.dtype)


BATCH_SPEC = {"nl_frames": nl_frames, "frame_sum": frame_sum, "frame_virial": frame_virial}


@pytest.fixture()
def spec_kernels(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    for name, fn in BATCH_SPEC.items():
        monkeypatch.setattr(_lib, name, fn)
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    if b.numel() == 0:
        return 0.0
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _rotation(g):
    q, r = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    return q if float(torch.det(q)) > 0 else -q


def _frame(pos, types, r_max, cell=None, pbc=(True, True, True)):
    from allegro_b200 import data as D

    f = {D.POSITIONS_KEY: pos, D.ATOM_TYPE_KEY: types}
    if cell is not None:
        f[D.CELL_KEY], f[D.PBC_KEY] = cell, torch.tensor(pbc)
        ei, sh = D.neighbor_list(pos, r_max, cell, pbc, method="brute")
        f[D.EDGE_INDEX_KEY], f[D.EDGE_CELL_SHIFT_KEY] = ei, sh
    else:
        f[D.EDGE_INDEX_KEY] = D.neighbor_list(pos, r_max, None, (False,) * 3, method="brute")[0]
    return f


def _small_triclinic(r_max, ntypes, g):
    """4 atoms in a skewed cell about 0.9 r_max high: several images per axis, self-image edges."""
    cell = torch.tensor([[0.95, 0.0, 0.0], [0.35, 0.9, 0.0], [-0.2, 0.25, 1.0]], dtype=torch.float64) * r_max
    pos = torch.rand(4, 3, generator=g, dtype=torch.float64) @ cell + torch.tensor([0.0, -1.5, 2.0], dtype=torch.float64) * cell[0]
    return _frame(pos, torch.randint(0, ntypes, (4,), generator=g), r_max, cell)


def _mixed_frames(d, r_max, ntypes, seed, periodic_only=False):
    """The case's frame, a rotated and a translated copy, a small triclinic cell; unless ``periodic_only`` also a frame without
    edges and a one-atom frame (no cell)."""
    from allegro_b200 import data as D

    g = torch.Generator().manual_seed(seed)
    f0 = {k: d[k] for k in (D.POSITIONS_KEY, D.ATOM_TYPE_KEY, D.EDGE_INDEX_KEY, D.CELL_KEY, D.EDGE_CELL_SHIFT_KEY) if k in d}
    R = _rotation(g)
    f1 = dict(f0)
    f1[D.POSITIONS_KEY] = f0[D.POSITIONS_KEY] @ R
    if D.CELL_KEY in f0:
        f1[D.CELL_KEY] = f0[D.CELL_KEY].view(3, 3) @ R
    f2 = dict(f0)
    f2[D.POSITIONS_KEY] = f0[D.POSITIONS_KEY] + torch.tensor([3.1, -7.4, 12.9], dtype=torch.float64)
    frames = [f0, f1, _small_triclinic(r_max, ntypes, g), f2]
    if not periodic_only:
        far = torch.tensor([[0.0, 0.0, 0.0], [2.5 * r_max, 0.3, -0.1]], dtype=torch.float64)
        frames.insert(2, _frame(far, torch.randint(0, ntypes, (2,), generator=g), r_max))
        frames.insert(1, _frame(torch.zeros(1, 3, dtype=torch.float64), torch.zeros(1, dtype=torch.long), r_max))
    return frames


def _models(kw, sd):
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    oracle = AllegroOracle(**kw)
    oracle.load_state_dict(sd, strict=True)
    model = AllegroModel(**kw)
    model.load_state_dict(sd, strict=True)
    return oracle, model.model


def _check_batch(model, oracle, frames, tol, stress, route, r_max):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate, split

    if route == "prepared":
        frames = [{k: v for k, v in f.items() if k not in (D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY)} for f in frames]
        batch = collate(frames, r_max)
        assert D.CSR_KEY in batch
    else:
        batch = collate(frames)
    out = model._energy_and_forces_frames(batch, stress)
    B = len(frames)
    assert out[D.TOTAL_ENERGY_KEY].shape == (B, 1)
    parts = split(out)
    for b, (f, o) in enumerate(zip(frames, split(batch))):
        single = dict(o) if route == "prepared" else f
        one = model._energy_and_forces(single, stress)
        ref_in = dict(f)
        if route == "prepared":  # the oracle takes the same list as edge_index / edge_cell_shift
            csr, sv = o[D.CSR_KEY], o[D.EDGE_SHIFT_VEC_KEY]
            ref_in[D.EDGE_INDEX_KEY] = torch.stack([csr.ctr.long(), csr.nbr.long()])
            if D.CELL_KEY in f:
                ref_in[D.EDGE_CELL_SHIFT_KEY] = torch.round(sv @ torch.linalg.inv(f[D.CELL_KEY].view(3, 3)))
        ref = oracle(ref_in)
        p = parts[b]
        keys = [D.PER_ATOM_ENERGY_KEY, D.FORCE_KEY, D.EDGE_ENERGY_KEY, D.TOTAL_ENERGY_KEY] + ([D.STRESS_KEY, D.VIRIAL_KEY] if stress else [])
        for k in keys + [D.EDGE_FEATURES_KEY]:
            assert _rel(p[k], one[k]) < tol, (b, k, "single", _rel(p[k], one[k]))
        for k in keys:
            scale = float(ref[D.PER_ATOM_ENERGY_KEY].abs().sum()) if k == D.TOTAL_ENERGY_KEY else None
            err = float((p[k].double() - ref[k].double()).abs().max()) / scale if scale else _rel(p[k], ref[k])
            assert err < tol, (b, k, "oracle", err)
    return out


CASES = ["c1_lmax1_L1", "c2_lmax2_L2", "c2_lmax2_L2_f32", "c5_lmax3_L3_5species", "per_edge_type_cutoff", "cluster_open_unsorted",
         "spline_embed_f32", "spline_embed_per_edge_type_cutoff"]


@pytest.mark.parametrize("route", ["edge_index", "prepared"])
@pytest.mark.parametrize("name", CASES)
def test_batched_host_path_equals_single_frames_and_oracle(name, route, spec_kernels):
    rec = MODELS[name]
    kw = rec["kwargs"]
    oracle, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    tol = 1e-10 if kw["model_dtype"] == "float64" else 5e-5
    frames = _mixed_frames(rec["data"], kw["r_max"], len(kw["type_names"]), seed=len(name))
    _check_batch(model, oracle, frames, tol, False, route, kw["r_max"])


@pytest.mark.parametrize("name", ["c2_lmax2_L2", "c2_lmax2_L2_f32", "per_edge_type_cutoff"])
def test_batched_host_stress(name, spec_kernels):
    rec = MODELS[name]
    kw = rec["kwargs"]
    oracle, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    tol = 1e-10 if kw["model_dtype"] == "float64" else 5e-5
    frames = _mixed_frames(rec["data"], kw["r_max"], len(kw["type_names"]), seed=3, periodic_only=True)
    _check_batch(model, oracle, frames, tol, True, "edge_index", kw["r_max"])


@pytest.mark.parametrize("route", ["edge_index", "prepared"])
def test_batched_host_path_with_pair_potential(route, spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200 import systems
    from oracle.model_ref import AllegroOracle

    d = systems.make_system("c3", 2)  # 8 atoms in a 5.4 A cube at r_max 6: two images per side
    kw = systems.model_kwargs("c3", d[D.EDGE_INDEX_KEY].shape[1] / 8, "float64")
    kw.update(num_scalar_features=16, num_tensor_features=8, radial_chemical_embed_dim=16, scalar_embed_mlp_hidden_layers_width=16,
              allegro_mlp_hidden_layers_width=16, readout_mlp_hidden_layers_width=16, per_type_energy_scales=[0.7, 1.3, 0.9],
              per_type_energy_shifts=[0.1, -0.2, 0.3],
              pair_potential={"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["Li", "P", "S"]})
    sd = AllegroOracle(**kw).state_dict()
    oracle, model = _models(kw, sd)
    frames = _mixed_frames(d, 6.0, 3, seed=11)
    _check_batch(model, oracle, frames, 1e-10, False, route, 6.0)
    frames = _mixed_frames(d, 6.0, 3, seed=12, periodic_only=True)
    _check_batch(model, oracle, frames, 1e-10, True, route, 6.0)


# --------------------------------------------------------------------------- #
# neighbour list: the restated search is data.neighbor_list(method="brute") row for row
# --------------------------------------------------------------------------- #
def test_frames_list_rows_are_those_of_the_brute_force_list(spec_kernels):
    from allegro_b200 import data as D

    g = torch.Generator().manual_seed(5)
    r_max = 3.0
    frames = []
    cells = [torch.tensor([[4.0, 0, 0], [1.7, 3.6, 0], [-0.9, 1.1, 3.8]], dtype=torch.float64),   # skewed
             torch.tensor([[2.1, 0, 0], [0, 7.0, 0], [0, 0, 6.5]], dtype=torch.float64),          # narrower than r_max along x
             torch.tensor([[5.0, 0.3, 0], [0, 5.5, 0], [0.4, 0, 6.0]], dtype=torch.float64)]
    pbcs = [(True, True, True), (True, True, True), (True, False, True)]
    for cell, pbc in zip(cells, pbcs):
        pos = torch.rand(9, 3, generator=g, dtype=torch.float64) @ cell
        pos[2] += 3 * cell[0] - 2 * cell[2]  # raw coordinates several cells away
        frames.append((pos, cell, pbc))
    frames.append((torch.rand(7, 3, generator=g, dtype=torch.float64) * 4.0, None, (False,) * 3))  # molecule
    frames.append((torch.rand(1, 3, generator=g, dtype=torch.float64), None, (False,) * 3))       # one atom
    pos = torch.cat([f[0] for f in frames])
    sizes = [f[0].shape[0] for f in frames]
    fp = torch.tensor([0] + sizes).cumsum(0)
    cell = torch.stack([f[1] if f[1] is not None else torch.zeros(3, 3, dtype=torch.float64) for f in frames])
    pbc = torch.tensor([f[2] for f in frames])
    csr, sv = D.neighbor_csr_frames(pos, fp, cell, pbc, r_max)
    for b, (p, c, pb) in enumerate(frames):
        ei, sh = D.neighbor_list(p, r_max, c, pb, method="brute")
        e0, e1 = int(csr.row_ptr[fp[b]]), int(csr.row_ptr[fp[b + 1]])
        assert torch.equal(csr.ctr[e0:e1].long() - fp[b], ei[0]) and torch.equal(csr.nbr[e0:e1].long() - fp[b], ei[1])
        if c is not None:
            assert torch.equal(torch.round(sv[e0:e1] @ torch.linalg.inv(c)), sh)
        else:
            assert bool((sv[e0:e1] == 0).all())


# --------------------------------------------------------------------------- #
# helpers and validation
# --------------------------------------------------------------------------- #
def test_collate_split_round_trip():
    from allegro_b200 import data as D
    from allegro_b200.batch import collate, split

    rec = MODELS["c2_lmax2_L2"]
    frames = _mixed_frames(rec["data"], rec["kwargs"]["r_max"], 1, seed=2)
    batch = collate(frames)
    assert batch[D.BATCH_KEY].shape[0] == batch[D.POSITIONS_KEY].shape[0] and batch[D.NUM_NODES_KEY].shape[0] == len(frames)
    assert batch[D.CELL_KEY].shape == (len(frames), 3, 3)
    back = split(batch)
    for f, o in zip(frames, back):
        for k in (D.POSITIONS_KEY, D.ATOM_TYPE_KEY, D.EDGE_INDEX_KEY):
            assert torch.equal(o[k], f[k].reshape(o[k].shape)), k
        if D.CELL_KEY in f:
            assert torch.equal(o[D.CELL_KEY], f[D.CELL_KEY].view(3, 3)) and torch.equal(o[D.EDGE_CELL_SHIFT_KEY], f[D.EDGE_CELL_SHIFT_KEY])
        else:
            assert bool((o[D.CELL_KEY] == 0).all()) and not bool(o[D.PBC_KEY].any())


def _layout_case():
    rec = MODELS["c2_lmax2_L2"]
    kw = rec["kwargs"]
    _, model = _models(kw, unpack_state_dict(rec["state_dict"]))
    return model, _mixed_frames(rec["data"], kw["r_max"], 1, seed=4, periodic_only=True)


def test_unsorted_batch_is_rejected(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, frames = _layout_case()
    batch = collate(frames)
    b = batch[D.BATCH_KEY].clone()
    b[0], b[-1] = b[-1], b[0]
    batch[D.BATCH_KEY] = b
    with pytest.raises(ValueError, match="non-decreasing"):
        model._energy_and_forces_frames(batch, False)


def test_edge_across_frames_is_rejected(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, frames = _layout_case()
    batch = collate(frames)
    ei = batch[D.EDGE_INDEX_KEY].clone()
    ei[1, 0] = batch[D.POSITIONS_KEY].shape[0] - 1  # the first frame's first edge now ends in the last frame
    batch[D.EDGE_INDEX_KEY] = ei
    with pytest.raises(ValueError, match="two different frames"):
        model._energy_and_forces_frames(batch, False)


def test_num_atoms_must_agree_with_batch(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, frames = _layout_case()
    batch = collate(frames)
    num = batch[D.NUM_NODES_KEY].clone()
    num[0] -= 1
    num[1] += 1
    batch[D.NUM_NODES_KEY] = num
    with pytest.raises(ValueError, match="num_atoms"):
        model._energy_and_forces_frames(batch, False)


def test_mixed_edge_sources_are_rejected():
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    _, frames = _layout_case()
    frames[1] = {k: v for k, v in frames[1].items() if k not in (D.EDGE_INDEX_KEY, D.EDGE_CELL_SHIFT_KEY)}
    with pytest.raises(ValueError, match="edge_index"):
        collate(frames, 5.0)


def test_frame_over_the_cap_is_rejected(spec_kernels):
    from allegro_b200 import data as D

    n = D.FRAMES_MAX_ATOMS + 1
    pos = torch.rand(n + 3, 3, dtype=torch.float64) * 100
    with pytest.raises(ValueError, match="neighbor_csr"):
        D.neighbor_csr_frames(pos, torch.tensor([0, 3, n + 3]), None, None, 4.0)


def test_stress_needs_a_non_singular_cell_on_every_frame(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, frames = _layout_case()
    frames.append(_frame(torch.zeros(1, 3, dtype=torch.float64), torch.zeros(1, dtype=torch.long), 5.0))  # no cell: zero cell
    batch = collate(frames)
    with pytest.raises(ValueError, match="non-singular"):
        model._energy_and_forces_frames(batch, True)
    out = model._energy_and_forces_frames(batch, False)  # without stress the same batch is fine
    assert out[D.TOTAL_ENERGY_KEY].shape == (len(frames), 1)
    batch.pop(D.CELL_KEY)
    batch.pop(D.EDGE_CELL_SHIFT_KEY)
    with pytest.raises(ValueError, match="cell"):
        model._energy_and_forces_frames(batch, True)


def test_single_frame_entry_points_still_reject_batches(spec_kernels):
    from allegro_b200 import data as D
    from allegro_b200.batch import collate

    model, frames = _layout_case()
    batch = collate(frames)
    with pytest.raises(NotImplementedError, match="batched"):
        model._energy_and_forces(batch, False)
