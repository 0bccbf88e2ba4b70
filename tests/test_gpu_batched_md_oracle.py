"""``calculator.BatchedCalculator`` and its rebuild kernels (ab2_slots_*) against references that share no code with them.

A. The kernels called directly on the synthetic branch cases of tests/slot_cases.py, bitwise against their restatement
   (tests/slot_spec.py): place on frames of 1 .. 4096 atoms with slack below / above n_b, none, and one edge short, flags
   0 / 1 / 2 mixed; transpose on frames of 1 .. 4096 atoms between empty frames, with adversarial columns; check at
   exactly skin / 2 and the next representable value above it.
B. Large frames through the calculator: the real edges of every slot against the fp64 pair search of
   tests/nlist_lattice_oracle.py at r_list, padding exactly (ctr, ctr, (pad, 0, 0)) after them; a process whose first
   calculator needs less than 48 KB of transpose histogram still launches a 4096-atom one.
C. Outputs of every frame against the fp64 oracle (oracle/model_ref.py, tests/nonlin_oracle.py) across the model grid, on
   exact r_max lists built by the pair search from the positions the kernels saw: after the first build and after two
   replays in which different frames rebuilt inside the one captured graph; heavy padding (SLOT_HEADROOM = 4) gives the
   same outputs; skin = 0; a 4096-atom frame of the c2-shape fp32 model on a locality sub-sample (oracle/subsample.py).
D. A hot fp32 trajectory: at every step every pair within r_max - band is among the slots' real edges, and the forces of
   every frame that rebuilt equal the oracle's at that step and the step before.
The largest relative error per model, dtype and output is printed ("[batched-oracle]")."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nlist_lattice_oracle as LO
import nlist_oracle as O
import nonlin_oracle as NO
import slot_cases
import slot_spec
import test_gpu_batched_md as BM
from allegro_b200 import _lib
from allegro_b200 import calculator as C
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.model import AllegroModel
from oracle.model_ref import AllegroOracle
from oracle.subsample import ball, local_reference
from test_gpu_model import SMALL, _pair
from test_gpu_prune_model import _kwargs as _prune_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float64, torch.float32]
DTYPE_IDS = ["fp64", "fp32"]
SKIN = BM.SKIN
HERE = os.path.dirname(os.path.abspath(__file__))


# --------------------------------------------------------------------------- #
# A. the rebuild kernels at every branch
# --------------------------------------------------------------------------- #
def _dev(case):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in case.items()}


PLACE_ARGS = ("frame_ptr", "slot_ptr", "counts", "frame_flag", "row_ptr", "overflow", "rebuilds")


@pytest.mark.parametrize("mode", list(slot_cases.PLACE_SLACK))
def test_place_kernel_equals_the_spec(mode):
    ref = slot_cases.place_case(mode, seed=1)
    got = _dev(ref)
    _lib.slots_place(*(got[k] for k in PLACE_ARGS))
    slot_spec.slots_place(*(ref[k] for k in PLACE_ARGS))
    torch.cuda.synchronize()
    for k in ("frame_flag", "row_ptr", "overflow", "rebuilds"):
        assert torch.equal(got[k].cpu(), ref[k]), k
    assert (int(ref["overflow"][0]) > 0) == (mode == "one_over")


TRANSPOSE_ARGS = ("frame_ptr", "slot_ptr", "nbr", "frame_flag", "col_ptr", "col_perm", "max_frame_atoms")


@pytest.mark.parametrize("pattern", slot_cases.TRANSPOSE_PATTERNS)
def test_transpose_kernel_equals_the_stable_sort(pattern):
    ref = slot_cases.transpose_case(pattern, seed=2)
    got = _dev(ref)
    _lib.slots_transpose(*(got[k] for k in TRANSPOSE_ARGS))
    slot_spec.slots_transpose(*(ref[k] for k in TRANSPOSE_ARGS))
    torch.cuda.synchronize()
    for k in ("frame_flag", "col_ptr", "col_perm"):
        assert torch.equal(got[k].cpu(), ref[k]), k
    assert got["frame_flag"].cpu().tolist() == [0] * len(ref["sizes"])


@pytest.mark.parametrize("skin", [0.5, 0.3, 1.0 / 3.0])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_check_kernel_flags_only_beyond_half_the_skin(dtype, skin):
    pos, pos_ref, fp, half, want = slot_cases.check_case(dtype, skin)
    flag = torch.zeros(len(want), dtype=torch.int32, device=DEV)
    _lib.slots_check(pos.to(DEV), pos_ref.to(DEV), fp.to(DEV), half, flag)
    assert flag.cpu().tolist() == want


# --------------------------------------------------------------------------- #
# B. the slots' real edges against the fp64 pair search
# --------------------------------------------------------------------------- #
def _rows_of(frame, dtype):
    """the oracle's lattice rows of a frame: its cell as the kernels saw it (rounded to ``dtype``), open rows completed"""
    cell = frame.get(D.CELL_KEY)
    pbc = [bool(x) for x in frame[D.PBC_KEY]] if D.PBC_KEY in frame else [False] * 3
    return LO.complete(None if cell is None else cell.to(dtype).double().cpu().numpy(), pbc), pbc


def _slot_rows(calc, b):
    """(real (i, j, s) rows of frame b's slot, frame-local; the padding mask) -- every row's padding after its real edges"""
    fp, sp = calc._fp_host, calc.slot_ptr.cpu().tolist()
    s0, s1 = sp[b], sp[b + 1]
    ctr, nbr = calc.csr.ctr[s0:s1].long().cpu(), calc.csr.nbr[s0:s1].long().cpu()
    sh = calc.shift[s0:s1].cpu()
    pad = (nbr == ctr) & (sh[:, 0] == torch.tensor(calc.pad, dtype=sh.dtype)) & (sh[:, 1] == 0) & (sh[:, 2] == 0)
    # no real edge after a padding edge of the same row
    assert not bool((pad[:-1] & ~pad[1:] & (ctr[:-1] == ctr[1:])).any()), b
    return ctr[~pad] - fp[b], nbr[~pad] - fp[b], sh[~pad], pad


def _check_real_edges(calc, b, frame, pos, dtype, r):
    """frame b's real edges equal the fp64 pairs within ``r`` (up to pairs within the rounding band of it)"""
    fp = calc._fp_host
    n = fp[b + 1] - fp[b]
    ctr, nbr, sh, pad = _slot_rows(calc, b)
    if n == 0:
        assert pad.numel() == 0
        return
    rows, pbc = _rows_of(frame, dtype)
    p64 = pos[fp[b]:fp[b + 1]].double().cpu().numpy()
    img, dev = LO.images_of(sh.double().numpy(), rows)
    scale = max(1.0, float(sh.double().abs().max()) if sh.numel() else 1.0)
    assert dev <= (1e-6 if dtype == torch.float32 else 1e-13) * scale, (b, dev)
    got = np.concatenate([ctr.numpy()[:, None], nbr.numpy()[:, None], img], 1)
    band = LO.band_for(p64, rows, r, fp32=dtype == torch.float32)
    ref, dist = LO.pairs(p64, rows, pbc, r, reach=band)
    O.compare(got, ref, dist, r, band, n)


@pytest.mark.parametrize("kinds", [BM.MIXED, BM.LARGE], ids=["mixed", "large"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_real_edges_are_the_fp64_pairs(dtype, kinds):
    model, r_max, nt = BM._model(dtype)
    frames = BM._frames(kinds, dtype, r_max, nt, seed=8)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    if kinds == BM.LARGE:  # the dense frame: rows and columns longer than 256 edges
        ctr, nbr, _, _ = _slot_rows(calc, 0)
        assert int(torch.bincount(ctr).min()) > 256 and int(torch.bincount(nbr).min()) > 256
    for b, f in enumerate(frames):
        _check_real_edges(calc, b, f, pos, dtype, calc.r_list)
    # every frame moved inside its skin except the last one with atoms, which rebuilds alone
    g = torch.Generator().manual_seed(3)
    d = torch.randn(pos.shape, generator=g, dtype=torch.float64)
    pos = pos + (0.2 * d / d.norm(dim=-1, keepdim=True)).to(DEV, dtype)
    last = max(b for b in range(len(frames)) if calc.sizes[b])
    pos[calc._fp_host[last]] += torch.tensor([0.3, 0.0, 0.0], dtype=dtype, device=DEV)
    calc.compute(pos)
    assert calc.frame_rebuilds() == [2 if b == last else 1 for b in range(len(frames))]
    _check_real_edges(calc, last, frames[last], pos, dtype, calc.r_list)
    assert calc.n_captures == 1


_FRESH_PROCESS = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_batched_md as BM
from allegro_b200 import calculator as C
from allegro_b200 import data as D
model, r_max, nt = BM._model(torch.float32)
small = C.BatchedCalculator(model, BM._frames(("si", "one_atom"), torch.float32, r_max, nt, seed=1), r_max)
assert (8 + 1) * 4 * small._max_atoms <= 48 * 1024  # the transpose histogram of ab2_slots_transpose
frames = BM._frames(BM.LARGE, torch.float32, r_max, nt, seed=2)
big = C.BatchedCalculator(model, frames, r_max)
assert big._max_atoms == 4096
pos = torch.cat([f[D.POSITIONS_KEY] for f in frames])
BM._check_layout(big, pos)
print("ok")
"""


def test_small_histogram_first_does_not_stop_a_4096_atom_frame():
    """In a fresh process, a calculator whose transpose histogram fits the default 48 KB launches first; a later one with
    a 4096-atom frame (144 KB) still builds the layout of the spec."""
    code = _FRESH_PROCESS.format(root=os.path.dirname(HERE), tests=HERE)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


# --------------------------------------------------------------------------- #
# C. outputs against the fp64 oracle across the model grid
# --------------------------------------------------------------------------- #
GELU = dict(scalar_embed_mlp_nonlinearity="gelu", allegro_mlp_nonlinearity="gelu", readout_mlp_nonlinearity="gelu")
# fp32 bars: 1e-4, and for l_max = 3 the force bar of tests/test_gpu_fp32_grid.py (TOL_F["lmax3"])
GRID = {
    "c1": dict(tol_f32=(1e-4, 1e-4)),
    "c2_shape": dict(tol_f32=(1e-4, 1e-4)),               # L2_U32 of test_gpu_fp32_grid: composed TP, fused readout
    "three_species_zbl": dict(tol_f32=(1e-4, 1e-4)),      # GRID_TABLE cutoffs, per-type scales and shifts, ZBL
    "spline_hco": dict(tol_f32=(1e-4, 1e-4)),             # spline embedding, asymmetric H/C/O cutoffs
    "lmax3_L3": dict(tol_f32=(1e-4, 2e-4)),               # baked fp64 kernels in fp64, reduced widths
    "gelu": dict(tol_f32=(1e-4, 1e-4)),
}
_ORACLES, _REFS = {}, {}
ERRORS = {}


def _grid_pair(name, dtype):
    """-> (oracle, AllegroModel on the device, r_max, number of types): both from one state dict"""
    dt = "float64" if dtype == torch.float64 else "float32"
    if name in ("c1", "c2_shape", "lmax3_L3"):
        sys_name, scale, over = {"c1": ("c1", 2, {}), "c2_shape": ("c2", 3, {}), "lmax3_L3": ("c5", 2, SMALL)}[name]
        oracle, model, _ = _pair(sys_name, scale, dt, **over)
        cfg = systems.CONFIGS[sys_name]
        return oracle, model, cfg["r_max"], len(cfg["type_names"])
    if name == "gelu":
        kw = systems.model_kwargs("c1", 16.0, "float64")
        kw.update(GELU)
        torch.manual_seed(0)
        oracle = NO.oracle(**kw)
    else:
        kw = _prune_kwargs({"three_species_zbl": "zbl", "spline_hco": "spline"}[name])
        if name == "three_species_zbl":
            kw = dict(kw, per_type_energy_scales=[2.5, 0.5, 1.25])
        oracle = AllegroOracle(**dict(kw, model_dtype="float64"))
    model = AllegroModel(**dict(kw, model_dtype=dt))
    model.load_state_dict(oracle.state_dict())
    return oracle, model.to(DEV), kw["r_max"], len(kw["type_names"])


def _oracle_of(name):
    if name not in _ORACLES:
        _ORACLES[name] = _grid_pair(name, torch.float64)[0]
    return _ORACLES[name]


def _oracle_frame(oracle, frame, pos64, r_max):
    """the fp64 oracle on frame ``frame`` at positions ``pos64`` [n,3] (CPU fp64), on the exact r_max list of the fp64 pair
    search -> {energy, atomic_energy, forces (, stress)}"""
    rows, pbc = _rows_of(frame, torch.float64)
    ref, _ = LO.pairs(pos64.numpy(), rows, pbc, r_max)
    d = {D.POSITIONS_KEY: pos64, D.ATOM_TYPE_KEY: frame[D.ATOM_TYPE_KEY].cpu(),
         D.EDGE_INDEX_KEY: torch.from_numpy(ref[:, :2].T.copy()).long()}
    if any(pbc):
        d[D.CELL_KEY] = torch.from_numpy(rows).double()
        d[D.EDGE_CELL_SHIFT_KEY] = torch.from_numpy(ref[:, 2:].copy()).double()
    out = oracle(d)
    res = {"energy": out[D.TOTAL_ENERGY_KEY].reshape(-1), "atomic_energy": out[D.PER_ATOM_ENERGY_KEY].reshape(-1),
           "forces": out[D.FORCE_KEY]}
    if any(pbc) and D.regular_cells(torch.from_numpy(rows).view(1, 3, 3)).all():
        res["stress"] = out[D.STRESS_KEY].reshape(3, 3)
    return {k: v.detach().double() for k, v in res.items()}


def _errs(got, ref):
    """relative errors of one frame: forces / atomic energies / stress on max |ref|, the energy on sum |E_i|"""
    out = {}
    scale_e = float(ref["atomic_energy"].abs().sum()) or 1.0
    out["energy"] = abs(float(got["energy"]) - float(ref["energy"])) / scale_e
    for k in ("atomic_energy", "forces", "stress"):
        if k in got and k in ref:
            a, b = got[k].double().cpu().reshape(ref[k].shape), ref[k]
            den = float(b.abs().max()) if b.numel() else 0.0
            out[k] = float((a - b).abs().max()) / (den if den > 0 else 1.0) if b.numel() else 0.0
    return out


def _check_frames(tag, name, dtype, calc, res, frames, pos_f32, refs, tol, stress_res=None):
    """every frame of ``calc`` against the oracle values ``refs[b]``; records the largest errors under (name, dtype)"""
    fp = calc._fp_host
    tol_e, tol_f = tol
    bars = {"energy": tol_e, "atomic_energy": tol_e, "forces": tol_f, "stress": tol_f}
    rec = ERRORS.setdefault((name, "fp64" if dtype == torch.float64 else "fp32"), {})
    for b in range(len(frames)):
        a0, a1 = fp[b], fp[b + 1]
        if a1 == a0:
            assert float(res["energy"][b]) == 0.0
            continue
        got = {"energy": res["energy"][b], "atomic_energy": res["atomic_energy"][a0:a1], "forces": res["forces"][a0:a1]}
        if stress_res is not None and b < stress_res["stress"].shape[0]:
            got["stress"] = stress_res["stress"][b]
        for k, e in _errs(got, refs[b]).items():
            rec[k] = max(rec.get(k, 0.0), e)
            assert e < bars[k], (tag, name, b, k, e)


def _refs(name, key, frames, pos64, r_max):
    """oracle values of every frame at the fp32-representable positions ``pos64``, shared by the fp64 and fp32 runs"""
    if (name, key) not in _REFS:
        fp = [0]
        for f in frames:
            fp.append(fp[-1] + f[D.POSITIONS_KEY].shape[0])
        _REFS[(name, key)] = [None if fp[b + 1] == fp[b] else _oracle_frame(_oracle_of(name), frames[b], pos64[fp[b]:fp[b + 1]], r_max)
                              for b in range(len(frames))]
    return _REFS[(name, key)]


def _grid_frames(dtype, r_max, nt, seed):
    """the mixed frames with fp32-representable positions and cells, so one oracle evaluation serves both dtypes"""
    return [{k: (v.to(dtype) if v.is_floating_point() else v) for k, v in f.items()}
            for f in BM._frames(BM.MIXED, torch.float32, r_max, nt, seed)]


PERIODIC = 4  # MIXED[:4]: si, fcc_sheared, hcp, short_axis -- the frames with stress


@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
@pytest.mark.parametrize("name", list(GRID))
def test_outputs_equal_the_oracle_across_rebuilds(name, dtype, monkeypatch):
    oracle, model, r_max, nt = _grid_pair(name, dtype)
    _ORACLES.setdefault(name, oracle)
    tol = (1e-9, 1e-9) if dtype == torch.float64 else GRID[name]["tol_f32"]
    frames = _grid_frames(dtype, r_max, nt, seed=11)
    B, fp = len(frames), [0]
    for f in frames:
        fp.append(fp[-1] + f[D.POSITIONS_KEY].shape[0])
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    per = C.BatchedCalculator(model, frames[:PERIODIC], r_max, skin=SKIN, compute_stress=True)
    p32 = torch.cat([f[D.POSITIONS_KEY] for f in frames]).float().clone()

    def step(p32):
        pos = p32.to(dtype)
        res = {k: v.clone() for k, v in calc.compute(pos).items()}
        sres = {k: v.clone() for k, v in per.compute(pos[:fp[PERIODIC]].clone()).items()}
        return res, sres

    res, sres = step(p32)
    _check_frames("first build", name, dtype, calc, res, frames, p32, _refs(name, "first", frames, p32.double().cpu(), r_max), tol, sres)
    # two replays: frame 0 rebuilds, then frames 2 and 5; every other atom moves inside the skin
    g = torch.Generator().manual_seed(12)
    want = [1] * B
    for moved in ([0], [2, 5]):
        d = torch.randn(p32.shape, generator=g, dtype=torch.float32)
        p32 = p32 + (0.05 * d / d.norm(dim=-1, keepdim=True)).to(DEV)
        for b in moved:
            p32[fp[b]] += torch.tensor([0.3, -0.1, 0.05], device=DEV)
            want[b] += 1
        res, sres = step(p32)
        assert calc.frame_rebuilds() == want
    _check_frames("after rebuilds", name, dtype, calc, res, frames, p32, _refs(name, "moved", frames, p32.double().cpu(), r_max), tol, sres)
    assert calc.n_captures == 1 and per.n_captures == 1 and calc.n_overflows == 0
    # four times the headroom: several times more padding than real edges, the same outputs
    monkeypatch.setattr(C, "SLOT_HEADROOM", 4.0)
    heavy = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    assert heavy.num_edges > 2 * calc.num_edges
    hres = heavy.compute(p32.to(dtype))
    for k in ("energy", "atomic_energy", "forces"):
        assert BM._rel(hres[k], res[k]) < tol[1], k


def test_skin_zero_equals_the_oracle():
    """skin = 0: every move rebuilds the moved frames, and the list is the exact r_max list"""
    name, dtype = "c1", torch.float64
    oracle, model, r_max, nt = _grid_pair(name, dtype)
    frames = _grid_frames(dtype, r_max, nt, seed=11)
    calc = C.BatchedCalculator(model, frames, r_max, skin=0.0)
    p32 = torch.cat([f[D.POSITIONS_KEY] for f in frames]).float().clone()
    res = {k: v.clone() for k, v in calc.compute(p32.double()).items()}
    _check_frames("skin 0", "c1_skin0", dtype, calc, res, frames, p32, _refs(name, "first", frames, p32.double().cpu(), r_max), (1e-9, 1e-9))
    p32[calc._fp_host[0]] += torch.tensor([1e-3, 0.0, 0.0], device=DEV)
    res = calc.compute(p32.double())
    assert calc.frame_rebuilds()[0] == 2 and calc.frame_rebuilds()[1:] == [1] * (len(frames) - 1)
    fp = calc._fp_host
    for b in range(len(frames)):
        if fp[b + 1] > fp[b]:
            _check_real_edges(calc, b, frames[b], p32.double(), dtype, r_max)
    ref = _oracle_frame(oracle, frames[0], p32[fp[0]:fp[1]].double().cpu(), r_max)
    e = _errs({"energy": res["energy"][0], "atomic_energy": res["atomic_energy"][fp[0]:fp[1]], "forces": res["forces"][fp[0]:fp[1]]}, ref)
    assert max(e.values()) < 1e-9, e


def test_4096_atom_frame_c2_shape_fp32_subsample():
    """A 4096-atom Cu frame next to small ones, the c2-shape fp32 model: the locality sub-sample of the oracle for the large
    frame, the whole oracle for the small ones."""
    oracle, model, r_max, nt = _grid_pair("c2_shape", torch.float32)
    g = torch.Generator().manual_seed(13)
    pos, cell = systems._lattice(systems._FCC, 3.615, (8, 8, 16), 0.08, g)
    big = {D.POSITIONS_KEY: pos.float().to(DEV), D.ATOM_TYPE_KEY: torch.zeros(4096, dtype=torch.long).to(DEV),
           D.CELL_KEY: cell.float().to(DEV), D.PBC_KEY: torch.tensor((True,) * 3)}
    frames = [big] + _grid_frames(torch.float32, r_max, nt, seed=14)[5:]  # cluster, one atom, empty
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    p = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    res = {k: v.clone() for k, v in calc.compute(p).items()}
    fp = calc._fp_host
    p64 = p.double().cpu()
    rows, pbc = _rows_of(big, torch.float32)
    ref, _ = LO.pairs(p64[:4096].numpy(), rows, pbc, r_max)
    d = {D.POSITIONS_KEY: p64[:4096], D.ATOM_TYPE_KEY: big[D.ATOM_TYPE_KEY].cpu(), D.CELL_KEY: torch.from_numpy(rows),
         D.EDGE_INDEX_KEY: torch.from_numpy(ref[:, :2].T.copy()).long(), D.EDGE_CELL_SHIFT_KEY: torch.from_numpy(ref[:, 2:].copy()).double()}
    atoms = ball(p64[:4096], 8, seed=0)
    centres, e_ref, f_ref = local_reference(oracle, d, atoms)
    e = res["atomic_energy"][:4096].double().cpu()[centres]
    f = res["forces"][:4096].double().cpu()[atoms]
    err_e = float((e - e_ref).abs().max()) / float(e_ref.abs().max())
    err_f = float((f - f_ref).abs().max()) / float(f_ref.abs().max())
    rec = ERRORS.setdefault(("c2_shape_4096", "fp32"), {})
    rec["atomic_energy"], rec["forces"] = err_e, err_f
    assert err_e < 1e-4 and err_f < 1e-4, (err_e, err_f)
    refs = [None] + [None if fp[b + 1] == fp[b] else _oracle_frame(oracle, frames[b], p64[fp[b]:fp[b + 1]], r_max) for b in range(1, len(frames))]
    small = {k: v for k, v in res.items()}
    for b in range(1, len(frames)):
        if refs[b] is not None:
            got = {"energy": small["energy"][b], "atomic_energy": small["atomic_energy"][fp[b]:fp[b + 1]], "forces": small["forces"][fp[b]:fp[b + 1]]}
            for k, v in _errs(got, refs[b]).items():
                assert v < 1e-4, (b, k, v)


# --------------------------------------------------------------------------- #
# D. never a stale list
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("name", ["c2_shape", "three_species_zbl"])
def test_hot_fp32_trajectory_never_misses_a_pair(name):
    dtype = torch.float32
    _, model, r_max, nt = _grid_pair(name, dtype)
    oracle = _oracle_of(name)
    frames = _grid_frames(dtype, r_max, nt, seed=15)
    calc = C.BatchedCalculator(model, frames, r_max, skin=SKIN)
    fp, B = calc._fp_host, len(frames)
    pos = torch.cat([f[D.POSITIONS_KEY] for f in frames]).clone()
    g = torch.Generator().manual_seed(16)
    mass, dt, kB, acc_unit = 28.0, 1.0, 8.617333e-5, 9.64853e-3
    temps = torch.linspace(600.0, 4000.0, B, dtype=torch.float64)
    per_atom_T = torch.cat([temps[b].repeat(fp[b + 1] - fp[b]) for b in range(B)])
    vel = (torch.randn(pos.shape, generator=g, dtype=torch.float64) * (kB * per_atom_T / mass * acc_unit).sqrt().unsqueeze(1)).to(DEV, dtype)
    forces = calc.compute(pos)["forces"].clone()
    prev_pos, prev_forces = pos.clone(), forces.clone()
    rebuilt_steps, checked = 0, 0
    rec = ERRORS.setdefault((name + "_trajectory", "fp32"), {})
    for step in range(30):
        vel = vel + 0.5 * dt * forces / mass * acc_unit
        pos = pos + dt * vel
        before = calc.frame_rebuilds()
        forces = calc.compute(pos)["forces"].clone()
        after = calc.frame_rebuilds()
        for b in range(B):
            n = fp[b + 1] - fp[b]
            if n == 0:
                continue
            # every pair inside r_max - band at the current positions is a real edge of the slot
            ctr, nbr, sh, _ = _slot_rows(calc, b)
            rows, pbc = _rows_of(frames[b], dtype)
            p64 = pos[fp[b]:fp[b + 1]].double().cpu().numpy()
            img, _ = LO.images_of(sh.double().numpy(), rows)
            band = LO.band_for(p64, rows, r_max, fp32=True)
            ref, dist = LO.pairs(p64, rows, pbc, r_max)
            must = O.keys(ref[dist < r_max - band], n)
            have = O.keys(np.concatenate([ctr.numpy()[:, None], nbr.numpy()[:, None], img], 1), n)
            assert np.isin(must, have).all(), (step, b)
            if after[b] == before[b]:
                continue
            # a rebuild of frame b: its forces against the oracle at this step and the step before
            for p, fo in ((pos, forces), (prev_pos, prev_forces)):
                r = _oracle_frame(oracle, frames[b], p[fp[b]:fp[b + 1]].double().cpu(), r_max)
                e = _errs({"energy": torch.zeros(()), "atomic_energy": torch.zeros(0), "forces": fo[fp[b]:fp[b + 1]]},
                          {"energy": torch.zeros(()), "atomic_energy": torch.zeros(0), "forces": r["forces"]})["forces"]
                rec["forces"] = max(rec.get("forces", 0.0), e)
                assert e < 1e-4, (step, b, e)
                checked += 1
        rebuilt_steps += after != before
        prev_pos, prev_forces = pos.clone(), forces.clone()
        vel = vel + 0.5 * dt * forces / mass * acc_unit
    assert rebuilt_steps >= 3 and checked >= 6, (rebuilt_steps, checked)
    assert calc.n_captures == 1 + calc.n_overflows


def test_zz_report_errors():
    """prints the largest relative error per model, dtype and output of the tests above (nothing to assert)"""
    for (name, dt), errs in sorted(ERRORS.items()):
        print(f"\n[batched-oracle] {name:22s} {dt}: " + "  ".join(f"{k} {v:.2e}" for k, v in sorted(errs.items())))
