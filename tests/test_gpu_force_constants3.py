"""phonons.third_order_force_constants on the GPU: the ab2_fc3_* kernels against tests/fc3_spec.py, the locality argument
on the device (fp64 models equal full-frame mixed differences of energy_and_forces across the architecture grid and the
cell kinds), the tie to the harmonic path, the fp64 oracle's third derivatives, the properties of a third-order tensor,
determinism across chunkings and atom subsets, every refusal, and the 10 976-atom c2 frame in small chunks."""
import pytest
import torch

import fc3_spec
import fc_spec
from fc3_oracle import third_derivatives
from fc_oracle import synthetic_list
from test_gpu_force_constants import ARCH, _cell_frame, _dev_csr, _model
from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200 import systems
from allegro_b200.calculator import prune_table
from allegro_b200.model import AllegroModel
from allegro_b200.phonons import force_constants, third_order_force_constants

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---- kernels against the restatement -----------------------------------------------------------------------------------
@pytest.mark.parametrize("pdt,adt", [(torch.float64, torch.float64), (torch.float32, torch.float32), (torch.float64, torch.float32)])
@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (1, 2, 1), (2, 7, 2), (3, 12, 3), (5, 6, 5)])
def test_kernels_match_the_spec(seed, n, isolated, pdt, adt):
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated, dtype=pdt)
    g = torch.Generator().manual_seed(seed + 7)
    atoms = torch.randperm(n, generator=g)[:4]
    csr = _dev_csr(row_ptr, ctr, nbr)
    h = float(torch.tensor(0.0625, dtype=pdt))
    pair_ptr, pair_col = fc3_spec.pairs(atoms, row_ptr, ctr, nbr, n)
    pj = atoms.repeat_interleave(pair_ptr[1:] - pair_ptr[:-1])
    iptr, icen, ioff, pe = fc3_spec.intersections(pj, pair_col, row_ptr, ctr, nbr, n)
    rptr, col = fc_spec.columns(iptr, icen, row_ptr, nbr, n)
    # the plan on the device
    atoms_d = atoms.to(DEV)
    cp, ce, _, _ = _lib.fc_centres(atoms_d, csr, n)
    dpp, dpc = _lib.fc_columns(cp, ce, csr, n)
    assert torch.equal(dpp.cpu(), pair_ptr) and torch.equal(dpc.cpu().long(), pair_col)
    Kptr, Ken, _, _ = _lib.fc_centres(torch.arange(n, device=DEV), csr, n)
    pj_d, pk_d = pj.to(DEV, torch.int32), dpc
    di = _lib.fc3_pairs(pj_d, pk_d, Kptr, Ken, csr)
    for got, ref in zip(di, (iptr, icen, ioff, pe)):
        assert torch.equal(got.cpu().long(), ref.long())
    drp, dcol = _lib.fc_columns(di[0], di[1], csr, n)
    assert torch.equal(drp.cpu(), rptr) and torch.equal(dcol.cpu().long(), col)
    Pe_d = _lib._prefix(di[3])
    Cp, Ep = fc3_spec.unit_prefix(iptr, pe)
    U = 9 * pj.shape[0]
    blocks = torch.full((col.shape[0], 3, 3, 3), float("nan"), dtype=torch.float64, device=DEV)
    gref = torch.Generator().manual_seed(seed + 11)
    for u0, u1 in ((0, U), (0, 1), (1, 5), (5, U)) if U > 5 else ((0, U),):
        Cb, Eb = int(4 * (Cp[u1] - Cp[u0])), int(4 * (Ep[u1] - Ep[u0]))
        ref = fc3_spec.gather(pos, shift, h, adt, pj, pair_col, iptr, icen, ioff, pe, row_ptr, nbr, u0, u1)
        gvec = torch.randn(Eb, 3, generator=gref, dtype=torch.float64).to(adt)
        if Eb:
            got = _lib.fc3_gather(pos.to(DEV), shift.to(DEV), h, adt, pj_d, pk_d, di[0], di[1], di[2], Pe_d, csr, u0, u1, Cb, Eb)
            for a, b in zip(got[:4], ref[:4]):
                assert torch.equal(a.cpu().long(), b.long())
            assert torch.equal(got[4].cpu(), ref[4])  # the same operations in the positions' dtype, one rounding
        _lib.fc3_fold(gvec.to(DEV), h, di[0], di[1], di[2], Pe_d, csr, n, drp, dcol, u0, u1, blocks)
        want = fc3_spec.fold(gvec, h, iptr, icen, ioff, pe, row_ptr, ctr, nbr, rptr, col, u0, u1)
        bl = blocks.cpu()
        for (t, alpha, beta), v in want.items():
            torch.testing.assert_close(bl[t, alpha, beta], v, rtol=1e-12, atol=1e-12)
    assert not bool(blocks.isnan().any())


# ---- references ----------------------------------------------------------------------------------------------------------
def _full_fd3(model, pos, cell, types, pbc, pairs, h, r_list, cutoffs=None):
    """-(F++ - F+- - F-+ + F--) / (4h^2) of whole displaced frames from energy_and_forces, on a fixed list at r_list
    -> [P,N,3,3,3]."""
    inner = model.model
    prune = {} if cutoffs is None else dict(types=types.to(torch.int32), cutoffs=cutoffs)
    csr, sv = D.neighbor_csr(pos, r_list, cell, (pbc,) * 3, **prune)
    out = torch.zeros(len(pairs), pos.shape[0], 3, 3, 3, dtype=torch.float64)
    for p, (j, k) in enumerate(pairs):
        for alpha in range(3):
            for beta in range(3):
                fs = []
                for s1, s2 in fc3_spec.SIGNS:
                    q = pos.clone()
                    q[j, alpha] += s1 * h
                    q[k, beta] += s2 * h
                    d = {D.POSITIONS_KEY: q, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
                    if cell is not None:
                        d[D.CELL_KEY] = cell
                    fs.append(inner.energy_and_forces(d)[D.FORCE_KEY].double().cpu())
                out[p, :, alpha, beta] = -((fs[0] + fs[3]) - (fs[1] + fs[2])) / (4 * h * h)
    return out


def _pair_blocks(fc, j, k):
    """[N,3,3,3] fp64 on the CPU: the blocks of pair (j, k), zero where the pair has none."""
    a = fc.atoms.tolist().index(j)
    ks = fc.pair_col[int(fc.pair_ptr[a]):int(fc.pair_ptr[a + 1])].tolist()
    p = int(fc.pair_ptr[a]) + ks.index(k)
    out = torch.zeros(fc.num_atoms, 3, 3, 3, dtype=torch.float64)
    r = slice(int(fc.row_ptr[p]), int(fc.row_ptr[p + 1]))
    out[fc.col[r].cpu()] = fc.blocks[r].cpu()
    return out


def _atom_scale(fc, a):
    """max |block| of displaced atom a (row a): the scale errors are measured against."""
    p0, p1 = int(fc.pair_ptr[a]), int(fc.pair_ptr[a + 1])
    return float(fc.blocks[int(fc.row_ptr[p0]):int(fc.row_ptr[p1])].abs().max())


def _sampled(fc, pos, cell, j):
    """k = j, j's nearest pair atom and its farthest (minimum-image distance)."""
    a = fc.atoms.tolist().index(j)
    ks = fc.pair_col[int(fc.pair_ptr[a]):int(fc.pair_ptr[a + 1])].tolist()
    d = (pos[ks] - pos[j]).double()
    if cell is not None:
        c = cell.double()
        f = d @ torch.linalg.inv(c)
        d = (f - f.round()) @ c
    r = d.norm(dim=1).cpu()
    r[ks.index(j)] = float("inf")
    near = ks[int(r.argmin())]
    r[ks.index(j)] = -1.0
    far = ks[int(r.argmax())]
    return list(dict.fromkeys([j, near, far]))


def _check_full(model, pos, cell, types, pbc, j, h, tol, label):
    fc = third_order_force_constants(model, pos, cell, types, pbc=pbc, atoms=torch.tensor([j]), displacement=h)
    ks = _sampled(fc, pos, cell, j)
    ref = _full_fd3(model, pos, cell, types, pbc, [(j, k) for k in ks], h, model.model.r_max + 2 * h, prune_table(model, 2 * h))
    got = torch.stack([_pair_blocks(fc, j, k) for k in ks])
    err = float((got - ref).abs().max()) / _atom_scale(fc, 0)
    print(f"{label}: pairs {ks}, clusters vs full-frame mixed differences {err:.2e} of the atom's max |block|")
    assert err <= tol, err
    return fc


@pytest.mark.parametrize("arch", list(ARCH) + ["spline"])
def test_fp64_equals_full_frame_differences_across_the_grid(arch):
    _, model, kw = _model(None, "float64", arch)
    kind = "ortho" if arch != "spline" else "open"
    pos, cell, types, pbc = _cell_frame(kind, kw)
    if arch == "spline":
        pos = pos[:6] * 0.6
        types = types[:6]
    _check_full(model, pos, cell, types, pbc, 3, 0.01, 1e-9, arch)


@pytest.mark.parametrize("kind", ["ortho", "hcp", "short", "open"])
def test_fp64_equals_full_frame_differences_across_cells(kind):
    _, model, kw = _model(None, "float64")
    pos, cell, types, pbc = _cell_frame(kind, kw)
    _check_full(model, pos, cell, types, pbc, 1, 0.01, 1e-9, kind)
    if kind == "open":  # the isolated atom: the single pair (j, j) with one zero block
        j = pos.shape[0] - 1
        fc = third_order_force_constants(model, pos, cell, types, pbc=pbc, atoms=torch.tensor([j]))
        assert fc.pair_col.tolist() == [j] and fc.col.tolist() == [j] and bool((fc.blocks == 0).all())


def test_equals_the_central_difference_of_the_harmonic_constants():
    """Phi3(j, k, i)_{alpha beta gamma} = (Phi2(k, i)_{beta gamma}(r + h e_{j alpha}) - Phi2(...)(r - h e_{j alpha})) / (2h)
    with the same h: the same four force evaluations, so equal up to rounding, on every pair of the displaced atoms."""
    _, model, kw = _model(None, "float64")
    pos, cell, types, pbc = _cell_frame("hcp", kw)
    h = 0.01
    atoms = [0, 9]
    fc3 = third_order_force_constants(model, pos, cell, types, atoms=torch.tensor(atoms), displacement=h)
    for a, j in enumerate(atoms):
        ks = fc3.pair_col[int(fc3.pair_ptr[a]):int(fc3.pair_ptr[a + 1])]
        ref = torch.zeros(ks.shape[0], pos.shape[0], 3, 3, 3, dtype=torch.float64)
        for alpha in range(3):
            d = []
            for s in (1.0, -1.0):
                q = pos.clone()
                q[j, alpha] += s * h
                d.append(force_constants(model, q, cell, types, atoms=ks, displacement=h).dense().cpu())
            ref[:, :, alpha] = (d[0] - d[1]) / (2 * h)
        got = torch.stack([_pair_blocks(fc3, j, int(k)) for k in ks.tolist()])
        err = float((got - ref).abs().max()) / _atom_scale(fc3, a)
        print(f"atom {j}: {ks.shape[0]} pairs, against the harmonic path {err:.2e}")
        assert err <= 1e-9, err


def test_against_the_oracle_third_derivatives():
    oracle, m64, kw = _model(None, "float64")
    _, m32, _ = _model(None, "float32")
    pos, cell, types, pbc = _cell_frame("ortho", kw)
    j = 7
    p, c = pos.double().cpu(), cell.double().cpu()
    ei, sh = D.neighbor_list(p, kw["r_max"], c, (True, True, True))
    f64 = third_order_force_constants(m64, pos, cell, types, atoms=torch.tensor([j]), displacement=1e-3)
    ks = _sampled(f64, pos, cell, j)
    T = third_derivatives(oracle, p, types.cpu(), ei[0], ei[1], sh.double() @ c, torch.tensor([j] * len(ks)), torch.tensor(ks))
    scale = float(T.abs().max())
    e64 = float((torch.stack([_pair_blocks(f64, j, k) for k in ks]) - T).abs().max()) / scale
    f32 = third_order_force_constants(m32, pos.float(), cell.float(), types, atoms=torch.tensor([j]), displacement=0.03)
    e32 = float((torch.stack([_pair_blocks(f32, j, k) for k in ks]) - T).abs().max()) / scale
    # measured on an H100 (700 W): fp64 6.9e-6 (the h^2 term at h = 1e-3), fp32 6.2e-3 (mostly the h^2 term at h = 0.03)
    print(f"vs oracle third derivatives, pairs {ks}: fp64 model h=1e-3 {e64:.2e} (bar 2e-5); fp32 model h=0.03 {e32:.2e} (bar 1e-2)")
    assert e64 < 2e-5, e64
    assert e32 < 1e-2, e32


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_properties_and_determinism(dtype):
    _, model, kw = _model(None, dtype)
    pdt = torch.float64 if dtype == "float64" else torch.float32
    pos, cell, types, pbc = _cell_frame("hcp", kw, pdt)
    n = pos.shape[0]
    h = 0.01 if dtype == "float64" else 0.03
    full = third_order_force_constants(model, pos, cell, types, displacement=h)
    assert torch.equal(full.atoms.cpu(), torch.arange(n))
    Dn = full.dense().cpu()
    scale = float(full.blocks.abs().max())
    # translation invariance by construction: each edge's difference enters two columns with opposite signs
    asr = float(Dn.sum(2).abs().max()) / scale
    # Phi(j,k)_{abc} = Phi(k,j)_{bac}: the same four geometries (bitwise for fp32); full permutation symmetry to O(h^2)
    swap = float((Dn - Dn.permute(1, 0, 2, 4, 3, 5)).abs().max()) / scale
    perm = max(float((Dn - Dn.permute(*o)).abs().max()) / scale for o in ((2, 1, 0, 5, 4, 3), (0, 2, 1, 3, 5, 4), (1, 2, 0, 4, 5, 3)))
    print(f"{dtype}: sum over i {asr:.2e}, j<->k swap {swap:.2e}, other permutations {perm:.2e}")
    assert asr < 1e-13
    if dtype == "float32":
        assert swap == 0.0
    else:
        assert swap < 1e-10
    # measured on an H100 (700 W): 6.7e-5 (fp64, h = 0.01) and 6.5e-4 (fp32, h = 0.03)
    assert perm < (2e-4 if dtype == "float64" else 2e-3)
    # a subset, and other chunkings, give the same blocks (fp64: the tensor-product adjoint's atomics, divided by 4h^2)
    tol = 0.0 if dtype == "float32" else 1e-10
    worst = [0.0]

    def same(fc, rows):
        for b, a in enumerate(rows):
            assert torch.equal(fc.pair_col[int(fc.pair_ptr[b]):int(fc.pair_ptr[b + 1])], full.pair_col[int(full.pair_ptr[a]):int(full.pair_ptr[a + 1])])
            pa, pb = int(full.pair_ptr[a]), int(fc.pair_ptr[b])
            ra = slice(int(full.row_ptr[pa]), int(full.row_ptr[int(full.pair_ptr[a + 1])]))
            rb = slice(int(fc.row_ptr[pb]), int(fc.row_ptr[int(fc.pair_ptr[b + 1])]))
            assert torch.equal(fc.col[rb], full.col[ra])
            d = float((fc.blocks[rb] - full.blocks[ra]).abs().max()) / scale
            worst[0] = max(worst[0], d)
            assert d <= tol, (a, d)

    sub = torch.tensor([n - 1, 3, 0])
    same(third_order_force_constants(model, pos, cell, types, atoms=sub, displacement=h), sub.tolist())
    # the smallest valid cap is one unit's four jobs: read it from the refusal of a smaller one
    with pytest.raises(ValueError) as ei:
        third_order_force_constants(model, pos, cell, types, atoms=sub, displacement=h, max_edges=1)
    one = int(str(ei.value).split("the ")[1].split(" edges")[0])
    for cap in (one, 7 * one + 3):
        same(third_order_force_constants(model, pos, cell, types, atoms=sub, displacement=h, max_edges=cap), sub.tolist())
    print(f"{dtype}: subsets and chunkings differ by at most {worst[0]:.2e} of max |block| (bar {tol:g})")


def test_refusals():
    _, model, kw = _model(None, "float64")
    pos, cell, types, pbc = _cell_frame("ortho", kw)
    n = pos.shape[0]
    from allegro_b200.committee import Committee

    f = third_order_force_constants
    with pytest.raises(TypeError):
        f(Committee([model.model]), pos, cell, types)
    with pytest.raises(TypeError):
        f(object(), pos, cell, types)
    with pytest.raises(RuntimeError):
        f(model, pos.cpu(), cell, types)
    with pytest.raises(RuntimeError):
        f(model, pos, cell, types.cpu())
    for h in (0.0, -0.01, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            f(model, pos, cell, types, displacement=h)
    for atoms in (torch.tensor([[0, 1]]), torch.tensor([0.0, 1.0]), torch.tensor([-1]), torch.tensor([n]), torch.tensor([2, 2])):
        with pytest.raises(ValueError):
            f(model, pos, cell, types, atoms=atoms)
    for bad in (pos[:, :2].contiguous(), pos.to(torch.float16), pos.unsqueeze(0)):
        with pytest.raises(ValueError):
            f(model, bad, cell, types)
    for bad in (types[:-1], types.unsqueeze(-1), types.double()):
        with pytest.raises(ValueError):
            f(model, pos, cell, bad)
    flat = cell.clone()
    flat[2] = flat[0] + flat[1]
    for c in (None, flat):
        with pytest.raises(ValueError):
            f(model, pos, c, types)
    for cap in (0, 1 << 31):
        with pytest.raises(ValueError):
            f(model, pos, cell, types, max_edges=cap)
    big = torch.zeros(_lib.FC_MAX_ATOMS + 1, 3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError):
        f(model, big, None, torch.zeros(big.shape[0], dtype=torch.int64, device=DEV), pbc=False)
    with pytest.raises(ValueError):  # known once the plan is: one unit's four jobs exceed max_edges
        f(model, pos, cell, types, atoms=torch.tensor([0]), max_edges=8)


def test_c2_frame_in_small_chunks():
    """The 10 976-atom c2 frame, fp32 model: 2 random displaced atoms in chunks of <= 60 k edges against full-frame mixed
    differences on sampled pairs.  The error is the fp32 rounding of the displaced full-frame positions (|r| up to 50 A)
    divided by 4 h^2: measured 6.0e-4 and 6.5e-4 of the atom's largest block on an H100 (700 W), bar 2e-3."""
    pos, cell, types = systems.make_positions("c2")
    kw = systems.model_kwargs("c2", 42.0, "float32")
    m = AllegroModel(**kw).to(DEV)
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    g = torch.Generator().manual_seed(5)
    atoms = torch.randperm(pos.shape[0], generator=g)[:2]
    h = 0.03
    fc = third_order_force_constants(m, pos, cell, types, atoms=atoms, displacement=h, max_edges=60_000)
    for a, j in enumerate(atoms.tolist()):
        ks = _sampled(fc, pos, cell, j)
        ref = _full_fd3(m, pos, cell, types, True, [(j, k) for k in ks], h, kw["r_max"] + 2 * h)
        got = torch.stack([_pair_blocks(fc, j, k) for k in ks])
        err = float((got - ref).abs().max()) / _atom_scale(fc, a)
        print(f"c2 fp32 atom {j}: {int(fc.pair_ptr[a + 1] - fc.pair_ptr[a])} pairs, sampled {ks}: rel {err:.2e}")
        assert err < 2e-3, err
