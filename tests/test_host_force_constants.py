"""Force constants from displacement clusters, on the CPU: the plain-torch restatement of the plan (tests/fc_spec.py)
against a brute-force construction, and the locality argument against the fp64 oracle -- the clusters alone give the
central differences of the full frame, and both approach the oracle's analytic Hessian as h^2."""
import pytest
import torch

import fc_spec
from fc_oracle import cluster_blocks, frame_list, full_fd_blocks, hessian_rows, rel, synthetic_list
from allegro_b200 import systems
from oracle.model_ref import AllegroOracle


def _brute(pos, row_ptr, ctr, nbr, shift, j):
    """C_j, the columns and every job's edges and edge vectors of atom j from the definitions."""
    C = sorted({j} | {int(c) for c, m in zip(ctr.tolist(), nbr.tolist()) if m == j})
    zs = [z for k in C for z in range(int(row_ptr[k]), int(row_ptr[k + 1]))]
    cols = sorted(set(C) | {int(nbr[z]) for z in zs})
    return C, cols, zs


@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (1, 2, 1), (2, 7, 2), (3, 12, 3), (4, 20, 0), (5, 6, 5)])
def test_spec_matches_brute_force(seed, n, isolated):
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated)
    g = torch.Generator().manual_seed(seed + 100)
    atoms = torch.randperm(n, generator=g)[: max(1, n - 1)]
    h = 0.0625
    cptr, cen, coff, ea = fc_spec.centres(atoms, row_ptr, ctr, nbr, n)
    fptr, col = fc_spec.columns(cptr, cen, row_ptr, nbr, n)
    for a, j in enumerate(atoms.tolist()):
        C, cols, zs = _brute(pos, row_ptr, ctr, nbr, shift, j)
        assert cen[cptr[a]:cptr[a + 1]].tolist() == C
        assert col[fptr[a]:fptr[a + 1]].tolist() == cols
        assert int(ea[a]) == len(zs)
        for alpha in range(3):
            u = 3 * a + alpha
            rp, cb, cz, nz, vb = fc_spec.gather(pos, shift, h, torch.float64, atoms, cptr, cen, coff, ea, row_ptr, nbr, u, u + 1)
            Cb = 2 * len(C)
            assert cb.tolist() == C + C and rp[-1] == 2 * len(zs) and cz.shape[0] == 2 * len(zs)
            assert (nz - Cb).tolist() == [int(nbr[z]) for z in zs] * 2
            assert cz.tolist() == [q for q in range(Cb) for _ in range(int(rp[q + 1] - rp[q]))]
            for s, sl in ((1.0, slice(0, len(zs))), (-1.0, slice(len(zs), 2 * len(zs)))):
                q = pos.clone()
                q[j, alpha] += s * h
                z = torch.tensor(zs, dtype=torch.int64)
                ref = q[nbr[z]] - q[ctr[z]] + shift[z] if zs else torch.zeros(0, 3, dtype=pos.dtype)
                torch.testing.assert_close(vb[sl], ref, rtol=0, atol=1e-12)
    # a chunk of isolated atoms has no edge at all (the E == 0 path)
    iso = [i for i in range(n) if int(row_ptr[i + 1] - row_ptr[i]) == 0 and not bool((nbr == i).any())]
    assert len(iso) >= isolated
    if iso:
        a_iso = torch.tensor(iso[:1])
        cp, ce, co, e = fc_spec.centres(a_iso, row_ptr, ctr, nbr, n)
        assert ce.tolist() == iso[:1] and int(e.sum()) == 0
        rp, cb, cz, nz, vb = fc_spec.gather(pos, shift, h, torch.float64, a_iso, cp, ce, co, e, row_ptr, nbr, 0, 3)
        assert rp.tolist() == [0] * 7 and cz.numel() == 0
        fp, cl = fc_spec.columns(cp, ce, row_ptr, nbr, n)
        assert cl.tolist() == iso[:1]


def _c1(dtype="float64", **over):
    d = systems.make_system("c1", None)
    kw = systems.model_kwargs("c1", d["edge_index"].shape[1] / d["pos"].shape[0], dtype)
    kw.update(over)
    return AllegroOracle(**kw), kw, d


def _fcc(n_atoms):
    """A 1- or 2-atom FCC cell (a = 3.6) whose atoms see their own images within r_max = 4."""
    a = 3.6
    cell = torch.tensor([[0.0, a / 2, a / 2], [a / 2, 0.0, a / 2], [a / 2, a / 2, 0.0]], dtype=torch.float64)
    pos = torch.tensor([[0.05, -0.03, 0.02]], dtype=torch.float64)
    if n_atoms == 2:
        cell = cell * torch.tensor([[2.0], [1.0], [1.0]], dtype=torch.float64)
        pos = torch.cat([pos, pos + cell[0] / 2 + torch.tensor([0.04, 0.0, -0.02], dtype=torch.float64)])
    return pos, cell


@pytest.mark.parametrize("case", ["c1", "fcc1", "fcc2"])
def test_clusters_give_the_full_frame_differences(case):
    oracle, kw, d = _c1()
    h = 0.01
    if case == "c1":
        pos, cell = d["pos"], d["cell"]
        atoms = torch.tensor([0, 37])
    else:
        pos, cell = _fcc(1 if case == "fcc1" else 2)
        atoms = torch.arange(pos.shape[0])
    types = torch.zeros(pos.shape[0], dtype=torch.int64)
    row_ptr, ctr, nbr, sv = frame_list(pos, cell, (True, True, True), kw["r_max"] + h)
    if case != "c1":
        assert bool((ctr == nbr).any())  # self-images
    loc = cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, sv, atoms, h)
    full = full_fd_blocks(oracle, pos, cell, types, ctr, nbr, sv, atoms, h)
    err = rel(loc, full)
    print(f"{case}: clusters vs full frame rel {err:.2e}")
    assert err <= 1e-12, err


def test_clusters_approach_the_oracle_hessian():
    oracle, kw, d = _c1()
    pos, cell = d["pos"], d["cell"]
    types = torch.zeros(pos.shape[0], dtype=torch.int64)
    atoms = torch.tensor([5, 50])
    H = None
    errs = []
    for h in (1e-3, 1e-4):
        row_ptr, ctr, nbr, sv = frame_list(pos, cell, (True, True, True), kw["r_max"] + h)
        if H is None:
            H = hessian_rows(oracle, pos, types, ctr, nbr, sv, atoms)
        errs.append(rel(cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, sv, atoms, h), H))
    print(f"clusters vs Hessian rel: h=1e-3 {errs[0]:.2e}, h=1e-4 {errs[1]:.2e}")
    assert errs[1] < 1e-5 and errs[1] < errs[0] / 20
