"""Third-order force constants from pair clusters, on the CPU: the plain-torch restatement of the plan (tests/fc3_spec.py)
against a brute-force construction, and the locality argument against the fp64 oracle -- C_j n C_k alone gives the mixed
central differences of the full frame, and both approach the oracle's third derivatives as h^2."""
import pytest
import torch

import fc3_spec
import fc_spec
from fc3_oracle import cluster_blocks, full_fd_blocks, third_derivatives
from fc_oracle import frame_list, synthetic_list
from test_host_force_constants import _c1, _fcc


def _centres(ctr, nbr, j):
    return {j} | {int(c) for c, m in zip(ctr.tolist(), nbr.tolist()) if m == j}


@pytest.mark.parametrize("seed,n,isolated", [(0, 1, 0), (1, 2, 1), (2, 7, 2), (3, 12, 3), (5, 6, 5)])
def test_spec_matches_brute_force(seed, n, isolated):
    pos, row_ptr, ctr, nbr, shift = synthetic_list(seed, n, isolated=isolated)
    g = torch.Generator().manual_seed(seed + 200)
    atoms = torch.randperm(n, generator=g)[: max(1, n - 1)]
    h = 0.0625
    pair_ptr, pair_col = fc3_spec.pairs(atoms, row_ptr, ctr, nbr, n)
    pj = atoms.repeat_interleave(pair_ptr[1:] - pair_ptr[:-1])
    pk = pair_col
    iptr, icen, ioff, pe = fc3_spec.intersections(pj, pk, row_ptr, ctr, nbr, n)
    rptr, col = fc_spec.columns(iptr, icen, row_ptr, nbr, n)
    C = [_centres(ctr, nbr, i) for i in range(n)]
    for a, j in enumerate(atoms.tolist()):
        # the pairs of j are exactly the atoms k with C_j n C_k non-empty
        assert pair_col[pair_ptr[a]:pair_ptr[a + 1]].tolist() == [k for k in range(n) if C[j] & C[k]]
    for p in range(pj.shape[0]):
        j, k = int(pj[p]), int(pk[p])
        I = sorted(C[j] & C[k])
        zs = [z for c in I for z in range(int(row_ptr[c]), int(row_ptr[c + 1]))]
        assert icen[iptr[p]:iptr[p + 1]].tolist() == I and int(pe[p]) == len(zs)
        assert col[rptr[p]:rptr[p + 1]].tolist() == sorted(set(I) | {int(nbr[z]) for z in zs})
        for ab in range(9):
            alpha, beta = ab // 3, ab % 3
            u = 9 * p + ab
            rp, cb, cz, nz, vb = fc3_spec.gather(pos, shift, h, torch.float64, pj, pk, iptr, icen, ioff, pe, row_ptr, nbr, u, u + 1)
            Cb, E = 4 * len(I), len(zs)
            assert cb.tolist() == I * 4 and int(rp[-1]) == 4 * E and cz.shape[0] == 4 * E
            assert (nz - Cb).tolist() == [int(nbr[z]) for z in zs] * 4
            assert cz.tolist() == [q for q in range(Cb) for _ in range(int(rp[q + 1] - rp[q]))]
            for sigma, (s1, s2) in enumerate(fc3_spec.SIGNS):
                q = pos.clone()
                q[j, alpha] += s1 * h
                q[k, beta] += s2 * h
                z = torch.tensor(zs, dtype=torch.int64)
                ref = q[nbr[z]] - q[ctr[z]] + shift[z] if zs else torch.zeros(0, 3, dtype=pos.dtype)
                torch.testing.assert_close(vb[sigma * E:(sigma + 1) * E], ref, rtol=0, atol=1e-12)
    # an isolated atom: the single pair (j, j), its cluster {j} without edges, and the one column j
    iso = [i for i in range(n) if int(row_ptr[i + 1] - row_ptr[i]) == 0 and not bool((nbr == i).any())]
    assert len(iso) >= isolated
    if iso:
        j = iso[0]
        pp, pc = fc3_spec.pairs(torch.tensor([j]), row_ptr, ctr, nbr, n)
        assert pc.tolist() == [j]
        ip, ic, io, e = fc3_spec.intersections(torch.tensor([j]), pc, row_ptr, ctr, nbr, n)
        assert ic.tolist() == [j] and int(e.sum()) == 0
        rp, cb, cz, nz, vb = fc3_spec.gather(pos, shift, h, torch.float64, torch.tensor([j]), pc, ip, ic, io, e, row_ptr, nbr, 0, 9)
        assert rp.tolist() == [0] * 37 and cz.numel() == 0
        assert fc_spec.columns(ip, ic, row_ptr, nbr, n)[1].tolist() == [j]


def _sampled_pairs(row_ptr, ctr, nbr, pos, cell, n, j):
    """k = j, j's nearest neighbour and the farthest of j's pairs (minimum-image distance)."""
    _, cols = fc3_spec.pairs(torch.tensor([j]), row_ptr, ctr, nbr, n)
    cols = cols.tolist()
    d = pos[cols] - pos[j]
    if cell is not None:
        f = d @ torch.linalg.inv(cell)
        d = (f - f.round()) @ cell
    r = d.norm(dim=1)
    r[cols.index(j)] = float("inf")
    near = cols[int(r.argmin())]
    r[cols.index(j)] = -1.0
    far = cols[int(r.argmax())]
    return sorted({j, near, far}, key=[j, near, far].index)


@pytest.mark.parametrize("case", ["c1", "fcc1", "fcc2"])
def test_clusters_give_the_full_frame_mixed_differences(case):
    oracle, kw, d = _c1()
    h = 0.01
    if case == "c1":
        pos, cell = d["pos"], d["cell"]
    else:
        pos, cell = _fcc(1 if case == "fcc1" else 2)
    n = pos.shape[0]
    types = torch.zeros(n, dtype=torch.int64)
    row_ptr, ctr, nbr, sv = frame_list(pos, cell, (True, True, True), kw["r_max"] + 2 * h)
    if case != "c1":
        assert bool((ctr == nbr).any())  # self-images
    j = 5 if case == "c1" else 0
    if case == "c1":
        ks = _sampled_pairs(row_ptr, ctr, nbr, pos, cell, n, j)
        assert len(ks) == 3
    else:
        ks = fc3_spec.pairs(torch.tensor([j]), row_ptr, ctr, nbr, n)[1].tolist()  # every pair
    pj, pk = torch.full((len(ks),), j), torch.tensor(ks)
    loc = cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, sv, pj, pk, h)
    full = full_fd_blocks(oracle, pos, types, ctr, nbr, sv, pj, pk, h)
    # the pair k = j holds the displaced atom's largest block; a lone atom in its cell only translates rigidly: all zero
    scale = float(full.abs().max()) or 1.0
    err = float((loc - full).abs().max()) / scale
    print(f"{case}: pairs {ks}, clusters vs full frame {err:.2e} of max |block| {scale:.3g}")
    assert err <= 1e-10, err


def test_clusters_approach_the_oracle_third_derivatives():
    oracle, kw, d = _c1()
    pos, cell = d["pos"], d["cell"]
    n = pos.shape[0]
    types = torch.zeros(n, dtype=torch.int64)
    j = 5
    errs = []
    T = None
    for h in (1e-2, 1e-3):
        row_ptr, ctr, nbr, sv = frame_list(pos, cell, (True, True, True), kw["r_max"] + 2 * h)
        if T is None:
            ks = _sampled_pairs(row_ptr, ctr, nbr, pos, cell, n, j)
            pj, pk = torch.full((len(ks),), j), torch.tensor(ks)
            T = third_derivatives(oracle, pos, types, ctr, nbr, sv, pj, pk)
        loc = cluster_blocks(oracle, pos, types, row_ptr, ctr, nbr, sv, pj, pk, h)
        errs.append(float((loc - T).abs().max()) / float(T.abs().max()))
    # the sum over i of a third-derivative row is zero (translation invariance)
    assert float(T.sum(1).abs().max()) < 1e-12 * float(T.abs().max())
    print(f"clusters vs third derivatives: h=1e-2 {errs[0]:.2e}, h=1e-3 {errs[1]:.2e}")
    assert errs[1] < errs[0] / 50, errs
