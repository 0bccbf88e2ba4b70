"""Third-order force constants of the c2 frame from pair clusters (phonons.third_order_force_constants) against the
full-frame route.

    python tools/time_force_constants3.py [--reps 2] [--displacement 0.03] [--out FILE]

  clusters    third_order_force_constants on the 10 976-atom c2 frame with the fp32 c2 model (S = 64, U = 32, l_max 2, two
              layers, r_max 5), every pair of 1 and of 4 displaced atoms (36 jobs per pair): seconds, pairs and batched
              edges/s
  full frame  energy_and_forces on the whole displaced frame, one call per job (the list at r_max + 2h built once, outside
              the window), for the sampled pairs k = j, a nearest neighbour and the farthest pair of the first atom, all
              9 (alpha, beta) each: seconds per call, and the same route extrapolated to every pair of one atom
  agreement   the sampled pairs from both routes, max |difference| over the atom's max |block|
Times are host wall clock around work that ends in a device synchronise, best of --reps.  The card's name and power limit
are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from allegro_b200 import _lib  # noqa: E402
from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402
from allegro_b200.phonons import third_order_force_constants  # noqa: E402
from time_batched_md import card  # noqa: E402

DEV = "cuda"
SIGNS = ((1.0, 1.0), (1.0, -1.0), (-1.0, 1.0), (-1.0, -1.0))


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def plan_edges(csr, atoms, n):
    """(pairs, batched edges of every job) of the displaced atoms: 36 jobs of |E(C_j n C_k)| edges per pair."""
    cptr, cen, _, _ = _lib.fc_centres(atoms, csr, n)
    pair_ptr, pair_col = _lib.fc_columns(cptr, cen, csr, n)
    Kptr, Ken, _, _ = _lib.fc_centres(torch.arange(n, device=DEV), csr, n)
    pj = atoms.to(torch.int32).repeat_interleave(pair_ptr[1:] - pair_ptr[:-1])
    pe = _lib.fc3_pairs(pj, pair_col, Kptr, Ken, csr)[3]
    return int(pj.shape[0]), 36 * int(pe.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--displacement", type=float, default=0.03)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_force_constants3.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}", flush=True)
    h = a.displacement
    pos, cell, types = systems.make_positions("c2")
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    n = pos.shape[0]
    model = AllegroModel(**systems.model_kwargs("c2", 42.0, "float32")).to(DEV)
    inner = model.model
    csr, sv = D.neighbor_csr(pos, inner.r_max + 2 * h, cell)
    chosen = torch.randperm(n, generator=torch.Generator().manual_seed(3))[:4].to(DEV)
    rec = {"card": name, "power_limit": pl, "model": "c2 fp32", "atoms": n, "displacement": h}

    third_order_force_constants(model, pos, cell, types, atoms=chosen[:1], displacement=h)  # warm-up
    for A in (1, 4):
        atoms = chosen[:A]
        P, edges = plan_edges(csr, atoms, n)
        t = min(wall(lambda: third_order_force_constants(model, pos, cell, types, atoms=atoms, displacement=h))[0] for _ in range(a.reps))
        print(f"clusters, {A} displaced atom(s): {t * 1e3:.1f} ms for {P} pairs ({36 * P} jobs), {edges} edges, {edges / t:.3e} edges/s",
              flush=True)
        rec[f"clusters_{A}_atoms_s"], rec[f"pairs_{A}_atoms"], rec[f"edges_{A}_atoms"] = t, P, edges
        rec[f"edges_per_s_{A}_atoms"] = edges / t
    fc = third_order_force_constants(model, pos, cell, types, atoms=chosen[:1], displacement=h)
    j = int(chosen[0])
    ks = fc.pair_col.tolist()
    d = (pos[ks] - pos[j]).double()
    f = d @ torch.linalg.inv(cell.double())
    r = ((f - f.round()) @ cell.double()).norm(dim=1).cpu()
    r[ks.index(j)] = float("inf")
    near = ks[int(r.argmin())]
    r[ks.index(j)] = -1.0
    far = ks[int(r.argmax())]
    sampled = [j, near, far]

    # the full-frame route on the same list
    data = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
    inner.energy_and_forces(data)

    def full():
        out = torch.zeros(len(sampled), n, 3, 3, 3, dtype=torch.float64, device=DEV)
        for p, k in enumerate(sampled):
            for alpha in range(3):
                for beta in range(3):
                    fs = []
                    for s1, s2 in SIGNS:
                        q = pos.clone()
                        q[j, alpha] += s1 * h
                        q[k, beta] += s2 * h
                        fs.append(inner.energy_and_forces(dict(data, **{D.POSITIONS_KEY: q}))[D.FORCE_KEY].double())
                    out[p, :, alpha, beta] = -((fs[0] + fs[3]) - (fs[1] + fs[2])) / (4 * h * h)
        return out

    runs = [wall(full) for _ in range(a.reps)]
    t_full = min(t for t, _ in runs)
    ref = runs[0][1]
    per = t_full / (36 * len(sampled))
    P1 = len(ks)
    print(f"full frame: {per * 1e3:.3f} ms per call ({csr.num_edges} edges); every pair of one atom this way "
          f"({36 * P1} calls): {per * 36 * P1:.1f} s", flush=True)
    got = torch.zeros_like(ref)
    for p, k in enumerate(sampled):
        q = ks.index(k)
        rr = slice(int(fc.row_ptr[q]), int(fc.row_ptr[q + 1]))
        got[p, fc.col[rr]] = fc.blocks[rr]
    err = float((got - ref).abs().max()) / float(fc.blocks.abs().max())
    print(f"agreement on pairs {sampled} (all 9 (alpha, beta)): max |diff| / the atom's max |block| = {err:.2e}", flush=True)
    rec.update({"full_frame_s_per_call": t_full / (36 * len(sampled)), "full_frame_one_atom_s": per * 36 * P1,
                "speedup_one_atom": per * 36 * P1 / rec["clusters_1_atoms_s"], "agreement_rel": err, "sampled_pairs": sampled})
    print(json.dumps(rec), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
