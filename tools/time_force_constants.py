"""Force constants of the c2 frame from displacement clusters (phonons.force_constants) against the full-frame route.

    python tools/time_force_constants.py [--check-atoms 10] [--reps 2] [--out FILE]

  clusters    force_constants on the 10 976-atom c2 frame with the fp32 c2 model (S = 64, U = 32, l_max 2, two layers,
              r_max 5), every atom displaced (6 N jobs): total seconds, displacements/s and batched edges/s
  full frame  energy_and_forces on the whole displaced frame, one call per displacement (the list at r_max + h built
              once, outside the window), over 6 x --check-atoms displacements: seconds per displacement, and the c2
              energy_and_forces edge rate of the same calls
  agreement   the rows of those atoms from both routes, max |difference| over max |block|
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
from allegro_b200.phonons import force_constants  # noqa: E402
from time_batched_md import card  # noqa: E402

DEV = "cuda"


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check-atoms", type=int, default=10)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--displacement", type=float, default=0.01)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_force_constants.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}", flush=True)
    h = a.displacement
    pos, cell, types = systems.make_positions("c2")
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    n = pos.shape[0]
    model = AllegroModel(**systems.model_kwargs("c2", 42.0, "float32")).to(DEV)
    inner = model.model
    r_max = inner.r_max

    # the clusters: every atom displaced
    csr, sv = D.neighbor_csr(pos, r_max + h, cell)
    ea = _lib.fc_centres(torch.arange(n, device=DEV), csr, n)[3]
    edges = 6 * int(ea.sum())
    force_constants(model, pos, cell, types, atoms=torch.arange(64, device=DEV), displacement=h)  # warm-up
    t_fc = min(wall(lambda: force_constants(model, pos, cell, types, displacement=h))[0] for _ in range(a.reps))
    fc = force_constants(model, pos, cell, types, displacement=h)
    print(f"clusters: {t_fc:.3f} s for {6 * n} displacements, {6 * n / t_fc:.0f} displacements/s, {edges} edges, "
          f"{edges / t_fc:.3e} edges/s", flush=True)

    # the full-frame route on the same list
    check = torch.randperm(n, generator=torch.Generator().manual_seed(3))[: a.check_atoms].tolist()
    data = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
    inner.energy_and_forces(data)

    def full():
        rows = torch.zeros(len(check), n, 3, 3, dtype=torch.float64, device=DEV)
        for i, j in enumerate(check):
            for alpha in range(3):
                fs = []
                for s in (1.0, -1.0):
                    q = pos.clone()
                    q[j, alpha] += s * h
                    fs.append(inner.energy_and_forces(dict(data, **{D.POSITIONS_KEY: q}))[D.FORCE_KEY].double())
                rows[i, :, alpha] = -(fs[0] - fs[1]) / (2 * h)
        return rows

    runs = [wall(full) for _ in range(a.reps)]
    t_full = min(t for t, _ in runs)
    ref = runs[0][1]
    per = t_full / (6 * len(check))
    E_full = csr.num_edges
    print(f"full frame: {per * 1e3:.3f} ms per displacement ({E_full} edges, {E_full / per:.3e} edges/s); "
          f"every atom this way: {per * 6 * n:.1f} s", flush=True)
    got = torch.zeros_like(ref)
    for i, j in enumerate(check):  # fc.atoms is every atom in order: row j is atom j
        r = slice(int(fc.row_ptr[j]), int(fc.row_ptr[j + 1]))
        got[i, fc.col[r]] = fc.blocks[r]
    err = float((got - ref).abs().max() / ref.abs().max())
    print(f"agreement on {len(check)} atoms ({6 * len(check)} displacements): max |diff| / max |block| = {err:.2e}", flush=True)
    rec = {"card": name, "power_limit": pl, "model": "c2 fp32", "atoms": n, "displacement": h, "clusters_s": t_fc,
           "displacements_per_s": 6 * n / t_fc, "cluster_edges": edges, "cluster_edges_per_s": edges / t_fc,
           "full_frame_s_per_displacement": per, "full_frame_edges_per_s": E_full / per, "full_frame_all_atoms_s": per * 6 * n,
           "speedup": per * 6 * n / t_fc, "agreement_rel": err}
    print(json.dumps(rec), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
