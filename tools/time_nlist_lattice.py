"""Cost of the general-lattice device cell list against the orthorhombic one and the torch all-pairs search.

    python tools/time_nlist_lattice.py [--reps 20] [--steps 50] [--rounds 3] [--out FILE]

Frames: c2 (10 976 atoms) and the same fcc crystal at 29^3 cells (97 556 atoms), fp32 positions, list cutoff 5.5
(r_max 5 + skin 0.5).  Every search is timed with CUDA events around one call (median of ``--reps``, all variants
alternated).  Three searches through the same layer, ``_lib`` with the grid computed once outside the timed region
(bin, sort by bin, count, prefix sum, fill; one device->host read of the edge count):
  ortho   : the cubic cell, cell_grid -> _lib.neighbor_csr (ab2_nl_*);
  lattice : the same cubic cell, lattice_grid -> _lib.neighbor_csr_lattice (ab2_nl_lattice_*);
  tilted  : the same crystal in the unimodular basis (a + b, b, a + c), lattice_grid -> _lib.neighbor_csr_lattice.
And the two a user calls, through data.neighbor_csr (grid choice on the host plus the EdgeCSR wrapper included):
  api-cubic (orthorhombic route) and api-tilted (lattice route).
The torch all-pairs search (neighbor_list method="brute") of the tilted frame is timed where its [N,N,3] fp64 buffers
fit on the card; the frames it skips are listed.  Then the MD calculator on c2 (fp32 model): rebuild cost (list plus
CUDA-graph capture) and the graph-replayed step, tilted against cubic, alternated.  The card's name and power limit
are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from allegro_b200 import _lib  # noqa: E402
from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402

DEV = "cuda"
R_LIST = 5.5
TILT = torch.tensor([[1.0, 1.0, 0.0], [0.0, 1.0, 0.0], [1.0, 0.0, 1.0]], dtype=torch.float64)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def _timed_ms(fn):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0.record()
    out = fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1), out


def searches(pos, cell):
    pbc = (True, True, True)
    box, origin, ncell = D.cell_grid(pos, R_LIST, torch.diagonal(cell).tolist(), pbc)
    cubic = D.lattice_grid(pos, R_LIST, cell, pbc)
    tilted_cell = TILT @ cell
    tilted = D.lattice_grid(pos, R_LIST, tilted_cell, pbc)
    cell_d, tilted_d = cell.to(DEV), tilted_cell.to(DEV)
    return {
        "ortho": lambda: _lib.neighbor_csr(pos, R_LIST, box, ncell, pbc, origin)[0],
        "lattice": lambda: _lib.neighbor_csr_lattice(pos, R_LIST, *cubic, pbc)[0],
        "tilted": lambda: _lib.neighbor_csr_lattice(pos, R_LIST, *tilted, pbc)[0],
        "api-cubic": lambda: D.neighbor_csr(pos, R_LIST, cell_d)[0].row_ptr,
        "api-tilted": lambda: D.neighbor_csr(pos, R_LIST, tilted_d)[0].row_ptr,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_nlist_lattice.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}")
    rec = {"card": name, "power_limit": pl, "r_list": R_LIST, "search_ms": {}, "edges": {}, "brute_ms": {}, "brute_skipped": []}
    free = torch.cuda.mem_get_info()[0]
    for label, scale in (("c2", None), ("fcc-29^3", 29)):
        pos, cell, _ = systems.make_positions("c2", scale) if scale else systems.make_positions("c2")
        n = pos.shape[0]
        pos = pos.to(torch.float32).to(DEV)
        fns = searches(pos, cell)
        edges = {k: int(f()[-1]) for k, f in fns.items()}  # warm-up; every search finds the same number of pairs
        assert len(set(edges.values())) == 1, edges
        per = {k: [] for k in fns}
        for _ in range(a.reps):
            for k, f in fns.items():
                per[k].append(_timed_ms(f)[0])
        med = {k: statistics.median(v) for k, v in per.items()}
        rec["search_ms"][label], rec["edges"][label] = med, edges
        print(f"{label:9s} N={n:6d} E={edges['ortho']}  " + "  ".join(f"{k} {med[k]:.3f} ms" for k in fns)
              + f"  lattice/ortho {med['lattice'] / med['ortho']:.2f}  tilted/ortho {med['tilted'] / med['ortho']:.2f}"
              + f"  api-tilted/api-cubic {med['api-tilted'] / med['api-cubic']:.2f}")
        # torch all-pairs on the tilted cell: about 33 N^2 bytes of fp64 temporaries per image
        need = 33 * n * n * 2
        if need < 0.8 * free:
            tilted = TILT @ cell
            pos64 = pos.double()
            t0 = time.perf_counter()
            torch.cuda.synchronize()
            ei, _ = D.neighbor_list(pos64, R_LIST, tilted.to(DEV), (True, True, True), method="brute")
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            rec["brute_ms"][label] = ms
            print(f"{label:9s} torch brute force (tilted, fp64, one call): {ms:.1f} ms, E={ei.shape[1]}")
            del ei
            torch.cuda.empty_cache()
        else:
            rec["brute_skipped"].append(label)
            print(f"{label:9s} torch brute force skipped: needs about {need / 1e9:.0f} GB of temporaries")
    calculator(a, rec)
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


def calculator(a, rec):
    from allegro_b200.calculator import AllegroCalculator
    from allegro_b200.model import AllegroModel

    d = systems.make_system("c2")
    n, e = d[D.POSITIONS_KEY].shape[0], d[D.EDGE_INDEX_KEY].shape[1]
    model = AllegroModel(**systems.model_kwargs("c2", e / n, "float32")).to(DEV)
    pos = d[D.POSITIONS_KEY].to(torch.float32).to(DEV)
    types = d[D.ATOM_TYPE_KEY].to(DEV)
    cells = {"cubic": d[D.CELL_KEY].view(3, 3).to(DEV), "tilted": (TILT @ d[D.CELL_KEY].view(3, 3)).to(DEV)}
    calcs = {k: AllegroCalculator(model, 5.0, skin=0.5) for k in cells}
    for k, c in calcs.items():
        c.compute(pos, cells[k], types)
    out = {k: calcs[k].compute(pos, cells[k], types)["forces"].clone() for k in cells}
    dev = float((out["cubic"] - out["tilted"]).abs().max() / out["cubic"].abs().max())
    rebuild = {k: [] for k in cells}
    step = {k: [] for k in cells}
    for _ in range(a.rounds):
        for k, c in calcs.items():
            rebuild[k].append(_timed_ms(lambda: c._rebuild(pos, cells[k], types))[0])
        for k, c in calcs.items():
            ms, _ = _timed_ms(lambda: [c.compute(pos, cells[k], types) for _ in range(a.steps)])
            step[k].append(ms / a.steps)
    med_r = {k: statistics.median(v) for k, v in rebuild.items()}
    med_s = {k: statistics.median(v) for k, v in step.items()}
    rec["calculator"] = {"rebuild_ms": med_r, "step_ms": med_s, "rebuild_rounds": rebuild, "step_rounds": step, "max_rel_force_dev": dev,
                         "edges": {k: c.num_edges for k, c in calcs.items()}}
    for k in cells:
        print(f"calculator {k:7s} rebuild (list + graph capture) {med_r[k]:.1f} ms   graph-replayed step {med_s[k]:.3f} ms   "
              f"E={calcs[k].num_edges}")
    print(f"calculator tilted vs cubic: max relative force deviation {dev:.2e}")


if __name__ == "__main__":
    main()
