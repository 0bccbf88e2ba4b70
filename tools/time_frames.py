"""Many small frames: the per-frame loop against batched evaluation (energy_and_forces_frames).

    python tools/time_frames.py [--frames 512] [--loop-frames 64] [--batch 8 64 512] [--reps 3] [--out FILE]

c2 model kwargs (S = 64, U = 32, l_max 2, two layers, r_max 5) in fp32 (the composed two-layer path) and fp64, on three
kinds of seeded frames built from systems.py primitives:
  si64     64-atom Si diamond cells (2x2x2, a = 5.431 A), jittered: small periodic cells (2.2 r_max)
  fcc_tri  sheared 2x2x2 FCC cells (32 atoms): triclinic
  cluster  21-atom random non-periodic clusters: molecule-sized
and reports ms per frame and atoms/s for
  (a) the loop users run today: data.neighbor_list + energy_and_forces, one frame at a time
  (b) the same loop with the lists prebuilt (model only)
  (c) batch.collate (device neighbour list) + energy_and_forces_frames at each batch size; the list alone is timed too.
Before timing, (c) is checked against (b) on the same frames.  Times are host wall clock around work that ends in a
device synchronise, best of --reps passes.  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.batch import collate  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

DEV = "cuda"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def make_frames(kind: str, count: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    frames = []
    for _ in range(count):
        if kind == "si64":
            pos, cell = systems._lattice(systems._DIAMOND, 5.431, (2, 2, 2), 0.15, g)
        elif kind == "fcc_tri":
            pos, cell = systems._lattice(systems._FCC, 3.615, (2, 2, 2), 0.1, g)
            shear = torch.eye(3, dtype=torch.float64)
            shear[1, 0], shear[2, 0], shear[2, 1] = 0.1 + 0.1 * float(torch.rand(1, generator=g)), -0.15, 0.12
            pos, cell = pos @ shear, cell @ shear
        elif kind == "cluster":
            pts = []
            while len(pts) < 21:
                p = (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 5.0
                if all(float((p - q).norm()) > 2.2 for q in pts):
                    pts.append(p)
            pos, cell = torch.stack(pts), None
        else:
            raise KeyError(kind)
        f = {D.POSITIONS_KEY: pos.to(DEV), D.ATOM_TYPE_KEY: torch.zeros(pos.shape[0], dtype=torch.long, device=DEV)}
        if cell is not None:
            f[D.CELL_KEY] = cell.to(DEV)
        frames.append(f)
    return frames


def with_list(f, r_max):
    f = dict(f)
    cell = f.get(D.CELL_KEY)
    pbc = (True,) * 3 if cell is not None else (False,) * 3
    ei, sh = D.neighbor_list(f[D.POSITIONS_KEY], r_max, cell, pbc)
    f[D.EDGE_INDEX_KEY] = ei
    if cell is not None:
        f[D.EDGE_CELL_SHIFT_KEY] = sh
    return f


def timed(fn, reps):
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--loop-frames", type=int, default=64, help="frames timed in the per-frame loops (a) and (b)")
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 64, 512])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dtypes", nargs="+", default=["float32", "float64"])
    ap.add_argument("--kinds", nargs="+", default=["si64", "fcc_tri", "cluster"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_frames.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}")
    results = []
    for dtype in a.dtypes:
        model = AllegroModel(**systems.model_kwargs("c2", 40.0, dtype)).to(DEV)
        m = model.model
        r_max = m.r_max
        for kind in a.kinds:
            frames = make_frames(kind, a.frames, seed=7)
            n_atoms = [f[D.POSITIONS_KEY].shape[0] for f in frames]
            loop = frames[: a.loop_frames]
            pre = [with_list(f, r_max) for f in loop]
            # (c) against (b) on the same frames, before any timing
            bs0 = min(a.batch[0], len(pre))
            out_c = m.energy_and_forces_frames(collate(frames[:bs0], r_max))
            e_c = out_c[D.TOTAL_ENERGY_KEY].double().cpu().reshape(-1)
            e_b = torch.stack([m.energy_and_forces(f)[D.TOTAL_ENERGY_KEY].double().cpu().reshape(()) for f in pre[:bs0]])
            f_c = out_c[D.FORCE_KEY].double().cpu()
            f_b = torch.cat([m.energy_and_forces(f)[D.FORCE_KEY].double().cpu() for f in pre[:bs0]])
            de = float((e_c - e_b).abs().max() / e_b.abs().max().clamp(min=1e-30))
            dfm = float((f_c - f_b).abs().max() / f_b.abs().max().clamp(min=1e-30))
            tol = 1e-9 if dtype == "float64" else 1e-4
            assert de < tol and dfm < tol, (dtype, kind, de, dfm)
            n_loop = sum(n_atoms[: len(loop)])

            def run_a():
                for f in loop:
                    m.energy_and_forces(with_list(f, r_max))

            def run_b():
                for f in pre:
                    m.energy_and_forces(f)

            ta, tb = timed(run_a, a.reps), timed(run_b, a.reps)
            row = dict(dtype=dtype, kind=kind, atoms_per_frame=n_atoms[0],
                       a_loop_ms_per_frame=1e3 * ta / len(loop), a_atoms_per_s=n_loop / ta,
                       b_model_only_ms_per_frame=1e3 * tb / len(pre), b_atoms_per_s=n_loop / tb, check_rel_E=de, check_rel_F=dfm)
            for bs in a.batch:
                groups = [frames[i: i + bs] for i in range(0, len(frames), bs)]

                def run_c():
                    for grp in groups:
                        m.energy_and_forces_frames(collate(grp, r_max))

                def run_nl():
                    for grp in groups:
                        collate(grp, r_max)

                run_c()  # warm every shape of the window
                tc, tnl = timed(run_c, a.reps), timed(run_nl, a.reps)
                nf = sum(len(gp) for gp in groups)
                row[f"c{bs}_ms_per_frame"] = 1e3 * tc / nf
                row[f"c{bs}_atoms_per_s"] = sum(n_atoms[: nf]) / tc
                row[f"c{bs}_list_ms_per_frame"] = 1e3 * tnl / nf
            row["edges_per_frame"] = collate(frames[:1], r_max)[D.CSR_KEY].num_edges
            results.append(row)
            line = (f"{dtype:8s} {kind:8s} N={n_atoms[0]:3d} E={row['edges_per_frame']:5d}  (a) {row['a_loop_ms_per_frame']:7.3f} ms/frame"
                    f"  (b) {row['b_model_only_ms_per_frame']:7.3f}")
            for bs in a.batch:
                line += f"  (c,{bs}) {row[f'c{bs}_ms_per_frame']:7.4f} [list {row[f'c{bs}_list_ms_per_frame']:.4f}]"
            print(line, flush=True)
    rec = {"card": name, "power_limit": pl, "results": results}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
