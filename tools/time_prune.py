"""Time the per-edge-type pruning of the neighbour list (ab2_nl_prune_count / fill) and what it buys per step.

    python tools/time_prune.py [--rounds 3] [--steps 20] [--frames c3,c4] [--out /tmp/time_prune.json]

Two frames, fp32 models with per-edge-type cutoffs:
  c3   Li/P/S 46^3 = 97 336 atoms, r_max 6, {"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}
  c4   water-like, 40^3 O + 2 H each = 192 000 atoms, r_max 5, {"O": {"O": 5.0, "H": 4.5}, "H": 4.0}
For each: directed edges before and after pruning; the list build (data.neighbor_csr at r_max) with and without the
prune pass, and the prune pass alone (CUDA events around synchronised calls, median of 10); the graph-replayed step
(energy_and_forces) on the unpruned and on the pruned list, alternated over ``--rounds`` rounds in this one process,
and the largest difference between their energies and forces.  The card's name and power limit are recorded beside the
numbers.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.graph import GraphedEnergyForces  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

FRAMES = {
    "c3": dict(scale=None, table={"Li": 4.0, "P": {"Li": 5.0, "P": 4.5, "S": 6.0}, "S": 5.5}),
    "c4": dict(scale=40, table={"O": {"O": 5.0, "H": 4.5}, "H": 4.0}),
}


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        power = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "unknown"
    except (OSError, subprocess.SubprocessError, IndexError):
        power = "unknown"
    return {"gpu": name, "power_limit_and_max_sm_clock": power}


def _ms(fn, reps=10):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def run(name, rounds, steps):
    cfg = FRAMES[name]
    pos, cell, types = systems.make_positions(name, cfg["scale"])
    dev = torch.device("cuda")
    pos, cell, types = pos.to(dev, torch.float32), cell.to(dev, torch.float32), types.to(dev)
    n = pos.shape[0]
    r_max = systems.CONFIGS[name]["r_max"]
    kw = systems.model_kwargs(name, 40.0, "float32")
    kw.update(per_edge_type_cutoff=cfg["table"])
    model = AllegroModel(**kw).to(dev).model
    tab = model.edge_norm.rmax_table
    pbc = (True, True, True)

    csr, sv = D.neighbor_csr(pos, r_max, cell, pbc)
    pcsr, psv = D.prune_csr(csr, sv, pos, types, tab)
    res = {"frame": name, "atoms": n, "r_max": r_max, "table": cfg["table"], "edges": csr.num_edges, "edges_pruned": pcsr.num_edges,
           "edges_per_atom": csr.num_edges / n, "edges_per_atom_pruned": pcsr.num_edges / n, "kept_fraction": pcsr.num_edges / csr.num_edges}
    for _ in range(2):  # warm-up of both paths
        D.neighbor_csr(pos, r_max, cell, pbc, types=types, cutoffs=tab)
    res["build_ms"] = _ms(lambda: D.neighbor_csr(pos, r_max, cell, pbc))
    res["build_and_prune_ms"] = _ms(lambda: D.neighbor_csr(pos, r_max, cell, pbc, types=types, cutoffs=tab))
    res["prune_only_ms"] = _ms(lambda: D.prune_csr(csr, sv, pos, types, tab))

    def data(c, s):
        return {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.CSR_KEY: c, D.EDGE_SHIFT_VEC_KEY: s}

    lists = {"unpruned": (csr, sv), "pruned": (pcsr, psv)}
    outs, times = {}, {k: [] for k in lists}
    for rnd in range(rounds):
        for k, (c, s) in lists.items():  # alternated in the same process; one captured graph at a time (HBM)
            g = GraphedEnergyForces(model, data(c, s))
            o = g(pos)
            torch.cuda.synchronize()
            if rnd == 0:
                outs[k] = {q: o[q].double().clone() for q in (D.TOTAL_ENERGY_KEY, D.FORCE_KEY)}
            for _ in range(3):
                g(pos)

            def replay(g=g):
                for _ in range(steps):
                    g(pos)

            times[k].append(_ms(replay, reps=3) / steps)
            del g, o, replay
            torch.cuda.empty_cache()
    f_ref = outs["unpruned"][D.FORCE_KEY]
    res["max_abs_force_diff"] = float((outs["pruned"][D.FORCE_KEY] - f_ref).abs().max())
    res["max_abs_force"] = float(f_ref.abs().max())
    res["energy_diff"] = float((outs["pruned"][D.TOTAL_ENERGY_KEY] - outs["unpruned"][D.TOTAL_ENERGY_KEY]).abs().max())
    res["energy"] = float(outs["unpruned"][D.TOTAL_ENERGY_KEY].reshape(-1)[0])
    res["step_ms_rounds"] = times
    res["step_ms"] = {k: statistics.median(v) for k, v in times.items()}
    res["step_ratio_pruned_over_unpruned"] = res["step_ms"]["pruned"] / res["step_ms"]["unpruned"]
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--frames", default="c3,c4")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_prune.py needs a CUDA device")
    out = {"card": card(), "results": []}
    for f in a.frames.split(","):
        try:
            out["results"].append(run(f, a.rounds, a.steps))
        except torch.OutOfMemoryError as e:  # recorded, not measured
            out["results"].append({"frame": f, "not_measured": f"out of memory: {str(e).splitlines()[0]}"})
            torch.cuda.empty_cache()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
