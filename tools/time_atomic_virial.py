"""Cost of the per-atom virial and the heat current on the flagship frame.

    python tools/time_atomic_virial.py [--rounds 3] [--steps 50] [--reps 20] [--out FILE]

c2 at full size (10 976 atoms, 461 154 edges, S = 64, U = 32, l_max 2, two layers) in fp32, replayed from CUDA graphs in
three configurations: off (today's step) / atomic_virial / atomic_virial + heat_current.  The three graphs are captured
first and then alternated, ``--steps`` replays each per round over ``--rounds`` rounds, timed with CUDA events; the
median ms per step of each configuration is printed.  Separately the eager per-kernel cost of force_scatter against
force_virial_scatter (CUDA events around each launch, ``--reps`` eager steps each, median).  The card's name and power
limit are printed with the numbers.
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

from allegro_b200 import _lib  # noqa: E402
from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.graph import GraphedEnergyForces  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

DEV = "cuda"
CONFIGS = {"off": {}, "atomic_virial": dict(atomic_virial=True), "atomic_virial+heat_current": dict(atomic_virial=True, heat_current=True)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_atomic_virial.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}")
    d = systems.make_system("c2")
    n, e = d[D.POSITIONS_KEY].shape[0], d[D.EDGE_INDEX_KEY].shape[1]
    model = AllegroModel(**systems.model_kwargs("c2", e / n, "float32")).to(DEV)
    data = {k: v.to(DEV) for k, v in d.items()}
    data[D.VELOCITY_KEY] = torch.randn(n, 3, generator=torch.Generator().manual_seed(0), dtype=torch.float64).to(DEV)
    print(f"# c2: {n} atoms, {e} edges, fp32")
    graphs = {}
    for cfg, kw in CONFIGS.items():
        graphs[cfg] = GraphedEnergyForces(model, data, **kw)
    # the three graphs compute the same forces; the new outputs exist only where asked for
    outs = {cfg: g() for cfg, g in graphs.items()}
    torch.cuda.synchronize()
    for cfg, o in outs.items():
        assert torch.equal(o[D.FORCE_KEY], outs["off"][D.FORCE_KEY]), cfg
        assert (D.ATOMIC_VIRIAL_KEY in o) == ("atomic_virial" in cfg) and (D.HEAT_CURRENT_KEY in o) == ("heat_current" in cfg), cfg
    per = {cfg: [] for cfg in CONFIGS}
    for _ in range(3):  # warm-up replays
        for g in graphs.values():
            g()
    for r in range(a.rounds):
        for cfg, g in graphs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            for _ in range(a.steps):
                g()
            t1.record()
            torch.cuda.synchronize()
            per[cfg].append(t0.elapsed_time(t1) / a.steps)
    med = {cfg: statistics.median(v) for cfg, v in per.items()}
    for cfg in CONFIGS:
        extra = 100.0 * (med[cfg] / med["off"] - 1.0)
        print(f"graph replay  {cfg:28s} {med[cfg]:.4f} ms/step  ({extra:+.2f} % vs off)   rounds {['%.4f' % x for x in per[cfg]]}")
    # eager per-kernel cost of the scatter
    kern = {}
    for cfg, key in (("off", "force_scatter"), ("atomic_virial", "force_virial_scatter")):
        for _ in range(3):
            model.model.energy_and_forces(data, **CONFIGS[cfg])
        _lib.PROF.reset()
        _lib.PROF.enabled = True
        for _ in range(a.reps):
            model.model.energy_and_forces(data, **CONFIGS[cfg])
        times = _lib.PROF.times_ms()
        _lib.PROF.enabled = False
        ts = [t for k, v in times.items() if k.split("@")[0] == key for t in v]
        kern[key] = statistics.median(ts)
        print(f"eager kernel  {key:28s} {kern[key] * 1e3:.1f} us (median of {len(ts)})")
    rec = {"card": name, "power_limit": pl, "atoms": n, "edges": e, "dtype": "float32", "graph_ms_per_step": med, "graph_rounds_ms": per,
           "kernel_us": {k: v * 1e3 for k, v in kern.items()}}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
