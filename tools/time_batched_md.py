"""Molecular dynamics of many small frames: calculator.BatchedCalculator (one graph, in-graph Verlet-list rebuilds)
against the two ways the project could run the same trajectories before it.

    python tools/time_batched_md.py [--frames 64 512] [--kinds si64 fcc32 mixed] [--steps 100] [--reps 3]
                                    [--loop-frames 16] [--temperature 600] [--out FILE]

The fp32 c2 model (S = 64, U = 32, l_max 2, two layers, r_max 5, skin 0.5) on seeded frames: 64-atom Si diamond cells,
sheared 32-atom FCC cells, or the two alternating ("mixed").  Velocity Verlet at 1 fs with a per-step velocity
rescale to --temperature (the caller's thermostat; the calculators own none), started from the same velocities for
every arm:
  (s) BatchedCalculator.compute per step                                  -> ms/step, atom-steps/s, rebuilds per frame,
                                                                             padded / real edges, overflow re-captures
  (a) one AllegroCalculator (graph replay, re-capture per rebuild) per frame, on the first --loop-frames frames, scaled
      to the whole batch
  (b) batch.collate (exact r_max list) + energy_and_forces_frames, rebuilt every step
The arms alternate inside each of --reps passes of --steps steps; times are host wall clock around steps that end in a
device synchronise, best and median over the passes.  Before timing, (s) is checked against (b) on the same positions.
The card's name and power limit are printed with the numbers.
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

from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.batch import collate  # noqa: E402
from allegro_b200.calculator import AllegroCalculator, BatchedCalculator  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

DEV = "cuda"
KB = 8.617333e-5          # eV / K
ACC = 9.64853e-3          # eV / (A amu) -> A / fs^2
MASS = {"si64": 28.086, "fcc32": 63.546}


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
    frames, masses = [], []
    for i in range(count):
        k = kind if kind != "mixed" else ("si64", "fcc32")[i % 2]
        if k == "si64":
            pos, cell = systems._lattice(systems._DIAMOND, 5.431, (2, 2, 2), 0.05, g)
        else:
            pos, cell = systems._lattice(systems._FCC, 3.615, (2, 2, 2), 0.05, g)
            shear = torch.eye(3, dtype=torch.float64)
            shear[1, 0], shear[2, 0], shear[2, 1] = 0.1 + 0.1 * float(torch.rand(1, generator=g)), -0.15, 0.12
            pos, cell = pos @ shear, cell @ shear
        frames.append({D.POSITIONS_KEY: pos.to(DEV, torch.float32), D.ATOM_TYPE_KEY: torch.zeros(pos.shape[0], dtype=torch.long, device=DEV),
                       D.CELL_KEY: cell.to(DEV, torch.float32)})
        masses.append(torch.full((pos.shape[0], 1), MASS[k], dtype=torch.float32))
    return frames, torch.cat(masses).to(DEV)


class Verlet:
    """velocity Verlet at dt fs with a velocity rescale to T0 every step (all on the device, no host read)"""

    def __init__(self, pos, mass, T0, seed, dt=1.0):
        g = torch.Generator().manual_seed(seed)
        self.pos, self.mass, self.T0, self.dt = pos.clone(), mass, T0, dt
        self.vel = (torch.randn(pos.shape, generator=g) * (KB * T0 * ACC / mass.cpu()).sqrt()).to(DEV)
        self.F = None

    def step(self, forces_of):
        if self.F is None:
            self.F = forces_of(self.pos)
        self.vel += 0.5 * self.dt * self.F / self.mass * ACC
        self.pos += self.dt * self.vel
        self.F = forces_of(self.pos)
        self.vel += 0.5 * self.dt * self.F / self.mass * ACC
        T = (self.mass * self.vel * self.vel).sum() / (3 * self.pos.shape[0] * KB * ACC)
        self.vel *= (self.T0 / T.clamp(min=1e-6)).sqrt()


def timed_steps(traj, forces_of, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        traj.step(forces_of)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--kinds", nargs="+", default=["si64", "fcc32", "mixed"])
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-frames", type=int, default=16)
    ap.add_argument("--temperature", type=float, default=600.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_batched_md.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}")
    model = AllegroModel(**systems.model_kwargs("c2", 40.0, "float32")).to(DEV)
    m = model.model
    r_max, skin = float(m.r_max), 0.5
    results = []
    for kind in a.kinds:
        for B in a.frames:
            frames, mass = make_frames(kind, B, seed=11)
            n_atoms = sum(f[D.POSITIONS_KEY].shape[0] for f in frames)
            pos0 = torch.cat([f[D.POSITIONS_KEY] for f in frames])
            calc = BatchedCalculator(model, frames, r_max, skin=skin)

            def forces_s(p):
                return calc.compute(p)["forces"]

            def forces_b(p):
                fs, o = [], 0
                for f in frames:
                    k = f[D.POSITIONS_KEY].shape[0]
                    g = dict(f)
                    g[D.POSITIONS_KEY] = p[o:o + k]
                    fs.append(g)
                    o += k
                return m.energy_and_forces_frames(collate(fs, r_max))[D.FORCE_KEY]

            L = min(a.loop_frames, B)
            n_loop = sum(f[D.POSITIONS_KEY].shape[0] for f in frames[:L])
            singles = [AllegroCalculator(model, r_max, skin=skin, pbc=(True, True, True)) for _ in range(L)]
            offs = [0]
            for f in frames[:L]:
                offs.append(offs[-1] + f[D.POSITIONS_KEY].shape[0])

            def forces_a(p):
                return torch.cat([singles[i].compute(p[offs[i]:offs[i + 1]], frames[i][D.CELL_KEY], frames[i][D.ATOM_TYPE_KEY])["forces"]
                                  for i in range(L)])

            # (s) against (b) on the same positions, before any timing
            fs_, fb_ = forces_s(pos0).double(), forces_b(pos0).double()
            check = float((fs_ - fb_).abs().max() / fb_.abs().max())
            assert check < 1e-4, check
            ts, ta, tb = Verlet(pos0, mass, a.temperature, 1), Verlet(pos0[:n_loop], mass[:n_loop], a.temperature, 1), Verlet(pos0, mass, a.temperature, 1)
            for traj, fn in ((ts, forces_s), (ta, forces_a), (tb, forces_b)):
                timed_steps(traj, fn, a.warmup)
            r0, caps0 = calc.frame_rebuilds(), calc.n_captures
            t_s, t_a, t_b = [], [], []
            for _ in range(a.reps):
                t_s.append(timed_steps(ts, forces_s, a.steps))
                t_a.append(timed_steps(ta, forces_a, a.steps) * B / L)
                t_b.append(timed_steps(tb, forces_b, a.steps))
            r1 = calc.frame_rebuilds()
            timed_total = a.reps * a.steps
            real = calc.real_edges()
            row = dict(kind=kind, frames=B, atoms=n_atoms, steps_timed=timed_total, check_rel_F=check,
                       s_ms_per_step_best=1e3 * min(t_s), s_ms_per_step_median=1e3 * statistics.median(t_s),
                       s_atom_steps_per_s=n_atoms / min(t_s),
                       s_rebuilds_per_frame=sum(y - x for x, y in zip(r0, r1)) / B, s_rebuild_interval_steps=(timed_total * B / max(1, sum(y - x for x, y in zip(r0, r1)))),
                       s_padded_over_real_edges=(calc.num_edges - real) / max(real, 1), s_edges=calc.num_edges, s_real_edges=real,
                       s_overflow_recaptures=calc.n_captures - caps0, s_overflows_total=calc.n_overflows,
                       a_loop_frames=L, a_ms_per_step_scaled_best=1e3 * min(t_a), a_ms_per_step_scaled_median=1e3 * statistics.median(t_a),
                       a_atom_steps_per_s=n_atoms / min(t_a),
                       b_ms_per_step_best=1e3 * min(t_b), b_ms_per_step_median=1e3 * statistics.median(t_b), b_atom_steps_per_s=n_atoms / min(t_b))
            results.append(row)
            print(f"{kind:6s} B={B:4d} N={n_atoms:6d}  (s) {row['s_ms_per_step_best']:8.3f} ms/step {row['s_atom_steps_per_s']:.3e} atom-steps/s"
                  f"  rebuilds/frame {row['s_rebuilds_per_frame']:.2f}  pad/real {row['s_padded_over_real_edges']:.3f}"
                  f"  recaptures {row['s_overflow_recaptures']}  |  (a) {row['a_ms_per_step_scaled_best']:9.3f}  (b) {row['b_ms_per_step_best']:8.3f}",
                  flush=True)
            del calc, singles
            torch.cuda.empty_cache()
    rec = {"card": name, "power_limit": pl, "model": "c2 fp32", "skin": skin, "temperature_K": a.temperature, "results": results}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
