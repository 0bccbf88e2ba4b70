"""A committee of K models (committee.Committee) against K separate calculators, and the statistics kernels alone.

    python tools/time_committee.py [--ks 1 2 4] [--steps 50] [--reps 3] [--frames 512] [--out FILE]

  c2    the fp32 c2 model (10 976 Cu atoms, S = 64, U = 32, l_max 2, two layers, r_max 5, skin 0.5), K seeds:
        AllegroCalculator(Committee(K members)) against K AllegroCalculators, one per member, on the same positions
        (no rebuild inside the timed window: both arms replay their graphs)
  si64  the --frames 64-atom Si frames of tools/time_batched_md.py at K = 4: BatchedCalculator(Committee) against four
        BatchedCalculators
  stats ab2_committee_moments (G = 3 and G = 1) and ab2_frame_extrema at c2 size, K members, CUDA events over many launches
The arms alternate inside each of --reps passes; step times are host wall clock around steps that end in a device
synchronise, best and median over the passes.  torch.cuda.max_memory_allocated is read after each arm is built and has
run, from a reset peak.  The card's name and power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from allegro_b200 import _lib  # noqa: E402
from allegro_b200 import data as D  # noqa: E402
from allegro_b200 import systems  # noqa: E402
from allegro_b200.calculator import AllegroCalculator, BatchedCalculator  # noqa: E402
from allegro_b200.committee import Committee  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402
from time_batched_md import card, make_frames  # noqa: E402

DEV = "cuda"


def members(K):
    return [AllegroModel(**systems.model_kwargs("c2", 40.0, "float32", seed=100 + k)).to(DEV) for k in range(K)]


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def peak_after(build, run):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    obj = build()
    run(obj)
    torch.cuda.synchronize()
    return obj, torch.cuda.max_memory_allocated() - base


def compare(name, build_c, build_s, step_c, step_s, steps, reps, warmup):
    c, mem_c = peak_after(build_c, lambda o: [step_c(o) for _ in range(warmup)])
    s, mem_s = peak_after(build_s, lambda o: [step_s(o) for _ in range(warmup)])
    tc, ts = [], []
    for _ in range(reps):
        tc.append(timed(lambda: step_c(c), steps))
        ts.append(timed(lambda: step_s(s), steps))
    return c, s, dict(case=name, committee_ms_best=1e3 * min(tc), committee_ms_median=1e3 * statistics.median(tc),
                      separate_ms_best=1e3 * min(ts), separate_ms_median=1e3 * statistics.median(ts),
                      committee_peak_MiB=mem_c / 2**20, separate_peak_MiB=mem_s / 2**20)


def kernel_ms(fn, iters=200):
    for _ in range(10):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--batched-k", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_committee.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}", flush=True)
    results = []

    # c2: one committee calculator against K single-model calculators
    pos, cell, types = systems.make_positions("c2")
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    for K in a.ks:
        ms = members(K)
        r_max = float(ms[0].model.r_max)
        c, s, row = compare(
            f"c2 K={K}",
            lambda: AllegroCalculator(Committee(ms), r_max, skin=0.5),
            lambda: [AllegroCalculator(m, r_max, skin=0.5) for m in ms],
            lambda o: o.compute(pos, cell, types),
            lambda o: [x.compute(pos, cell, types) for x in o],
            a.steps, a.reps, a.warmup)
        F_c = c.compute(pos, cell, types)["forces"].double()
        F_s = torch.stack([x.compute(pos, cell, types)["forces"].double() for x in s]).mean(0)
        row.update(K=K, atoms=int(pos.shape[0]), check_rel_F=float((F_c - F_s).abs().max() / F_s.abs().max()),
                   launches_committee=c._graphed.launches_per_replay, launches_separate=sum(x._graphed.launches_per_replay for x in s))
        results.append(row)
        print(json.dumps(row), flush=True)
        del c, s, ms
        torch.cuda.empty_cache()

    # the statistics kernels alone at c2 size
    n = int(pos.shape[0])
    g = torch.Generator(device=DEV).manual_seed(3)
    fp = torch.tensor([0, n], dtype=torch.int32, device=DEV)
    for K in a.ks:
        F = [torch.randn(n, 3, generator=g, device=DEV) for _ in range(K)]
        E = [torch.randn(n, 1, generator=g, device=DEV) for _ in range(K)]
        sig = torch.rand(n, generator=g, device=DEV)
        row = dict(case=f"stats c2 K={K}", K=K, atoms=n,
                   moments_G3_us=1e3 * kernel_ms(lambda: _lib.committee_moments(F, 3)),
                   moments_G1_us=1e3 * kernel_ms(lambda: _lib.committee_moments(E, 1)),
                   frame_extrema_us=1e3 * kernel_ms(lambda: _lib.frame_extrema(sig, fp)))
        # bytes of the G = 3 call: K inputs read, the mean and the deviation written
        row["moments_G3_GBps"] = (K * n * 12 + n * 12 + n * 4) / (row["moments_G3_us"] * 1e-6) / 1e9
        results.append(row)
        print(json.dumps(row), flush=True)

    # si64 frames: one committee BatchedCalculator against K BatchedCalculators
    K = a.batched_k
    ms = members(K)
    r_max = float(ms[0].model.r_max)
    frames, _ = make_frames("si64", a.frames, seed=11)
    pos_b = torch.cat([f[D.POSITIONS_KEY] for f in frames])
    c, s, row = compare(
        f"si64 B={a.frames} K={K}",
        lambda: BatchedCalculator(Committee(ms), frames, r_max, skin=0.5),
        lambda: [BatchedCalculator(m, frames, r_max, skin=0.5) for m in ms],
        lambda o: o.compute(pos_b),
        lambda o: [x.compute(pos_b) for x in o],
        a.steps, a.reps, a.warmup)
    F_c = c.compute(pos_b)["forces"].double()
    F_s = torch.stack([x.compute(pos_b)["forces"].double() for x in s]).mean(0)
    row.update(K=K, frames=a.frames, atoms=int(pos_b.shape[0]), check_rel_F=float((F_c - F_s).abs().max() / F_s.abs().max()),
               n_captures=c.n_captures)
    results.append(row)
    print(json.dumps(row), flush=True)

    rec = {"card": name, "power_limit": pl, "model": "c2 fp32", "skin": 0.5, "results": results}
    print(json.dumps(rec))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rec, fh, indent=1)


if __name__ == "__main__":
    main()
