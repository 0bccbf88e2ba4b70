"""Forward-mode second derivatives on the c2 frame (phonons.hessian_vector_product / analytic_force_constants) against
one force evaluation and the finite-difference force constants.

    python tools/time_hessian.py [--reps 5] [--out FILE]

On the 10 976-atom c2 frame with the fp32 c2 model (S = 64, U = 32, l_max 2, two layers, r_max 5):
  forces   one energy_and_forces (the list built once, outside the window)
  hvp      one full-frame hessian_vector_product (its own list at r_max inside the window, like a caller's), and the
           library kernel launches of each
  fc       analytic_force_constants against force_constants (h = 0.01) for one and for four displaced atoms
Times are host wall clock around work that ends in a device synchronise, median of --reps after a warm-up call.  The
card's name and power limit are printed with the numbers.
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
from allegro_b200.model import AllegroModel  # noqa: E402
from allegro_b200.phonons import analytic_force_constants, force_constants, hessian_vector_product  # noqa: E402
from time_batched_md import card  # noqa: E402

DEV = "cuda"


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_hessian.py needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}", flush=True)
    pos, cell, types = systems.make_positions("c2")
    pos, cell, types = pos.to(DEV, torch.float32), cell.to(DEV, torch.float32), types.to(DEV)
    n = pos.shape[0]
    model = AllegroModel(**systems.model_kwargs("c2", 42.0, "float32")).to(DEV)
    inner = model.model
    csr, sv = D.neighbor_csr(pos, inner.r_max, cell)
    data = {D.POSITIONS_KEY: pos, D.CELL_KEY: cell, D.ATOM_TYPE_KEY: types, D.CSR_KEY: csr, D.EDGE_SHIFT_VEC_KEY: sv}
    res = {"card": name, "power_limit_w": pl, "atoms": n, "edges": csr.num_edges}
    res["forces_ms"] = 1e3 * timed(lambda: inner.energy_and_forces(data), a.reps)
    v = torch.randn(n, 3, generator=torch.Generator().manual_seed(0)).to(DEV)
    res["hvp_ms"] = 1e3 * timed(lambda: hessian_vector_product(model, pos, cell, types, v), a.reps)
    res["hvp_over_forces"] = res["hvp_ms"] / res["forces_ms"]
    for key, fn in (("forces_launches", lambda: inner.energy_and_forces(data)), ("hvp_launches", lambda: hessian_vector_product(model, pos, cell, types, v))):
        _lib.PROF.reset()
        fn()
        res[key] = _lib.PROF.launches  # launches of the library's kernels (torch's own elementwise ops not counted)
    print(f"energy_and_forces {res['forces_ms']:.2f} ms; hessian_vector_product {res['hvp_ms']:.2f} ms "
          f"({res['hvp_over_forces']:.2f} force evaluations); library launches {res['forces_launches']} / {res['hvp_launches']}", flush=True)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    for k in (1, 4):
        atoms = perm[:k]
        t_an = timed(lambda: analytic_force_constants(model, pos, cell, types, atoms=atoms), a.reps)
        t_fd = timed(lambda: force_constants(model, pos, cell, types, atoms=atoms, displacement=0.01), a.reps)
        res[f"fc{k}_analytic_ms"], res[f"fc{k}_fd_ms"], res[f"fc{k}_ratio"] = 1e3 * t_an, 1e3 * t_fd, t_an / t_fd
        print(f"{k} displaced atom(s): analytic {1e3 * t_an:.2f} ms, finite difference {1e3 * t_fd:.2f} ms, ratio {t_an / t_fd:.2f}",
              flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
