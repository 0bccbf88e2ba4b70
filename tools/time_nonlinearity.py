"""Step time of the c2 model (fp32, full size, CUDA-graph replay) with silu, mish and gelu MLP nonlinearities.

    python tools/time_nonlinearity.py [--steps 50] [--warmup 10] [--rounds 3]

The three models share the architecture and differ only in the three nonlinearity kwargs.  Each is checked against the
fp64 oracle on bench.py's locality sub-sample before it is timed; then the rounds alternate silu, mish, gelu in one
process, and per round the ms per graph-replayed step is recorded.  The parity check is repeated with the CUDA-core
linear layers only (IEEE functions, no fused kernels), to separate the fast fp32 activations from the model's own fp32
conditioning.  A last eager pass per model times the MLP kernels
(linear, mlp2, mlp2_readout, radial_bwd) with CUDA events (_lib.PROF).  Prints one JSON object, with the card's name and
power limit.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # nonlin_oracle: the fp64 oracle with mish / gelu

import bench  # noqa: E402
import nonlin_oracle  # noqa: E402
from allegro_b200 import _lib, systems  # noqa: E402
from allegro_b200 import data as D  # noqa: E402
from allegro_b200.graph import GraphedEnergyForces  # noqa: E402
from allegro_b200.model import AllegroModel  # noqa: E402

KERNELS = ("linear", "mlp2", "mlp2_readout", "radial_bwd")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    d = systems.make_system("c2", None)
    n, e = d[D.POSITIONS_KEY].shape[0], d[D.EDGE_INDEX_KEY].shape[1]
    data = {k: v.to(dev) for k, v in d.items()}
    runs = {}
    for nl in ("silu", "mish", "gelu"):
        kw = systems.model_kwargs("c2", e / n, "float32")
        kw.update(scalar_embed_mlp_nonlinearity=nl, allegro_mlp_nonlinearity=nl, readout_mlp_nonlinearity=nl)
        model = AllegroModel(**kw).to(dev)
        graphed = GraphedEnergyForces(model, data)
        for _ in range(args.warmup):
            out = graphed()
        torch.cuda.synchronize()
        try:
            with nonlin_oracle.nonlinearities():
                parity = bench.parity_check(model, out, d, kw, "float32")
        except AssertionError as err:  # recorded and reported with the times, not hidden
            parity = {"failed": str(err)}
        # the same model with the CUDA-core linear layers only (IEEE expf / erfcf / division instead of the fast fp32
        # forms, no fused MLP kernels): tells the model's fp32 conditioning from the fast activations
        _lib.set_option("linear_tc", 0)
        try:
            with nonlin_oracle.nonlinearities():
                core = bench.parity_check(model, model(data), d, kw, "float32")
        except AssertionError as err:
            core = {"failed": str(err)}
        finally:
            _lib.set_option("linear_tc", 1)
        runs[nl] = dict(model=model, graphed=graphed, parity=parity, parity_cuda_core=core, ms=[])
    for _ in range(args.rounds):
        for nl, r in runs.items():
            for _ in range(args.warmup):
                r["graphed"]()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            for _ in range(args.steps):
                r["graphed"]()
            t1.record()
            torch.cuda.synchronize()
            r["ms"].append(t0.elapsed_time(t1) / args.steps)
    result = {"gpu": bench.gpu_info(0), "atoms": n, "edges": e, "steps": args.steps, "rounds": args.rounds, "models": {}}
    for nl, r in runs.items():
        _lib.PROF.reset()
        _lib.PROF.enabled = True
        for _ in range(10):
            r["model"](data)
        times = _lib.PROF.times_ms()
        _lib.PROF.enabled = False
        per_kernel = {}
        for key, ts in times.items():
            kern = key.partition("@")[0]
            if kern in KERNELS:
                per_kernel[kern] = per_kernel.get(kern, 0.0) + sum(ts) / 10
        result["models"][nl] = {"ms_per_step": [round(x, 4) for x in r["ms"]], "median_ms": round(statistics.median(r["ms"]), 4),
                                "eager_kernel_ms_per_step": {k: round(v, 4) for k, v in sorted(per_kernel.items())},
                                "parity": {k: r["parity"].get(k) for k in ("rel_err_E", "rel_err_F", "tol", "failed")},
                                "parity_cuda_core": {k: r["parity_cuda_core"].get(k) for k in ("rel_err_E", "rel_err_F", "failed")}}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
