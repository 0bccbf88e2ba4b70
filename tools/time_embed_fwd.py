"""The forward of the scalar-embed MLP with its first layer folded into PQ, at the c2 edge count: the two launches
(radial_pq_fwd writes h, then the embed GEMM [w0 | x_0 | omega_0] = phi(h) @ W_fold in two column slices) against the fused
kernel (ab2_radial_embed_fwd), timed with CUDA events.

    python tools/time_embed_fwd.py [--reps 30] [--out FILE.json]

Two frames with 461 154 edges and the c2 shapes (hidden width 64, N = 256 output columns in [w0 | X[:, :64] | omega_0],
the middle segment strided as in the model): one species (c2) and two species (four type pairs).  The variants alternate,
rep by rep, after a warm-up; each rep times ten launches back to back, so that the host's per-call time does not enter.
The medians are reported with bytes per edge and the achieved TB/s against each one's algorithmic bytes: the radial
kernel reads vec, ctr / nbr and two type entries (28 B) and writes h (4 H B); the GEMM reads h once per column slice and
writes the outputs (4 N B); the fused kernel reads what the radial kernel reads and writes the outputs.  Whether the two
results are bitwise equal is reported too.  Prints one JSON object (with the card's name and power limit) and writes it
to --out.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from allegro_b200 import _lib  # noqa: E402

E, N_ATOMS, SEG, LD_MID, H, P_CUT = 461154, 10976, (96, 64, 96), 192, 64, 6.0
N = sum(SEG)
GEO = 12 + 8 + 8  # vec, ctr / nbr, two type entries
BATCH = 10  # launches per timed window


def frame(T, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    ctr = (torch.arange(E) * N_ATOMS // E).to(torch.int32)  # centre-sorted, as the CSR edges are
    nbr = torch.randint(0, N_ATOMS, (E,), generator=g, dtype=torch.int32)
    types = torch.randint(0, T, (N_ATOMS,), generator=g, dtype=torch.int32)
    u = torch.randn(E, 3, generator=g)
    vec = u / u.norm(dim=1, keepdim=True) * (2.0 + 3.0 * torch.rand(E, 1, generator=g))  # |r| in [2, 5): inside r_max = 5
    a = dict(vec=vec, ctr=ctr, nbr=nbr, types=types, rmax=torch.full((T, T), 5.0), bw=torch.arange(1, 9) * math.pi,
             PQ=torch.randn(T * T, 8, H, generator=g) / 2, W=torch.randn(H, N, generator=g) / math.sqrt(H))
    a = {k: v.to(dev) for k, v in a.items()}
    a["Wp"] = _lib.linear_pack(a["W"])
    return a


def outputs(dev):
    X = torch.empty(E, LD_MID, device=dev)
    return [torch.empty(E, SEG[0], device=dev), X[:, : SEG[1]], torch.empty(E, SEG[2], device=dev)]


def radial(a):
    return _lib.radial_pq_fwd(torch.float32, H, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"])


def gemm(a, outs, h):
    _lib.linear([h], a["W"], outs, act=_lib.ACT_SILU, W_packed=a["Wp"])


def fused(a, outs):
    ok = _lib.radial_embed_fwd(torch.float32, H, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], a["Wp"], outs)
    assert ok, "the fused kernel declined the c2 shapes"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as err:  # reported, not hidden
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({err})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    slices = 2  # N = 256 runs as two 128-column slices, each reading h
    per_edge = {"radial_fwd": GEO + 4 * H, "linear": slices * 4 * H + 4 * N, "fused": GEO + 4 * N}
    per_edge["two_launches"] = per_edge["radial_fwd"] + per_edge["linear"]
    res = {"gpu": card(), "edges": E, "H": H, "N": N, "reps": args.reps, "bytes_per_edge": per_edge, "frames": {}}
    for name, T in (("c2_one_species", 1), ("two_species", 2)):
        a = frame(T, dev)
        ref, got = outputs(dev), outputs(dev)
        gemm(a, ref, radial(a))
        fused(a, got)
        torch.cuda.synchronize()
        bitwise = all(torch.equal(x, y) for x, y in zip(ref, got))
        outs = outputs(dev)
        h = radial(a)
        for _ in range(3):  # warm-up
            gemm(a, outs, radial(a))
            fused(a, outs)
        ms = {"radial_fwd": [], "linear": [], "fused": []}
        run = {"radial_fwd": lambda: radial(a), "linear": lambda: gemm(a, outs, h), "fused": lambda: fused(a, outs)}
        for _ in range(args.reps):
            for key in ms:
                ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                run[key]()  # untimed: the device is busy when the window opens
                ev[0].record()
                for _ in range(BATCH):
                    run[key]()
                ev[1].record()
                torch.cuda.synchronize()
                ms[key].append(ev[0].elapsed_time(ev[1]) / BATCH)
        med = {k: statistics.median(v) for k, v in ms.items()}
        med["two_launches"] = med["radial_fwd"] + med["linear"]
        res["frames"][name] = {
            "type_pairs": T * T,
            "ms_median": {k: round(v, 4) for k, v in med.items()},
            "TB_per_s": {k: round(E * per_edge[k] / (med[k] * 1e-3) / 1e12, 3) for k in med},
            "speedup": round(med["two_launches"] / med["fused"], 3),
            "bitwise_equal": bitwise,
        }
        del a, ref, got, outs, h
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
