"""The end of the scalar-embed MLP's backward at the c2 edge count: the two launches (hidden_grad GEMM g_h = Gout @ W2^T,
then radial_pq_bwd with aux = h) against the fused kernel (ab2_radial_pq_bwd_gemm), timed with CUDA events.

    python tools/time_upstream_bwd.py [--reps 30] [--out FILE.json]

Two frames with 461 154 edges and the c2 shapes (Gout = [gw0 | gX[:, :64] | gomega], K = 256, the middle segment strided
as in the model, hidden width 64): one species (c2) and two species (c4-like, four type pairs).  The two variants
alternate, rep by rep, after a warm-up; the medians are reported with the achieved GB/s against each variant's algorithmic
bytes: per edge, the GEMM reads Gout and writes g_h, the adjoint reads g_h, h, vec, ctr / nbr and updates gvec; the fused
kernel reads Gout, vec, ctr / nbr and updates gvec.  The largest difference of the two gvec results, relative to the largest
gvec increment, is reported too.  Prints one JSON object (with the card's name and power limit) and writes it to --out.
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


def frame(T, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    ctr = (torch.arange(E) * N_ATOMS // E).to(torch.int32)  # centre-sorted, as the CSR edges are
    nbr = torch.randint(0, N_ATOMS, (E,), generator=g, dtype=torch.int32)
    types = torch.randint(0, T, (N_ATOMS,), generator=g, dtype=torch.int32)
    u = torch.randn(E, 3, generator=g)
    vec = u / u.norm(dim=1, keepdim=True) * (2.0 + 3.0 * torch.rand(E, 1, generator=g))  # |r| in [2, 5): inside r_max = 5
    K = sum(SEG)
    X = torch.randn(E, LD_MID, generator=g)
    a = dict(vec=vec, ctr=ctr, nbr=nbr, types=types, rmax=torch.full((T, T), 5.0), bw=torch.arange(1, 9) * math.pi,
             PQ=torch.randn(T * T, 8, H, generator=g) / 2, WT=torch.randn(K, H, generator=g) / math.sqrt(K),
             gw0=torch.randn(E, SEG[0], generator=g), X=X, gom=torch.randn(E, SEG[2], generator=g))
    a = {k: v.to(dev) for k, v in a.items()}
    a["gouts"] = [a["gw0"], a["X"][:, : SEG[1]], a["gom"]]
    a["WTp"] = _lib.linear_pack(a["WT"])
    a["h"] = _lib.radial_pq_fwd(torch.float32, H, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"])
    return a


def two_launches(a, gvec):
    g_h = torch.empty(E, H, device=gvec.device)
    _lib.linear(a["gouts"], a["WT"], [g_h], W_packed=a["WTp"])
    _lib.radial_pq_bwd(torch.float32, H, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], g_h, a["h"], gvec)


def fused(a, gvec):
    ok = _lib.radial_pq_bwd(torch.float32, H, P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], None, a["h"], gvec,
                            gemm=(a["gouts"], a["WTp"]))
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
    K = sum(SEG)
    bytes_two = E * ((K + H) * 4 + (2 * H * 4 + 12 + 8 + 24))  # GEMM: Gout, g_h; adjoint: g_h, h, vec, ctr / nbr, gvec read + write
    bytes_fused = E * (K * 4 + 12 + 8 + 24)
    res = {"gpu": card(), "edges": E, "K": K, "H": H, "reps": args.reps, "frames": {}}
    for name, T in (("c2_one_species", 1), ("c4_like_two_species", 2)):
        a = frame(T, dev)
        g0 = torch.zeros(E, 3, device=dev)
        g_two, g_fused = g0.clone(), g0.clone()
        two_launches(a, g_two)
        fused(a, g_fused)
        torch.cuda.synchronize()
        rel = float((g_fused - g_two).abs().max() / g_two.abs().max())
        ms = {"two_launches": [], "fused": []}
        gvec = torch.zeros(E, 3, device=dev)
        for _ in range(3):  # warm-up
            two_launches(a, gvec)
            fused(a, gvec)
        for _ in range(args.reps):
            for key, fn in (("two_launches", two_launches), ("fused", fused)):
                ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev[0].record()
                fn(a, gvec)
                ev[1].record()
                torch.cuda.synchronize()
                ms[key].append(ev[0].elapsed_time(ev[1]))
        med = {k: statistics.median(v) for k, v in ms.items()}
        res["frames"][name] = {
            "type_pairs": T * T,
            "ms_median": med,
            "ms_min": {k: min(v) for k, v in ms.items()},
            "algorithmic_bytes": {"two_launches": bytes_two, "fused": bytes_fused},
            "GB_per_s": {"two_launches": bytes_two / med["two_launches"] / 1e6, "fused": bytes_fused / med["fused"] / 1e6},
            "speedup": med["two_launches"] / med["fused"],
            "gvec_max_rel_diff": rel,
        }
        del a
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
