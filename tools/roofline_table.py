"""Per-op roofline table from a bench.py JSON line (its `kernels_ms_per_step` leg) -- post-processing only.

    python tools/roofline_table.py bench_line.json [--peak 3350]

Algorithmic bytes are the unavoidable global traffic of each op of the per-kernel pipeline (DESIGN.md section 4):
inputs read once, outputs written once, in the storage dtype; epilogue operands (silu' pre-activations, accumulated
gradients) count as reads.  The table shows where the step is relative to the HBM roofline op by op.
"""
import argparse
import json
import re
import sys


def mlp_fwd(E, b, dims):
    """2-or-more-layer MLP as separate GEMMs: every layer reads its input and writes its output."""
    return sum(E * b * (k + n) for k, n in zip(dims, dims[1:]))


def mlp_bwd(E, b, dims, accum_in=0):
    """legacy plan: g_h = (g_out W^T) * silu'(pre) per hidden layer (reads g_out, pre; writes g_h), last GEMM writes
    g_in (plus `accum_in` columns read for accumulation)."""
    tot = 0
    for k, n in reversed(list(zip(dims, dims[1:]))):
        tot += E * b * (n + k)          # read g_out[n], write g_in[k]
        if k != dims[0]:
            tot += E * b * k            # silu' epilogue reads pre[k]
    return tot + E * b * accum_in


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("json")
    ap.add_argument("--peak", type=float, default=None, help="HBM GB/s (default: roofline.peak of the JSON)")
    a = ap.parse_args()
    d = json.loads(open(a.json).read().strip().splitlines()[-1])
    w = d["config"]["workload"]
    E = int(re.search(r"(\d+) edges", w).group(1))
    N = int(re.search(r"(\d+) atoms", w).group(1))
    lmax = int(re.search(r"l_max=(\d+)", w).group(1))
    L = int(re.search(r"n_layers=(\d+)", w).group(1))
    S = int(re.search(r"S=(\d+)", w).group(1))
    U = int(re.search(r"U=(\d+)", w).group(1))
    b = {"f64": 8, "f32": 4, "bf16": 2}[d["dtype"]]
    acc = 8 if d["dtype"] == "f64" else 4
    D, n_ir = (lmax + 1) ** 2, lmax + 1
    nw, W = n_ir * U, S  # hidden widths = S in the benchmark configs
    peak = a.peak or d["roofline"]["peak"]
    per_edge_tp0 = b * nw + acc * D + 4 + b * U * D
    # round 2: the first scalar-embed layer is folded into the radial kernel (it emits the pre-activation h [E, W]) and the
    # embed linears into the MLP's last layer: upstream = radial kernel + ONE GEMM W -> (nw + S + nw) per direction
    folded = "radial_fwd@fwd.embed" in d["kernels_ms_per_step"] or "radial_fwd@fwd.radial" not in d["kernels_ms_per_step"]
    ops = {
        "radial_fwd@fwd.radial": E * (acc * 3 + 8 + b * S),
        "radial_fwd@fwd.embed": E * (acc * 3 + 8 + b * W),
        "linear@fwd.radial": mlp_fwd(E, b, [S, W, S]),
        "linear@fwd.embed": E * b * ((W if folded else S) + nw + S + nw),
        "sh_fwd@fwd.embed": E * acc * (3 + D),
        "edge_vec@fwd.radial": E * (8 + acc * 3),
        "linear@fwd.readout": mlp_fwd(E, b, [S * (L + 1), W, 1]),
        "linear@bwd.readout": mlp_bwd(E, b, [S * (L + 1), W, 1]),
        "linear@bwd.embed": E * b * (nw + S + nw + S),
        "linear@bwd.radial": (E * b * (nw + S + nw + W)) if folded else mlp_bwd(E, b, [S, W, S]),
        "radial_bwd@bwd.radial": E * (acc * 6 + 8 + (2 * b * W if folded else b * S)),
        "sh_bwd@bwd.embed": E * acc * (3 + D + 3),
        "edge_sum@fwd.readout": E * acc + N * acc,
        "edge_sum_bwd@bwd.readout": E * acc + N * acc,
        "force_scatter@bwd.radial": E * (acc * 3 + 4) + 2 * N * acc * 3,
    }
    for l in range(L):
        last = l == L - 1
        d_in = D  # benchmark configs: pruned irreps of the inner layers = the SH irreps
        d_out = 1 if last else D
        ops[f"env_sum@fwd.L{l}"] = E * (b * nw + acc * D) + N * acc * D * U
        ops[f"env_bwd@bwd.L{l}"] = E * (2 * b * nw + 3 * acc * D) + N * acc * D * U
        if l == 0:
            ops["tp_fwd@fwd.L0"] = E * (b * nw + acc * D + 4 + b * U * d_out) + N * acc * D * U
            ops["tp_bwd@bwd.L0"] = E * (2 * b * nw + 3 * acc * D + 4 + b * U * d_out) + 2 * N * acc * D * U
        else:
            ops[f"tp_fwd@fwd.L{l}"] = E * (b * U * d_in + b * U * d_out + 4) + N * acc * D * U
            ops[f"tp_bwd@bwd.L{l}"] = E * (2 * b * U * d_in + b * U * d_out + 4) + 2 * N * acc * D * U
        dims = [S * (l + 1) + U, W, S + (0 if last else nw)]
        ops[f"linear@fwd.L{l}"] = mlp_fwd(E, b, dims)
        ops[f"linear@bwd.L{l}"] = mlp_bwd(E, b, dims, accum_in=S * (l + 1) + (0 if last else U))
    # last latent MLP + readout in one kernel (ab2_mlp2_readout), P = S L, both hidden widths W:
    #   forward  reads X[:, :P], s; writes pre_L, x_L, pre_r, Ez
    #   backward reads gEz, pre_r, pre_L; writes gX[:, :P], gs
    P = S * L
    ops["mlp2_readout@fwd.L%d" % (L - 1)] = E * b * (P + U + W + S + W + 1)
    ops["mlp2_readout@bwd.readout"] = E * b * (1 + W + W + P + U)
    # two-layer models: the tensor products composed per centre (ab2_tp_chain_*), no V_1 / gV_1; per edge Y, w0 and the
    # compact [E][U] scalars or their gradients, per centre the gamma rows read and (backward) ggamma written
    per_edge_chain = b * nw + acc * D + 4
    ops["tp_chain_fwd@fwd.L0"] = E * (per_edge_chain + b * U) + N * acc * D * U
    ops["tp_chain_fwd@fwd.L1"] = E * (per_edge_chain + b * U) + 2 * N * acc * D * U
    ops["tp_chain_bwd@bwd.L1"] = E * (per_edge_chain + b * U) + 2 * N * acc * D * U
    ops["tp_chain_bwd@bwd.L0"] = E * (2 * b * nw + 3 * acc * D + 4 + 2 * b * U) + 3 * N * acc * D * U
    k = d["kernels_ms_per_step"]
    rows, tot_ms, tot_b = [], 0.0, 0
    for name, ms in sorted(k.items(), key=lambda kv: -kv[1]):
        by = ops.get(name)
        tot_ms += ms
        if by is None:
            rows.append((name, ms, None, None, None))
            continue
        tot_b += by
        gbs = by / ms / 1e6
        rows.append((name, ms, by / 1e6, gbs, gbs / peak))
    print(f"| op | ms/step | algorithmic MB | GB/s | frac of {peak:.0f} GB/s |")
    print("|---|---|---|---|---|")
    for name, ms, mb, gbs, fr in rows:
        print(f"| {name} | {ms:.3f} | {'' if mb is None else f'{mb:.0f}'} | {'' if gbs is None else f'{gbs:.0f}'} | {'' if fr is None else f'{fr:.2f}'} |")
    print(f"| **sum of kernels** | {tot_ms:.3f} | {tot_b / 1e6:.0f} | {tot_b / tot_ms / 1e6:.0f} | {tot_b / tot_ms / 1e6 / peak:.2f} |")
    print(f"\nstep (graph replay): {d['ms_per_step']:.3f} ms; all algorithmic bytes at peak: {tot_b / peak / 1e6:.3f} ms")


if __name__ == "__main__":
    sys.exit(main())
