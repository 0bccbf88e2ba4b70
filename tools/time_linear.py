"""Micro-benchmark of ab2_linear on the GPU (tensor-core vs CUDA-core path, stage knock-outs).

    python tools/time_linear.py --mlp2   # ab2_mlp2 against the two launches it replaces, c2 shapes
"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from allegro_b200 import _lib

M = 461154
dev = "cuda"
shapes = [([64], [96, 64, 96]), ([64], [64, 96]), ([64, 32], [64]), ([64, 64, 64], [64]), ([64], [64]), ([96, 64, 96], [64])]


def run(awid, owid, dtype, debug=0, tc=True, epi=0, accum=False, reps=10):
    K, N = sum(awid), sum(owid)
    a = [torch.randn(M, w, device=dev, dtype=dtype) for w in awid]
    W = torch.randn(K, N, device=dev, dtype=dtype) * 0.1
    o = [torch.zeros(M, w, device=dev, dtype=dtype) for w in owid]
    aux = torch.randn(M, N, device=dev, dtype=dtype) if epi else None
    pk = _lib.linear_pack(W) if tc else None
    _lib.set_option("tc_debug", debug)
    acc = [accum] * len(owid)
    for _ in range(3):
        _lib.linear(a, W, o, o_accum=acc, epi=epi, aux=aux, W_packed=pk)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        _lib.linear(a, W, o, o_accum=acc, epi=epi, aux=aux, W_packed=pk)
    t1.record()
    torch.cuda.synchronize()
    _lib.set_option("tc_debug", 0)
    ms = t0.elapsed_time(t1) / reps
    esz = 4 if dtype == torch.float32 else 2
    byts = M * (K + N * (2 if accum else 1) + (N if epi else 0)) * esz
    return ms, byts / ms / 1e6


def time_ms(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


# the c2 two-layer SiLU MLPs: (name, backward, A widths, hidden width, output widths, output accumulate flags)
mlp2_shapes = [
    ("fwd.L0", False, [64, 32], 64, [64, 96], [False, False]),
    ("fwd.L1", False, [128, 32], 64, [64], [False]),
    ("fwd.readout", False, [192], 64, [1], [False]),
    ("bwd.readout", True, [1], 64, [192], [False]),
    ("bwd.L1", True, [64], 64, [128, 32], [True, False]),
    ("bwd.L0", True, [64, 96], 64, [64, 32], [True, True]),
]


def run_mlp2(name, backward, awid, H, owid, accum):
    """ab2_mlp2 against the two ab2_linear launches it replaces (the pair as PackedMLP ran it before)."""
    K, N = sum(awid), sum(owid)
    a = [torch.randn(M, w, device=dev) for w in awid]
    W1, W2 = torch.randn(K, H, device=dev) * 0.1, torch.randn(H, N, device=dev) * 0.1
    o = [torch.zeros(M, w, device=dev) for w in owid]
    pre = torch.randn(M, H, device=dev)
    h = torch.empty(M, H, device=dev)
    p1, p2 = _lib.linear_pack(W1), _lib.linear_pack(W2)

    def fused():
        assert _lib.mlp2(a, W1, W2, o, pre, o_accum=accum, backward=backward, W1_packed=p1, W2_packed=p2)

    if not backward:
        def pair():
            _lib.linear(a, W1, [h], W_packed=p1)
            _lib.linear([h], W2, o, o_accum=accum, act=_lib.ACT_SILU, W_packed=p2)
    elif K == 1:  # readout: one gradient column, zero-padded to K = 16
        W1p = torch.zeros(16, H, device=dev)
        W1p[:1] = W1
        p1p = _lib.linear_pack(W1p)

        def pair():
            gp = torch.zeros(M, 16, device=dev)
            gp[:, :1] = a[0]
            _lib.linear([gp], W1p, [h], epi=_lib.EPI_MUL_DSILU, aux=pre, W_packed=p1p)
            _lib.linear([h], W2, o, o_accum=accum, W_packed=p2)
    else:
        def pair():
            _lib.linear(a, W1, [h], epi=_lib.EPI_MUL_DSILU, aux=pre, W_packed=p1)
            _lib.linear([h], W2, o, o_accum=accum, W_packed=p2)
    t_pair, t_fused = time_ms(pair), time_ms(fused)
    floats = K + H + N + sum(w for w, ac in zip(owid, accum) if ac)  # fused kernel's HBM traffic (pre written or read)
    print(f"mlp2 {name:12s} K={K:3d} H={H} N={N:3d}: two launches {t_pair*1e3:6.0f}us  fused {t_fused*1e3:6.0f}us "
          f"({M * floats * 4 / t_fused / 1e6:5.0f}GB/s)  {t_pair / t_fused:4.2f}x", flush=True)


if "--mlp2" in sys.argv:
    for shp in mlp2_shapes:
        run_mlp2(*shp)
    sys.exit(0)

shapes += [([128], [192, 128, 192]), ([128, 64], [128]), ([128], [128, 192]), ([192, 128, 192], [128])]  # c3-sized layers
for tma in (1, 0):
    _lib.set_option("linear_tma", tma)
    print(f"--- linear_tma={tma} ({'TMA producer + converter groups' if tma else 'round-1 cp.async producers'}) ---", flush=True)
    for awid, owid in shapes:
        K, N = sum(awid), sum(owid)
        line = f"K={K:3d} N={N:3d}:"
        for name, kw in [("full", {}), ("dsilu", dict(epi=1)), ("accum", dict(accum=True)), ("dsilu+acc", dict(epi=1, accum=True))]:
            ms, gbs = run(awid, owid, torch.float32, **kw)
            line += f"  {name} {ms*1e3:6.0f}us ({gbs:5.0f}GB/s)"
        print(line, flush=True)
_lib.set_option("linear_tma", 1)
