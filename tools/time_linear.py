"""Micro-benchmark of ab2_linear on the GPU (tensor-core vs CUDA-core path, stage knock-outs).

    python tools/time_linear.py --mlp2   # ab2_mlp2 against the two launches it replaces, c2 shapes
    python tools/time_linear.py --mlp2-readout   # ab2_mlp2_readout against the two ab2_mlp2 calls it replaces, c2 shapes
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


def run_mlp2_readout(S=64, U=32, H=64, L=2):
    """ab2_mlp2_readout (last latent MLP + readout) against the two ab2_mlp2 calls it replaces, each direction."""
    P = S * L
    X = torch.randn(M, P + S, device=dev)
    s = torch.randn(M, 3 * U, device=dev)[:, :U]
    W1l, W2l, W1r, w2r = (torch.randn(P + U, H, device=dev) * 0.1, torch.randn(H, S, device=dev) * 0.1,
                          torch.randn(P + S, H, device=dev) * 0.1, torch.randn(H, 1, device=dev) * 0.1)
    W1rT, W2lT, W1lT = W1r.T.contiguous(), W2l.T.contiguous(), W1l.T.contiguous()
    pk = _lib.linear_pack
    fwd_p = [pk(W1l), pk(W2l), pk(W1r[:P].contiguous()), pk(W1r[P:].contiguous())]
    bwd_p = [pk(W1rT), pk(W2lT), pk(W1lT)]
    p1l, p2l, p1r, p2r, pT1r, pT2l, pT1l = pk(W1l), pk(W2l), pk(W1r), pk(w2r), pk(W1rT), pk(W2lT), pk(W1lT)
    pre_l, pre_r, Ez, gEz = torch.randn(M, H, device=dev), torch.randn(M, H, device=dev), torch.empty(M, 1, device=dev), torch.randn(M, 1, device=dev)
    gX, gs = torch.empty(M, P + S, device=dev), torch.empty(M, 3 * U, device=dev)[:, :U]
    w2rT = w2r.T.contiguous()

    def fwd_pair():
        assert _lib.mlp2([X[:, :P], s], W1l, W2l, [X[:, P:]], pre_l, W1_packed=p1l, W2_packed=p2l)
        assert _lib.mlp2([X], W1r, w2r, [Ez], pre_r, W1_packed=p1r, W2_packed=p2r)

    def fwd_fused():
        assert _lib.mlp2_readout(False, X[:, :P], s, X[:, P:], pre_l, pre_r, Ez, w2r, fwd_p, S)

    def bwd_pair():
        assert _lib.mlp2([gEz], w2rT, W1rT, [gX], pre_r, backward=True, W2_packed=pT1r)
        assert _lib.mlp2([gX[:, P:]], W2lT, W1lT, [gX[:, :P], gs], pre_l, o_accum=[True, False], backward=True, W1_packed=pT2l, W2_packed=pT1l)

    def bwd_fused():
        assert _lib.mlp2_readout(True, gX[:, :P], gs, None, pre_l, pre_r, gEz, w2r, bwd_p, S)

    # fused kernels' HBM traffic in floats per row (forward: X[:, :P], s in; pre_L, x_L, pre_r, Ez out;
    # backward: gEz, pre_r, pre_L in; gX[:, :P], gs out)
    for name, pair, fused, floats in (("fwd", fwd_pair, fwd_fused, P + U + H + S + H + 1), ("bwd", bwd_pair, bwd_fused, 1 + 2 * H + P + U)):
        t_pair, t_fused = time_ms(pair), time_ms(fused)
        print(f"mlp2_readout {name} P={P} S={S} U={U} H={H}: two mlp2 {t_pair*1e3:6.0f}us  fused {t_fused*1e3:6.0f}us "
              f"({M * floats * 4 / t_fused / 1e6:5.0f}GB/s)  {t_pair / t_fused:4.2f}x", flush=True)


if "--mlp2-readout" in sys.argv:
    run_mlp2_readout()
    sys.exit(0)

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
