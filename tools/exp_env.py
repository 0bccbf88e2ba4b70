"""env_sum / env_bwd split variants: parity against split=1 and timing; linear knock-outs; raw
HBM read / write / copy rates.  Run on the GPU box."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from allegro_b200 import _lib, systems
from allegro_b200 import data as D

dev = "cuda"


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e3


d = systems.make_system("c2", 14)
n = d[D.POSITIONS_KEY].shape[0]
csr = D.build_csr(d[D.EDGE_INDEX_KEY].to(dev), n)
E = csr.num_edges
print("atoms", n, "edges", E, flush=True)
for dt in (torch.float32, torch.float64):
    acc = _lib.ACC_DTYPE[dt]
    for lmax, U in ((2, 32), (3, 64)) if dt == torch.float32 else ((2, 32),):
        Dm = (lmax + 1) ** 2
        g = torch.Generator(device=dev).manual_seed(1)
        Y = torch.randn(E, Dm, device=dev, dtype=acc, generator=g)
        w = torch.randn(E, (lmax + 1) * U, device=dev, dtype=dt, generator=g)
        gg = torch.randn(n, Dm, U, device=dev, dtype=acc, generator=g)
        ref = None
        for split in (1, 2, 4):
            _lib.set_option("env_split", split)
            gam = _lib.env_sum(dt, lmax, n, U, csr.row_ptr, Y, w, 0.3)
            gw = torch.empty_like(w)
            gY = torch.zeros_like(Y)
            _lib.env_bwd(dt, lmax, U, csr.ctr, Y, w, gg, 0.3, gw, gY, row_ptr=csr.row_ptr)
            torch.cuda.synchronize()
            if ref is None:
                ref = (gam.clone(), gw.clone(), gY.clone())
            err = [float((a - b).abs().max() / b.abs().max()) for a, b in zip((gam, gw, gY), ref)]
            t_sum = timeit(lambda: _lib.env_sum(dt, lmax, n, U, csr.row_ptr, Y, w, 0.3, out=gam))
            t_bwd = timeit(lambda: _lib.env_bwd(dt, lmax, U, csr.ctr, Y, w, gg, 0.3, gw, gY, row_ptr=csr.row_ptr))
            print(f"{str(dt)[6:]:8s} lmax={lmax} U={U} split={split}: env_sum {t_sum:7.1f} us  env_bwd {t_bwd:7.1f} us  rel.err vs split=1 {err}", flush=True)
_lib.set_option("env_split", 1)

# ---- raw HBM rates (torch kernels; 2 GiB buffers >> L2) ----
x = torch.empty(1 << 29, device=dev, dtype=torch.float32)
y = torch.empty_like(x)
GB = x.numel() * 4 / 1e9
print(f"write (zero_) {GB / timeit(x.zero_, 10) * 1e6:7.0f} GB/s", flush=True)
print(f"read  (sum)   {GB / timeit(lambda: x.sum(), 10) * 1e6:7.0f} GB/s", flush=True)
print(f"copy  (r+w)   {2 * GB / timeit(lambda: y.copy_(x), 10) * 1e6:7.0f} GB/s", flush=True)
del x, y

# ---- wgmma linear stage knock-outs (fp32 split path) ----
M = 461154
for awid, owid in (([64], [96, 64, 96]), ([64, 64, 64], [64]), ([64], [64]), ([128], [128])):
    K, N = sum(awid), sum(owid)
    a = [torch.randn(M, wd, device=dev) for wd in awid]
    W = torch.randn(K, N, device=dev) * 0.1
    o = [torch.zeros(M, wd, device=dev) for wd in owid]
    pk = _lib.linear_pack(W)
    line = f"K={K:3d} N={N:3d} ({M * (K + N) * 4 / 1e6:5.0f} MB):"
    for name, dbg in (("full", 0), ("no-store", 1), ("no-load", 2), ("no-mma", 4), ("no-load+mma", 6), ("store-only", 6), ("load-only", 5)):
        _lib.set_option("tc_debug", dbg)
        t = timeit(lambda: _lib.linear(a, W, o, W_packed=pk), 10)
        line += f"  {name} {t:5.0f}us"
    _lib.set_option("tc_debug", 0)
    print(line, flush=True)
