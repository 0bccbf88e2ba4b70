"""GPU baseline for SURVEY row a13: the REFERENCE's own Triton tensor-product kernel (oracle/_ref/ref_triton, staged
verbatim from the reference checkout by oracle/build_ref.py) timed next to this package's kernels on the same GPU, same
shapes (c2 layer 0: E = 460 992 edges, U = 32, 9 x 9 -> 9), plus a parity check between the two.

What is compared
  reference, kernel only : TritonContracter._contract(x1, x2g) -- x2g is the environment already gathered per edge
  reference, operator    : TritonContracter.forward(x1, x2, idxs, N) -- scale, scatter to atoms, gather per edge, kernel
                           (allegro/nn/_strided/_contract.py:185-211); the weighted env x2 [E,U,9] is an input
                           (MakeWeightedChannels output, a separate torch op upstream)
  ours                   : ab2_env_sum (MakeWeightedChannels + scatter fused, per-centre) + ab2_tp_fwd / ab2_tp_bwd
Backward of the reference runs through its registered autograd (two more kernel launches + the scatter's adjoint)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from allegro_b200 import _lib, data as D
from allegro_b200.nn import Contracter
from oracle import build_ref

dev = "cuda"
ref = build_ref.load()
N, deg, U, lmax = 10976, 42, 32, 2
E, Dd = N * deg, 9
torch.manual_seed(0)
sh, out_irreps = "1x0e+1x1o+1x2e", "1x0e+1x1o+1x2e"
ctr = torch.arange(N).repeat_interleave(deg).to(dev)
csr = D.build_csr(torch.stack([ctr, (ctr + 1) % N]), N)


def timeit(fn, reps=10):
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


tri = ref.TritonContracter(irreps_in1=sh, irreps_in2=sh, irreps_out=out_irreps, mul=U, path_channel_coupling=True,
                           scatter_factor=0.15).to(dev).eval()
ours = Contracter(sh, sh, out_irreps, mul=U, scatter_factor=0.15)
ours.load_state_dict({k: v.cpu() for k, v in tri.state_dict().items()})
x1 = torch.randn(E, U, Dd, device=dev)
x2 = torch.randn(E, U, Dd, device=dev)          # weighted per-edge environment (reference layout [z][u][j])
gout = torch.randn(E, U, Dd, device=dev)

# ---- reference: kernel only and whole operator, forward and forward+backward ----
x2g = (0.15 * torch.zeros(N, U, Dd, device=dev).index_add_(0, ctr, x2))[ctr].contiguous()
t_ref_k = timeit(lambda: tri._contract(x1, x2g))
t_ref_op = timeit(lambda: tri(x1, x2, ctr, N))
x1r, x2r = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)


def ref_fb():
    x1r.grad = x2r.grad = None
    tri(x1r, x2r, ctr, N).backward(gout)


t_ref_fb = timeit(ref_fb)
out_ref = tri(x1, x2, ctr, N)
ref_fb()

# ---- ours: internal layout [z][d][u], env sum fused with the weighting upstream; here the same inputs ----
ijk, _, _ = ours.sparse_table()
tab, cgw = ijk.to(dev), ours.cgw(torch.float32, dev)
Vi = x1.transpose(1, 2).contiguous()
gam = (0.15 * torch.zeros(N, U, Dd, device=dev).index_add_(0, ctr, x2)).transpose(1, 2).contiguous()  # [N][d][u]
Vout = torch.empty(E, Dd, U, device=dev)
go = gout.transpose(1, 2).contiguous()
gVin = torch.empty(E, Dd, U, device=dev)
gg = torch.empty(N, Dd, U, device=dev)
fwd = lambda: _lib.tp_fwd(torch.float32, lmax, N, E, U, Dd, Dd, tab, cgw, csr.row_ptr, csr.ctr, gam, Vi, None, None, Vout)
bwd = lambda: _lib.tp_bwd(torch.float32, lmax, N, E, U, Dd, Dd, tab, cgw, csr.row_ptr, csr.ctr, gam, Vi, None, None, go, gVin, None, None, gg)
t_f, t_b = timeit(fwd), timeit(bwd)
fwd(); bwd()
err_f = float((Vout.transpose(1, 2) - out_ref).abs().max() / out_ref.abs().max())
err_b = float((gVin.transpose(1, 2) - x1r.grad).abs().max() / x1r.grad.abs().max())
# d/dx2 of the reference = 0.15 * ggamma[ctr] (adjoint of scatter+gather); compare on the atoms
gg_ref = torch.zeros(N, U, Dd, device=dev).index_add_(0, ctr, x2r.grad) / (deg * 0.15)  # every edge of a centre carries the same row
err_g = float((gg.transpose(1, 2) - gg_ref).abs().max() / gg_ref.abs().max())
print(f"shapes: E={E} U={U} 9x9->9 fp32, nnz={tab.shape[0]}")
print(f"reference Triton kernel only (fwd)        : {t_ref_k:7.0f} us")
print(f"reference operator fwd (scatter+gather+k) : {t_ref_op:7.0f} us")
print(f"reference operator fwd+bwd (autograd)     : {t_ref_fb:7.0f} us")
print(f"ours tp_fwd (explicit Vin)                : {t_f:7.0f} us   ({t_ref_k / t_f:.1f}x vs kernel, {t_ref_op / t_f:.1f}x vs operator)")
print(f"ours tp_fwd + tp_bwd                      : {t_f + t_b:7.0f} us   ({t_ref_fb / (t_f + t_b):.1f}x vs operator fwd+bwd)")
print(f"parity ours vs reference Triton: out {err_f:.1e}  d/dx1 {err_b:.1e}  d/dgamma {err_g:.1e}")

# ---- ours, OPERATOR level (row a14: the plug-in replacement of the reference's kernel back-ends, strided [z][u][i]
#      layout, unsorted idxs, generic SIMT kernels + the recursively differentiable autograd function) ----
oursd = ours.to(dev)
oursd.weights.requires_grad_(False)
with torch.no_grad():
    t_op_f = timeit(lambda: oursd(x1, x2, ctr, N))
x1o, x2o = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)


def ours_fb():
    x1o.grad = x2o.grad = None
    oursd(x1o, x2o, ctr, N).backward(gout)


t_op_fb = timeit(ours_fb)
oursd.weights.requires_grad_(True)


def ours_fb_w():
    x1o.grad = x2o.grad = oursd.weights.grad = None
    oursd(x1o, x2o, ctr, N).backward(gout)


t_op_fbw = timeit(ours_fb_w, reps=3)
err_op = float((oursd(x1, x2, ctr, N) - out_ref).abs().max() / out_ref.abs().max())
print(f"ours OPERATOR fwd (no grad)                : {t_op_f:7.0f} us   ({t_ref_op / t_op_f:.1f}x vs reference operator fwd)")
print(f"ours OPERATOR fwd+bwd (x1, x2)             : {t_op_fb:7.0f} us   ({t_ref_fb / t_op_fb:.1f}x vs reference operator fwd+bwd)")
print(f"ours OPERATOR fwd+bwd incl. weight grads   : {t_op_fbw:7.0f} us   (the reference's Triton path has no weight gradient)")
print(f"parity ours operator vs reference Triton operator: out {err_op:.1e}")
