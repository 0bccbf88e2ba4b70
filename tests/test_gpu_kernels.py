"""GPU parity tests, kernel by kernel, through the C ABI (ctypes) against the CPU oracle.

Tolerances follow the reference's own kernel tests
(/root/reference/tests/nn/test_contract_kernels.py:117: 1e-5 fp32 / 1e-10 fp64).
"""
import math

import numpy as np
import pytest
import torch

from allegro_b200 import _lib, o3
from allegro_b200 import data as D
from allegro_b200.nn import Contracter as B200Contracter
from oracle import nn_ref as R
from oracle import o3_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {torch.float64: 1e-10, torch.float32: 2e-5, torch.bfloat16: 3e-2}


def _rel(a, b):
    return (a.double().cpu() - b.double().cpu()).abs().max().item() / max(b.double().abs().max().item(), 1e-30)


def _csr_random(N, E, seed=0):
    g = torch.Generator().manual_seed(seed)
    ctr = torch.sort(torch.randint(0, N, (E,), generator=g)).values
    ei = torch.stack([ctr, torch.randint(0, N, (E,), generator=g)])
    return D.build_csr(ei.to(DEV), N), ctr


@pytest.mark.parametrize("lmax", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_sh_fwd_bwd(lmax, dtype):
    g = torch.Generator().manual_seed(lmax)
    vec = torch.randn(1000, 3, generator=g, dtype=torch.float64) * 2.0
    Yr = o3_ref.spherical_harmonics(lmax, vec)
    Y = _lib.sh_fwd(vec.to(DEV, dtype), lmax)
    assert _rel(Y, Yr) < TOL[dtype]
    gY = torch.randn(1000, (lmax + 1) ** 2, generator=g, dtype=torch.float64)
    v = vec.clone().requires_grad_(True)
    (gr,) = torch.autograd.grad((o3_ref.spherical_harmonics(lmax, v) * gY).sum(), v)
    gv = _lib.sh_bwd(vec.to(DEV, dtype), gY.to(DEV, dtype), lmax)
    assert _rel(gv, gr) < TOL[dtype] * 10
    # accumulate mode
    base = torch.ones(1000, 3, device=DEV, dtype=dtype)
    _lib.sh_bwd(vec.to(DEV, dtype), gY.to(DEV, dtype), lmax, out=base, accumulate=True)
    assert _rel(base - 1.0, gr) < TOL[dtype] * 100


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(1000, 96, 160), (77, 64, 1), (130, 5, 70), (64, 192, 64)])
def test_linear_concat_split_act_epi(dtype, shape):
    M, K, N = shape
    g = torch.Generator().manual_seed(M + K)
    k1 = K // 3 if K >= 3 else K
    widths = [k1, K - k1] if K - k1 > 0 else [K]
    # A segments are column slices of wider buffers (exercises leading dimensions)
    bufs = [torch.randn(M, w + 3, generator=g, dtype=torch.float64) for w in widths]
    segs = [b[:, 1 : 1 + w] for b, w in zip(bufs, widths)]
    W = torch.randn(K, N, generator=g, dtype=torch.float64) / math.sqrt(K)
    aux = torch.randn(M, N, generator=g, dtype=torch.float64)
    n1 = N // 2 if N >= 2 else N
    owid = [n1, N - n1] if N - n1 > 0 else [N]
    for act, epi in [(0, 0), (1, 0), (0, 1)]:
        A = torch.cat(segs, -1).to(dtype).double()
        if act:
            A = torch.nn.functional.silu(A)
        ref = A @ W.to(dtype).double()
        if epi:
            x = aux.to(dtype).double()
            s = torch.sigmoid(x)
            ref = ref * (s * (1 + x * (1 - s)))
        dsegs = [b.to(DEV, dtype)[:, 1 : 1 + w] for b, w in zip(bufs, widths)]
        obufs = [torch.full((M, w + 2), 0.5, device=DEV, dtype=dtype) for w in owid]
        osegs = [b[:, 2:] for b in obufs]
        accum = [False, True][: len(owid)]
        _lib.linear(dsegs, W.to(DEV, dtype), osegs, o_accum=accum, act=act, epi=epi, aux=aux.to(DEV, dtype) if epi else None)
        got = torch.cat([o.double().cpu() for o in osegs], -1)
        exp = ref.clone()
        if len(owid) > 1:
            exp[:, n1:] += 0.5
        scale = exp.abs().max().item()
        assert (got - exp).abs().max().item() / scale < (TOL[dtype] if dtype != torch.float32 else 1e-5)
        for b in obufs:  # padding columns untouched
            assert (b[:, :2] == 0.5).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(1000, [64, 32], [64, 96]), (77, [64], [96, 64, 96]), (40000, [64, 64, 64], [64]),
                                   (300, [64], [1]), (129, [64, 96], [64, 64, 32]), (5000, [32, 16], [32]), (128, [96, 64, 96], [64]),
                                   # c3-sized layers (S=128, U=64): wide outputs / W images beyond the shared-memory budget run as column slices
                                   (700, [128], [192, 128, 192]), (333, [128], [128, 192]), (260, [128, 128, 64], [128]),
                                   (515, [192, 128, 192], [128]), (200, [128], [384]), (150, [384], [128]), (90, [128, 192], [100, 60])])
@pytest.mark.parametrize("mode", ["plain", "silu_in", "dsilu_epi_accum"])
@pytest.mark.parametrize("tma", [1, 0], ids=["tma", "cpasync"])
def test_linear_tensor_core_path(dtype, shape, mode, tma):
    """wgmma path (16-byte aligned segments, K % 16 == 0) against an fp64 reference and against
    the CUDA-core kernel.  fp32 storage uses the 3-term bf16 split: held to 1e-4 (measured ~1e-5)."""
    M, awid, owid = shape
    K, N = sum(awid), sum(owid)
    if tma and (dtype != torch.float32 or any(w % 32 for w in awid)):
        pytest.skip("TMA producers need fp32 storage and 32-column segments (same kernel as the cp.async case otherwise)")
    _lib.set_option("linear_tma", tma)
    g = torch.Generator().manual_seed(M + K + N)
    abufs = [torch.randn(M, w + 8, generator=g, dtype=torch.float64) for w in awid]
    W = torch.randn(K, N, generator=g, dtype=torch.float64) / math.sqrt(K)
    aux = torch.randn(M, N, generator=g, dtype=torch.float64)
    act = 1 if mode == "silu_in" else 0
    epi = 1 if mode == "dsilu_epi_accum" else 0
    accum = [mode == "dsilu_epi_accum" and (i % 2 == 1) for i in range(len(owid))]
    A = torch.cat([b[:, 4 : 4 + w] for b, w in zip(abufs, awid)], -1).to(dtype).double()
    if act:
        A = torch.nn.functional.silu(A)
    ref = A @ W.to(dtype).double()
    if epi:
        x = aux.to(dtype).double()
        sg = torch.sigmoid(x)
        ref = ref * (sg * (1 + x * (1 - sg)))
    Wd = W.to(DEV, dtype)
    packed = _lib.linear_pack(Wd)
    assert packed is not None
    res = {}
    for name, pk in (("tc", packed), ("simt", None)):
        dsegs = [b.to(DEV, dtype)[:, 4 : 4 + w] for b, w in zip(abufs, awid)]
        obufs = [torch.full((M, w + 4), 0.25, device=DEV, dtype=dtype) for w in owid]
        osegs = [b[:, 4:] for b in obufs]
        _lib.linear(dsegs, Wd, osegs, o_accum=accum, act=act, epi=epi, aux=aux.to(DEV, dtype) if epi else None, W_packed=pk)
        got = torch.cat([o.double().cpu() for o in osegs], -1)
        for b in obufs:
            assert (b[:, :4] == 0.25).all()
        res[name] = got
    exp = ref.clone()
    o = 0
    for w, a in zip(owid, accum):
        if a:
            exp[:, o : o + w] += 0.25
        o += w
    scale = exp.abs().max().item()
    _lib.set_option("linear_tma", 1)
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    assert (res["tc"] - exp).abs().max().item() / scale < tol
    assert (res["simt"] - exp).abs().max().item() / scale < (1e-5 if dtype == torch.float32 else 2e-2)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("shape", [(3000, [64, 64, 64], [64]), (130, [64, 32], [32]), (77, [16], [48])])
def test_linear_prologue_mul_dsilu(dtype, shape):
    """act=ACT_MUL_DSILU: segment s of A is scaled by silu'(aux_s) on load (aux may be None per
    segment); tensor-core path (fp32) and CUDA-core path against an fp64 reference."""
    M, awid, owid = shape
    K, N = sum(awid), sum(owid)
    g = torch.Generator().manual_seed(K + N)
    A = [torch.randn(M, w, generator=g, dtype=torch.float64) for w in awid]
    X = [torch.randn(M, w, generator=g, dtype=torch.float64) if i != 1 else None for i, w in enumerate(awid)]
    W = torch.randn(K, N, generator=g, dtype=torch.float64) / math.sqrt(K)
    segs = []
    for a, x in zip(A, X):
        a = a.to(dtype).double()
        if x is not None:
            xq = x.to(dtype).double()
            sg = torch.sigmoid(xq)
            a = a * (sg * (1 + xq * (1 - sg)))
        segs.append(a)
    ref = torch.cat(segs, -1) @ W.to(dtype).double()
    Wd = W.to(DEV, dtype)
    for pk in ([_lib.linear_pack(Wd), None] if dtype == torch.float32 else [None]):
        out = torch.empty(M, N, device=DEV, dtype=dtype)
        _lib.linear([a.to(DEV, dtype) for a in A], Wd, [out], act=_lib.ACT_MUL_DSILU,
                    a_aux=[x.to(DEV, dtype) if x is not None else None for x in X], W_packed=pk)
        tol = 1e-12 if dtype == torch.float64 else (1e-4 if pk is not None else 1e-5)
        assert _rel(out, ref) < tol


@pytest.mark.parametrize("lmax", [1, 2, 3])
@pytest.mark.parametrize("U", [4, 32, 48, 64])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("fastpath", [True, False, "dense"])
def test_env_sum_and_bwd(lmax, U, dtype, fastpath):
    """fastpath "dense": contiguous w / gw rows, what the pipeline passes -- the TMA-staged streaming adjoint
    (env_stream.cu) takes these; the strided views exercise the round-1 kernels."""
    dense = fastpath == "dense"
    fastpath = bool(fastpath)
    N, E = 37, 600
    csr, ctr = _csr_random(N, E, seed=U)
    g = torch.Generator().manual_seed(lmax * 10 + U)
    Dd, n_ir = (lmax + 1) ** 2, lmax + 1
    acc = _lib.ACC_DTYPE[dtype]
    Y = torch.randn(E, Dd, generator=g, dtype=torch.float64)
    wbuf = torch.randn(E, n_ir * U + 5, generator=g, dtype=torch.float64)
    w_int = wbuf[:, 2 : 2 + n_ir * U]  # internal layout [r][u]
    w_q = w_int.to(dtype).double()
    sf = 0.3
    # oracle: MakeWeightedChannels (ref layout [u][r]) + scatter
    irreps = o3_ref.Irreps.spherical_harmonics(lmax)
    m = R.MakeWeightedChannels(irreps, U)
    w_ref = w_q.view(E, n_ir, U).transpose(1, 2).reshape(E, U * n_ir)
    A = m(Y.to(acc).double(), w_ref)  # [E,U,D]
    gam_ref = sf * R.scatter(A, ctr, N)  # [N,U,D]
    gam = _lib.env_sum(dtype, lmax, N, U, csr.row_ptr, Y.to(DEV, acc), wbuf.to(DEV, dtype)[:, 2 : 2 + n_ir * U], sf)
    assert _rel(gam.transpose(1, 2), gam_ref) < (1e-5 if dtype != torch.float64 else 1e-12)
    # backward
    gg = torch.randn(N, Dd, U, generator=g, dtype=torch.float64)
    Yt = Y.to(acc).double().clone().requires_grad_(True)
    wt = w_q.clone().requires_grad_(True)
    A2 = m(Yt, wt.view(E, n_ir, U).transpose(1, 2).reshape(E, U * n_ir))
    loss = (sf * R.scatter(A2, ctr, N) * gg.transpose(1, 2)).sum()
    gY_ref, gw_ref = torch.autograd.grad(loss, (Yt, wt))
    gw = torch.zeros(E, n_ir * U + 1, device=DEV, dtype=dtype)
    gY = torch.ones(E, Dd, device=DEV, dtype=acc)
    w_dev = wbuf.to(DEV, dtype)[:, 2 : 2 + n_ir * U]
    gw_view = gw[:, 1:]
    if dense:
        w_dev = w_dev.contiguous()
        gw_dense = torch.zeros(E, n_ir * U, device=DEV, dtype=dtype)
        gw_view = gw_dense
    _lib.env_bwd(dtype, lmax, U, csr.ctr, Y.to(DEV, acc), w_dev, gg.to(DEV, acc), sf, gw_view, gY,
                 row_ptr=csr.row_ptr if fastpath else None)
    if dense:
        gw[:, 1:] = gw_dense
    tol = {torch.float64: 1e-12, torch.float32: 1e-5, torch.bfloat16: 1e-2}[dtype]
    assert _rel(gw[:, 1:], gw_ref) < tol
    assert _rel(gY - 1.0, gY_ref) < (1e-5 if dtype != torch.float64 else 1e-12)


def _tp_case(lmax, layer, L, U, coupling, dtype, seed=0):
    """Build the oracle Contracter of Allegro layer `layer` and matching kernel tables."""
    sh = o3_ref.Irreps.spherical_harmonics(lmax)
    allowed = o3_ref.Irreps([(1, (l, p)) for l in range(lmax + 1) for p in (1, -1)])
    ins, outs = R.allegro_layer_irreps(sh, allowed, L)
    torch.manual_seed(seed)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        c = R.Contracter(ins[layer], sh, outs[layer], mul=U, path_channel_coupling=coupling, scatter_factor=None)
        b = B200Contracter(repr(ins[layer]), repr(sh), repr(outs[layer]), mul=U, path_channel_coupling=coupling)
    finally:
        torch.set_default_dtype(prev)
    b.load_state_dict(c.state_dict())
    return c, b


@pytest.fixture(params=[(1, 1, 8, 0, 1), (1, 1, 8, 0, 0), (1, 1, 8, 1, 1), (1, 1, 16, 0, 1), (1, 0, 8, 0, 1), (2, 0, 8, 0, 1), (0, 0, 8, 0, 1)],
                ids=["stream", "stream_shfl", "stream3", "stream_te16", "fast", "regM", "generic"])
def tp_fast(request):
    """Kernel families of the tensor product: TMA-staged streaming kernels (round 2, default where instantiated; "stream_shfl" =
    layer-0 backward with the per-edge shuffle reduction of gY instead of the shared-memory tile, "stream3" = with the
    three-consumer-warp layer-0 backward, the default where eligible), the round-1
    shared-memory-M / split kernels, the register-M kernels, the shape-generic kernels."""
    fast, stream, te, s3, gyt = request.param
    _lib.set_option("tp_fast", fast)
    _lib.set_option("tp_stream", stream)
    _lib.set_option("tp_stream_te", te)
    _lib.set_option("tp_stream3", s3)
    _lib.set_option("tp_stream_gytile", gyt)
    yield request.param
    _lib.set_option("tp_fast", 1)
    _lib.set_option("tp_stream", 1)
    _lib.set_option("tp_stream_te", 0)
    _lib.set_option("tp_stream3", 1)
    _lib.set_option("tp_stream_gytile", 1)


@pytest.mark.parametrize("case", [(1, 0, 1), (2, 0, 2), (2, 1, 2), (3, 0, 3), (3, 1, 3), (3, 2, 3), (1, 0, 2), (1, 1, 3)])
@pytest.mark.parametrize("coupling", [True, False])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("U", [8, 32, 40])
def test_tp_fwd_bwd_explicit(case, coupling, dtype, U, tp_fast):
    lmax, layer, L = case
    if U != 8 and (dtype == torch.float64 or not coupling):
        pytest.skip("channel-chunk coverage only needed once")
    N, E = 23, 300
    c, b = _tp_case(lmax, layer, L, U, coupling, dtype)
    csr, ctr = _csr_random(N, E, seed=layer)
    acc = _lib.ACC_DTYPE[dtype]
    g = torch.Generator().manual_seed(5)
    d_in, d_out, Dd = c.base_dim1, c.base_dim_out, (lmax + 1) ** 2
    V = torch.randn(E, U, d_in, generator=g, dtype=torch.float64).to(dtype).double()
    gam = torch.randn(N, U, Dd, generator=g, dtype=torch.float64).to(acc).double()
    gout = torch.randn(E, U, d_out, generator=g, dtype=torch.float64).to(dtype).double()
    Vt, gt = V.clone().requires_grad_(True), gam.clone().requires_grad_(True)
    out_ref = c._contract(Vt, gt[ctr])
    gV_ref, ggam_ref = torch.autograd.grad((out_ref * gout).sum(), (Vt, gt))
    ijk, _, _ = b.sparse_table()
    tab, cgw = ijk.to(DEV), b.cgw(acc, DEV)
    Vi = V.transpose(1, 2).contiguous().to(DEV, dtype)
    gi = gam.transpose(1, 2).contiguous().to(DEV, acc)
    Vout = torch.empty(E, d_out, U, device=DEV, dtype=dtype)
    _lib.tp_fwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gi, Vi, None, None, Vout)
    tol = {torch.float64: 1e-12, torch.float32: 2e-5, torch.bfloat16: 1e-2}[dtype]
    assert _rel(Vout.transpose(1, 2), out_ref.detach()) < tol
    gVin = torch.empty(E, d_in, U, device=DEV, dtype=dtype)
    ggam = torch.empty(N, Dd, U, device=DEV, dtype=acc)
    _lib.tp_bwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gi, Vi, None, None,
                gout.transpose(1, 2).contiguous().to(DEV, dtype), gVin, None, None, ggam)
    assert _rel(gVin.transpose(1, 2), gV_ref) < tol
    assert _rel(ggam.transpose(1, 2), ggam_ref) < (tol if dtype != torch.bfloat16 else 1e-5)


@pytest.mark.parametrize("lmax", [1, 2, 3])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("U", [8, 32, 40])
def test_tp_fwd_bwd_implicit_v0(lmax, dtype, U, tp_fast):
    """Layer 0 with Vin = Y (x) w0 formed on the fly (tensorembed.py:95)."""
    N, E, L = 19, 250, 2
    c, b = _tp_case(lmax, 0, L, U, True, dtype)
    csr, ctr = _csr_random(N, E, seed=3)
    acc = _lib.ACC_DTYPE[dtype]
    g = torch.Generator().manual_seed(9)
    Dd, n_ir, d_out = (lmax + 1) ** 2, lmax + 1, c.base_dim_out
    Y = torch.randn(E, Dd, generator=g, dtype=torch.float64).to(acc).double()
    w0 = torch.randn(E, n_ir * U, generator=g, dtype=torch.float64).to(dtype).double()  # internal [r][u]
    gam = torch.randn(N, U, Dd, generator=g, dtype=torch.float64).to(acc).double()
    gout = torch.randn(E, U, d_out, generator=g, dtype=torch.float64).to(dtype).double()
    m = R.MakeWeightedChannels(o3_ref.Irreps.spherical_harmonics(lmax), U)
    Yt, wt, gt = Y.clone().requires_grad_(True), w0.clone().requires_grad_(True), gam.clone().requires_grad_(True)
    V0 = m(Yt, wt.view(E, n_ir, U).transpose(1, 2).reshape(E, -1))
    out_ref = c._contract(V0, gt[ctr])
    gY_ref, gw_ref, ggam_ref = torch.autograd.grad((out_ref * gout).sum(), (Yt, wt, gt))
    ijk, _, _ = b.sparse_table()
    tab, cgw = ijk.to(DEV), b.cgw(acc, DEV)
    gi = gam.transpose(1, 2).contiguous().to(DEV, acc)
    Yd, wd = Y.to(DEV, acc), w0.to(DEV, dtype)
    Vout = torch.empty(E, d_out, U, device=DEV, dtype=dtype)
    _lib.tp_fwd(dtype, lmax, N, E, U, Dd, d_out, tab, cgw, csr.row_ptr, csr.ctr, gi, None, Yd, wd, Vout)
    tol = {torch.float64: 1e-12, torch.float32: 2e-5, torch.bfloat16: 1e-2}[dtype]
    assert _rel(Vout.transpose(1, 2), out_ref.detach()) < tol
    gw0 = torch.empty(E, n_ir * U, device=DEV, dtype=dtype)
    gY = torch.zeros(E, Dd, device=DEV, dtype=acc)
    ggam = torch.empty(N, Dd, U, device=DEV, dtype=acc)
    _lib.tp_bwd(dtype, lmax, N, E, U, Dd, d_out, tab, cgw, csr.row_ptr, csr.ctr, gi, None, Yd, wd,
                gout.transpose(1, 2).contiguous().to(DEV, dtype), None, gw0, gY, ggam)
    assert _rel(gw0, gw_ref) < tol
    assert _rel(gY, gY_ref) < (tol if dtype != torch.bfloat16 else 1e-5)
    assert _rel(ggam.transpose(1, 2), ggam_ref) < (tol if dtype != torch.bfloat16 else 1e-5)


@pytest.mark.parametrize("s3,gyt", [(1, 1), (0, 1), (0, 0)], ids=["stream3", "stream", "stream_shfl"])
def test_tp_stream_ragged_rows(s3, gyt):
    """Layer-0 streaming kernels on a ragged CSR with more centres than CTAs: empty centres (also leading / trailing), rows of
    1-3 edges (several centres begin inside one 8-edge stage), rows far longer than a stage.  Reference: the shape-generic
    kernels on the same device data (themselves held to the oracle above); ggamma of empty centres must come back zero and
    two runs must agree bitwise (every reduction is fixed-order)."""
    g = torch.Generator().manual_seed(11)
    N, U, lmax, Dd, n_ir = 3000, 32, 2, 9, 3
    deg = torch.randint(0, 4, (N,), generator=g)
    deg[torch.randint(0, N, (300,), generator=g)] = 0
    deg[torch.randint(0, N, (40,), generator=g)] = torch.randint(60, 200, (40,), generator=g)
    deg[:5] = 0
    deg[-7:] = 0
    ctr = torch.repeat_interleave(torch.arange(N), deg)
    E = int(ctr.numel())
    csr = D.build_csr(torch.stack([ctr, torch.randint(0, N, (E,), generator=g)]).to(DEV), N)
    _, b = _tp_case(lmax, 0, 2, U, True, torch.float32)
    ijk, _, _ = b.sparse_table()
    tab, cgw = ijk.to(DEV), b.cgw(torch.float32, DEV)
    Y = torch.randn(E, Dd, generator=g).to(DEV)
    w0 = torch.randn(E, n_ir * U, generator=g).to(DEV)
    gam = torch.randn(N, Dd, U, generator=g).to(DEV)
    gout = torch.randn(E, Dd, U, generator=g).to(DEV)

    def run():
        Vout = torch.empty(E, Dd, U, device=DEV)
        gw0 = torch.full((E, n_ir * U), float("nan"), device=DEV)
        gY = torch.ones(E, Dd, device=DEV)  # accumulated into
        ggam = torch.full((N, Dd, U), float("nan"), device=DEV)
        _lib.tp_fwd(torch.float32, lmax, N, E, U, Dd, Dd, tab, cgw, csr.row_ptr, csr.ctr, gam, None, Y, w0, Vout)
        _lib.tp_bwd(torch.float32, lmax, N, E, U, Dd, Dd, tab, cgw, csr.row_ptr, csr.ctr, gam, None, Y, w0, gout, None, gw0, gY, ggam)
        torch.cuda.synchronize()
        return Vout, gw0, gY, ggam

    try:
        _lib.set_option("tp_fast", 0)
        _lib.set_option("tp_stream", 0)
        ref = run()
        _lib.set_option("tp_fast", 1)
        _lib.set_option("tp_stream", 1)
        _lib.set_option("tp_stream3", s3)
        _lib.set_option("tp_stream_gytile", gyt)
        got, again = run(), run()
    finally:
        _lib.set_option("tp_fast", 1)
        _lib.set_option("tp_stream", 1)
        _lib.set_option("tp_stream3", 1)
        _lib.set_option("tp_stream_gytile", 1)
    for name, a, r in zip(("Vout", "gw0", "gY", "ggamma"), got, ref):
        assert bool(torch.isfinite(a).all()), name
        assert _rel(a, r) < 2e-5, name
    assert bool((got[3][deg == 0] == 0).all())
    for name, a, c in zip(("Vout", "gw0", "ggamma"), (got[0], got[1], got[3]), (again[0], again[1], again[3])):
        assert torch.equal(a, c), name


@pytest.mark.parametrize("layer", [0, 1, 2])
@pytest.mark.parametrize("implicit", [False, True])
def test_tp_baked64_matches_generic(layer, implicit):
    """fp64 kernels with the baked l_max = 3 table structure (csrc/tp_baked64.cu; the three layer shapes of BASELINE configs[4])
    against the shape-generic kernels on the same device data (those are held to the oracle above); U = 64 = two channel chunks,
    ragged CSR with empty centres."""
    if implicit and layer == 1:
        pytest.skip("only a first layer (d_in = d_env) has implicit input features")
    lmax, L, U, N = 3, 3, 64, 37
    _, b = _tp_case(lmax, layer, L, U, True, torch.float64)
    g = torch.Generator().manual_seed(21 + layer)
    deg = torch.randint(0, 9, (N,), generator=g)
    deg[3] = 0
    deg[-1] = 0
    ctr = torch.repeat_interleave(torch.arange(N), deg)
    E = int(ctr.numel())
    csr = D.build_csr(torch.stack([ctr, torch.randint(0, N, (E,), generator=g)]).to(DEV), N)
    ijk, _, _ = b.sparse_table()
    tab, cgw = ijk.to(DEV), b.cgw(torch.float64, DEV)
    d_in, d_out, Dd, n_ir = b.base_dim1, b.base_dim_out, 16, 4
    assert (d_in, d_out) == [(16, 31), (31, 16), (16, 1)][layer]
    dd = dict(dtype=torch.float64, generator=g)
    Y, w0 = torch.randn(E, Dd, **dd).to(DEV), torch.randn(E, n_ir * U, **dd).to(DEV)
    Vin = None if implicit else torch.randn(E, d_in, U, **dd).to(DEV)
    gam, gout = torch.randn(N, Dd, U, **dd).to(DEV), torch.randn(E, d_out, U, **dd).to(DEV)

    def run():
        Vout = torch.full((E, d_out, U), float("nan"), dtype=torch.float64, device=DEV)
        gVin = None if implicit else torch.full((E, d_in, U), float("nan"), dtype=torch.float64, device=DEV)
        gw0 = torch.full((E, n_ir * U), float("nan"), dtype=torch.float64, device=DEV) if implicit else None
        gY = torch.ones(E, Dd, dtype=torch.float64, device=DEV) if implicit else None
        ggam = torch.full((N, Dd, U), float("nan"), dtype=torch.float64, device=DEV)
        _lib.tp_fwd(torch.float64, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gam, Vin, Y if implicit else None, w0 if implicit else None, Vout)
        _lib.tp_bwd(torch.float64, lmax, N, E, U, d_in, d_out, tab, cgw, csr.row_ptr, csr.ctr, gam, Vin, Y if implicit else None,
                    w0 if implicit else None, gout, gVin, gw0, gY, ggam)
        torch.cuda.synchronize()
        return [t for t in (Vout, gVin, gw0, gY, ggam) if t is not None]

    try:
        _lib.set_option("tp_baked64", 0)
        ref = run()
        _lib.set_option("tp_baked64", 1)
        got = run()
    finally:
        _lib.set_option("tp_baked64", 1)
    for a, r in zip(got, ref):
        assert bool(torch.isfinite(a).all())
        assert _rel(a, r) < 1e-12
    # the baked kernels sum in a different order: bitwise identical results would mean they stood down
    assert any(not torch.equal(a, r) for a, r in zip(got, ref))


def test_edge_sum_force_scatter_transpose():
    N, E = 50, 900
    csr, ctr = _csr_random(N, E, seed=1)
    g = torch.Generator().manual_seed(2)
    for dtype in (torch.float64, torch.float32):
        Ez = torch.randn(E, generator=g, dtype=torch.float64)
        Ei = _lib.edge_sum(Ez.to(DEV, dtype), csr.row_ptr, 0.25)
        ref = torch.zeros(N, dtype=torch.float64).index_add_(0, ctr, 0.25 * Ez)
        assert _rel(Ei, ref) < TOL[dtype]
        gEi = torch.randn(N, generator=g, dtype=torch.float64)
        gEz = _lib.edge_sum_bwd(gEi.to(DEV, dtype), csr.ctr, 0.25)
        assert _rel(gEz, 0.25 * gEi[ctr]) < TOL[dtype]
        gv = torch.randn(E, 3, generator=g, dtype=torch.float64)
        F = _lib.force_scatter(gv.to(DEV, dtype), csr, N)
        assert torch.equal(F, _lib.force_scatter(gv.to(DEV, dtype), csr, N))  # deterministic: bitwise reproducible
        Fr = torch.zeros(N, 3, dtype=torch.float64).index_add_(0, ctr, gv).index_add_(0, csr.nbr.long().cpu(), -gv)
        assert _rel(F, Fr) < TOL[dtype] * 10
    x = torch.randn(33, 5, 7, generator=g).to(DEV)
    xi = _lib.transpose_ui(x, True)
    assert torch.equal(xi, x.transpose(1, 2).contiguous())
    assert torch.equal(_lib.transpose_ui(xi, False), x)


# --------------------------------------------------------------------------- #
# operator level: the reference's test_contract_kernels.py grid
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("irreps_in1", ["0e + 0o + 1e + 1o", "2o + 1e + 0e"])
@pytest.mark.parametrize("irreps_in2", ["0e + 0o + 1e + 1o"])
@pytest.mark.parametrize("irreps_out", ["0e + 0o + 1e + 1o", "1o + 2e"])
@pytest.mark.parametrize("coupling", [True, False])
@pytest.mark.parametrize("mul", [3, 8])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_contract_kernel_vs_base(irreps_in1, irreps_in2, irreps_out, coupling, mul, dtype):
    """tests/nn/test_contract_kernels.py:31-134: forward and grads wrt x1, x2 equal the base
    (here: oracle) Contracter; 17 edges -> 5 atoms, random scatter idxs."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(dtype)
    try:
        torch.manual_seed(0)
        i1, i2, io = o3_ref.Irreps(irreps_in1), o3_ref.Irreps(irreps_in2), o3_ref.Irreps(irreps_out)
        c_base = R.Contracter(i1, i2, io, mul=mul, path_channel_coupling=coupling)
        c_k = B200Contracter(irreps_in1, irreps_in2, irreps_out, mul=mul, instructions=c_base.instructions,
                             path_channel_coupling=coupling).to(DEV)
        c_k.load_state_dict(c_base.state_dict())
        E, N = 17, 5
        idx = torch.randint(0, N, (E,))
        x1, x2 = torch.randn(E, mul, i1.dim), torch.randn(E, mul, i2.dim)
        tol = {torch.float32: 1e-5, torch.float64: 1e-10}[dtype]
        for arg in (0, 1):
            a = [x1.clone(), x2.clone()]
            a[arg].requires_grad_(True)
            out_o = c_base(a[0], a[1], idx, torch.tensor([N]))
            go = torch.randn_like(out_o)
            (g_o,) = torch.autograd.grad(out_o, [a[arg]], go)
            b = [x1.clone().to(DEV), x2.clone().to(DEV)]
            b[arg].requires_grad_(True)
            out_k = c_k(b[0], b[1], idx.to(DEV), torch.tensor([N], device=DEV))
            (g_k,) = torch.autograd.grad(out_k, [b[arg]], go.to(DEV))
            torch.testing.assert_close(out_k.cpu(), out_o.detach(), atol=tol, rtol=tol)
            torch.testing.assert_close(g_k.cpu(), g_o, atol=tol, rtol=tol)
    finally:
        torch.set_default_dtype(prev)


@pytest.mark.parametrize("sorted_idx", [False, True], ids=["generic", "sorted"])
@pytest.mark.parametrize("coupling", [True, False])
@pytest.mark.parametrize("irreps", [("0e + 1o + 2e", "0e + 1o + 2e", "0e + 1o + 2e"), ("2o + 1e + 0e", "0e + 0o + 1e + 1o", "1o + 2e")])
def test_contracter_weight_grad_and_double_backward(irreps, coupling, sorted_idx):
    """Training support (SURVEY row f4): the reference's ``weights`` are Parameters and its einsum path is differentiable
    to any order through autograd (_contract.py:170-177, 213-251).  The B200 operator builds every derivative from four
    hand-written products; held here to the oracle's autograd: d/d(weights, x1, x2) of a scalar loss, and the second-order
    terms a force loss needs -- d/d(weights, x1, x2) of a function of dOut/dx1 and dOut/dx2."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        torch.manual_seed(3)
        i1, i2, io = (o3_ref.Irreps(x) for x in irreps)
        mul, E, N = 5, 23, 6
        c_base = R.Contracter(i1, i2, io, mul=mul, path_channel_coupling=coupling, scatter_factor=0.37)
        c_k = B200Contracter(irreps[0], irreps[1], irreps[2], mul=mul, instructions=c_base.instructions, path_channel_coupling=coupling,
                             scatter_factor=0.37).to(DEV)
        c_k.load_state_dict(c_base.state_dict())
        idx = torch.randint(0, N, (E,))
        if sorted_idx:  # centre-sorted indices + a full SH second operand take the fused pipeline's kernels (Contracter._fast_route)
            idx = torch.sort(idx).values
        x1, x2 = torch.randn(E, mul, i1.dim), torch.randn(E, mul, i2.dim)
        go, v1, v2 = torch.randn(E, mul, io.dim), torch.randn(E, mul, i1.dim), torch.randn(E, mul, i2.dim)

        def losses(c, dev):
            a = x1.clone().to(dev).requires_grad_(True)
            b = x2.clone().to(dev).requires_grad_(True)
            out = c(a, b, idx.to(dev), torch.tensor([N], device=dev))
            first = torch.autograd.grad((out * go.to(dev)).sum(), [c.weights, a, b], retain_graph=True)
            # "force-like" quantities, then a loss on them (double backward)
            ga, gb = torch.autograd.grad((out * torch.tanh(out)).sum(), [a, b], create_graph=True)
            loss2 = (ga * v1.to(dev)).sum() + (gb * v2.to(dev)).pow(2).sum()
            second = torch.autograd.grad(loss2, [c.weights, a, b])
            return [t.detach().cpu() for t in (out, *first, *second)]

        ref, got = losses(c_base, "cpu"), losses(c_k, DEV)
        route = c_k._tab_cache.get("route")
        assert (route is not None and route[3] is not None) == (sorted_idx and i2.dim == 9)
        for name, r, g in zip(("out", "dL/dw", "dL/dx1", "dL/dx2", "d2/dw", "d2/dx1", "d2/dx2"), ref, got):
            assert g.shape == r.shape, name
            assert _rel(g, r) < 1e-10, (name, float(_rel(g, r)))
    finally:
        torch.set_default_dtype(prev)


def test_contracter_scatter_factor_and_equivariance():
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        torch.manual_seed(3)
        irr = "0e+1o+2e"
        i = o3_ref.Irreps(irr)
        c_base = R.Contracter(i, i, i, mul=4, scatter_factor=0.21)
        c_k = B200Contracter(irr, irr, irr, mul=4, scatter_factor=0.21).to(DEV)
        c_k.load_state_dict(c_base.state_dict())
        E, N = 40, 7
        idx = torch.randint(0, N, (E,))
        x1, x2 = torch.randn(E, 4, 9), torch.randn(E, 4, 9)
        out = c_k(x1.to(DEV), x2.to(DEV), idx.to(DEV), N).cpu()
        assert (out - c_base(x1, x2, idx, N).detach()).abs().max() < 1e-12
        Rm = o3_ref.random_rotation(4)
        Dm = torch.block_diag(*[o3_ref.wigner_D_from_rotation(l, Rm) for l in (0, 1, 2)])
        out_r = c_k((x1 @ Dm.T).to(DEV), (x2 @ Dm.T).to(DEV), idx.to(DEV), N).cpu()
        assert (out_r - out @ Dm.T).abs().max() < 1e-9
        with pytest.raises(RuntimeError):
            c_k.cpu()(x1, x2, idx, N)  # no CPU path
    finally:
        torch.set_default_dtype(prev)
