"""Executable specification of the C-ABI kernels (include/allegro_b200.h) in plain torch -- TEST INFRASTRUCTURE.

Each function has the signature of the ctypes wrapper of the same name in allegro_b200/_lib.py and does, with
device-agnostic torch ops, what the header says the kernel does (adjoints by autograd of the forward definition, so
they are independent of the hand-derived backward kernels).  tests/test_host_pipeline.py monkeypatches these over the
wrappers to run the product's HOST logic -- weight packing and column permutations, segment views, accumulate flags, the
backward orchestration, CSR / permutation handling, stress -- on a CPU-only box against the oracle and the
reference-generated vectors.  It is never importable from the product (the product has no CPU path), and it says
nothing about the CUDA kernels themselves: those are checked against the oracle on the GPU.
"""
import torch

from allegro_b200 import _lib
from oracle import nn_ref as R
from oracle import o3_ref


def _l_of(D):
    return torch.tensor([o3_ref.Irreps.spherical_harmonics(int(round(D**0.5)) - 1).slices().index(s) for s in
                         o3_ref.Irreps.spherical_harmonics(int(round(D**0.5)) - 1).slices() for _ in range(s.stop - s.start)])


def _ctr_of(row_ptr):
    n = row_ptr.shape[0] - 1
    return torch.repeat_interleave(torch.arange(n, device=row_ptr.device), (row_ptr[1:] - row_ptr[:-1]).long())


def _dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def sh_fwd(vec, lmax):
    return o3_ref.spherical_harmonics(lmax, vec, method="recursive" if lmax > 3 else "explicit")


def sh_bwd(vec, gY, lmax, out=None, accumulate=False):
    if vec.shape[0] == 0 or lmax == 0:  # Y_0 is a constant: no gradient reaches the edge vectors
        g = torch.zeros_like(vec)
    else:
        v = vec.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            (g,) = torch.autograd.grad(sh_fwd(v, lmax), v, gY)
    if out is None:
        return g
    out.copy_(out + g if accumulate else g)
    return out


def linear(a_segs, W, o_segs, o_accum=None, act=_lib.ACT_NONE, epi=_lib.EPI_NONE, aux=None, W_packed=None, a_aux=None):
    cols = []
    for s, a in enumerate(a_segs):
        a = a.to(torch.float64)
        if act == _lib.ACT_SILU:
            a = torch.nn.functional.silu(a)
        elif act == _lib.ACT_MUL_DSILU and a_aux is not None and a_aux[s] is not None:
            a = a * _dsilu(a_aux[s].to(torch.float64))
        cols.append(a)
    A = torch.cat(cols, dim=-1)
    assert A.shape[1] == W.shape[0]
    out = A @ W.to(torch.float64)
    if epi == _lib.EPI_MUL_DSILU:
        out = out * _dsilu(aux.to(torch.float64))
    assert sum(o.shape[1] for o in o_segs) == W.shape[1]
    c = 0
    for s, o in enumerate(o_segs):
        chunk = out[:, c : c + o.shape[1]].to(o.dtype)
        if o_accum is not None and o_accum[s]:
            o += chunk
        else:
            o.copy_(chunk)
        c += o.shape[1]


def linear_pack(W):
    return None  # no tensor-core image on this path


def env_sum(dtype, lmax, N, U, row_ptr, Y, w, sf, out=None):
    D, n_ir = (lmax + 1) ** 2, lmax + 1
    E = Y.shape[0]
    wv = w[:, : n_ir * U].reshape(E, n_ir, U).to(Y.dtype)
    A = Y.unsqueeze(-1) * wv[:, _l_of(D)]                       # [E, D, U]
    gamma = torch.zeros(N, D, U, dtype=Y.dtype, device=Y.device).index_add_(0, _ctr_of(row_ptr), A) * sf
    if out is None:
        return gamma
    out.copy_(gamma)
    return out


def env_bwd(dtype, lmax, U, ctr, Y, w, ggamma, sf, gw, gY, row_ptr=None):
    D, n_ir = (lmax + 1) ** 2, lmax + 1
    E = Y.shape[0]
    l_of = _l_of(D)
    gg = ggamma[ctr.long()] * sf                                  # [E, D, U]
    wv = w[:, : n_ir * U].reshape(E, n_ir, U).to(Y.dtype)
    gwv = torch.zeros(E, n_ir, U, dtype=Y.dtype).index_add_(1, l_of, Y.unsqueeze(-1) * gg)
    gw[:, : n_ir * U] = gwv.reshape(E, n_ir * U).to(gw.dtype)
    gY += (wv[:, l_of] * gg).sum(-1)


def _tp(tab, cgw, ctr, gamma, Vin, d_out):
    E, _, U = Vin.shape
    out = torch.zeros(E, d_out, U, dtype=Vin.dtype)
    g = gamma[ctr.long()]
    for n, (i, j, k) in enumerate(tab.tolist()):
        out[:, k, :] = out[:, k, :] + cgw[n].unsqueeze(0) * Vin[:, i, :] * g[:, j, :]
    return out


def _implicit_v0(Y, w0, U):
    D = Y.shape[1]
    n_ir = int(round(D**0.5))
    return Y.unsqueeze(-1) * w0[:, : n_ir * U].reshape(Y.shape[0], n_ir, U).to(Y.dtype)[:, _l_of(D)]


def tp_fwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, row_ptr, ctr, gamma, Vin, Y, w0, Vout):
    V = _implicit_v0(Y, w0, U) if Vin is None else Vin.to(gamma.dtype)
    Vout.copy_(_tp(tab, cgw, ctr, gamma, V, d_out).to(Vout.dtype))


def tp_bwd(dtype, lmax, N, E, U, d_in, d_out, tab, cgw, row_ptr, ctr, gamma, Vin, Y, w0, gVout, gVin, gw0, gY, ggamma):
    n_ir = lmax + 1
    with torch.enable_grad():
        gam = gamma.detach().clone().requires_grad_(True)
        if Vin is None:
            Yr = Y.detach().clone().requires_grad_(True)
            wr = w0[:, : n_ir * U].detach().to(Y.dtype).clone().requires_grad_(True)
            out = _tp(tab, cgw, ctr, gam, _implicit_v0(Yr, wr, U), d_out)
            g_gam, g_Y, g_w = torch.autograd.grad(out, (gam, Yr, wr), gVout.to(out.dtype))
            gw0[:, : n_ir * U] = g_w.to(gw0.dtype)
            gY += g_Y
        else:
            Vr = Vin.detach().to(gamma.dtype).clone().requires_grad_(True)
            out = _tp(tab, cgw, ctr, gam, Vr, d_out)
            g_gam, g_V = torch.autograd.grad(out, (gam, Vr), gVout.to(out.dtype))
            gVin.copy_(g_V.to(gVin.dtype))
    ggamma.copy_(g_gam)


def edge_sum(Ez, row_ptr, factor):
    n = row_ptr.shape[0] - 1
    return torch.zeros(n, dtype=Ez.dtype).index_add_(0, _ctr_of(row_ptr), factor * Ez)


def edge_sum_bwd(gEi, ctr, factor):
    return factor * gEi[ctr.long()]


def force_scatter(gvec, csr, num_atoms_total):
    F = torch.zeros(num_atoms_total, 3, dtype=gvec.dtype)
    F.index_add_(0, _ctr_of(csr.row_ptr), gvec)
    F.index_add_(0, csr.nbr.long(), -gvec)
    return F


def edge_vec(pos, ctr, nbr, shift, acc_dtype):
    v = pos[nbr.long()] - pos[ctr.long()]
    if shift is not None:
        v = v + shift
    return v.to(acc_dtype)


def _radial(dtype, S_rc, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb):
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    x = (vec.norm(dim=-1) / rmax_table[tc, tn]).unsqueeze(-1)
    bw = bessel_w.reshape(1, -1)
    basis = torch.sinc(x * bw) * bw * R.polynomial_cutoff(x, float(p_cut))   # sin(pi w x)/(pi x) f_p(x)
    return torch.cat([cemb[tc], nemb[tn]], dim=-1) * (basis @ Wb)


def radial_fwd(dtype, S_rc, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb):
    return _radial(dtype, S_rc, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb).to(dtype)


def radial_bwd(dtype, S_rc, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb, g_e0, gvec):
    v = vec.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        e0 = _radial(dtype, S_rc, p_cut, v, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb)
        (g,) = torch.autograd.grad(e0, v, g_e0.to(e0.dtype))
    gvec += g


def _radial_pq(p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, PQ):
    T = rmax_table.shape[0]
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    x = (vec.norm(dim=-1) / rmax_table[tc, tn]).unsqueeze(-1)
    bw = bessel_w.reshape(1, -1)
    basis = torch.sinc(x * bw) * bw * R.polynomial_cutoff(x, float(p_cut))
    return torch.einsum("zn,znc->zc", basis, PQ.reshape(T * T, bw.shape[1], -1)[tc * T + tn])


def radial_pq_fwd(dtype, S, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, PQ):
    return _radial_pq(p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, PQ).to(dtype)


def radial_pq_bwd(dtype, S, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, PQ, g_out, aux, gvec):
    v = vec.detach().clone().requires_grad_(True)
    g = g_out.to(vec.dtype)
    if aux is not None:
        g = g * _dsilu(aux.to(vec.dtype))
    with torch.enable_grad():
        out = _radial_pq(p_cut, v, ctr, nbr, types, rmax_table, bessel_w, PQ)
        (gv,) = torch.autograd.grad(out, v, g)
    gvec += gv


def _zbl(p_cut, qq, vec, ctr, nbr, types, Z, rmax_table):
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    r = vec.norm(dim=-1)
    zi, zj = Z[tc], Z[tn]
    xs = (zi**0.23 + zj**0.23) * r / 0.46850
    phi = 0.18175 * torch.exp(-3.19980 * xs) + 0.50986 * torch.exp(-0.94229 * xs) + 0.28022 * torch.exp(-0.40290 * xs) + 0.02817 * torch.exp(-0.20162 * xs)
    return qq * zi * zj / r * phi * R.polynomial_cutoff(r / rmax_table[tc, tn], float(p_cut))


def zbl(p_cut, qq, vec, ctr, nbr, types, Z, rmax_table, gvec):
    v = vec.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        e = _zbl(p_cut, qq, v, ctr, nbr, types, Z, rmax_table)
        if gvec is not None:
            (gv,) = torch.autograd.grad(e.sum(), v)
            gvec += gv
    return e.detach()


# ---- operator-level kernels (reference "strided" layout [z][u][i], unsorted scatter indices) -----------------------
def transpose_ui(x, to_internal):
    return x.transpose(1, 2).contiguous()


def op_scatter_env(x2, idxs, n, sf):
    return torch.zeros((n,) + tuple(x2.shape[1:]), dtype=x2.dtype).index_add_(0, idxs, sf * x2)


def op_gather_rows(src, idxs, sf):
    return sf * src[idxs]


def op_contract(mode, U, d1, d2, dout, tab, cgw, a, b, idxs, out):
    res = torch.zeros_like(out)
    for n, (i, j, k) in enumerate(tab.tolist()):
        c = cgw[n].unsqueeze(0)
        if mode == 0:
            res[:, :, k] += c * a[:, :, i] * b[idxs][:, :, j]
        elif mode == 1:
            res[:, :, i] += c * a[:, :, k] * b[idxs][:, :, j]
        else:
            term = torch.zeros(a.shape[0], U, d2, dtype=a.dtype)
            term[:, :, j] = c * a[:, :, i] * b[:, :, k]
            res.index_add_(0, idxs, term)
    out.copy_(res) if mode != 2 else out.add_(res)
    return out


def op_contract_wgrad(U, d1, d2, dout, tab, x1, gamma, gout, idxs):
    out = torch.zeros(tab.shape[0], U, dtype=x1.dtype)
    g = gamma[idxs]
    for n, (i, j, k) in enumerate(tab.tolist()):
        out[n] = (x1[:, :, i] * g[:, :, j] * gout[:, :, k]).sum(0)
    return out


OPERATOR = ("transpose_ui", "op_scatter_env", "op_gather_rows", "op_contract", "op_contract_wgrad")

ALL = ("zbl", "radial_pq_fwd", "radial_pq_bwd", "sh_fwd", "sh_bwd", "linear", "linear_pack", "env_sum", "env_bwd", "tp_fwd", "tp_bwd", "edge_sum", "edge_sum_bwd",
       "force_scatter", "edge_vec", "radial_fwd", "radial_bwd")
