"""Plain-torch restatement of the tangent kernels (csrc/hvp.cu, csrc/radial.cu ab2_radial_*_jvp / _hvp, csrc/fc.cu tangent
mode; include/allegro_b200.h) -- TEST INFRASTRUCTURE.

Each function has the signature of its ctypes wrapper in allegro_b200/_lib.py and states the kernel's algebra explicitly:
the chain through u = r/|r| (SH) or x = |r|/r_max (radial basis, ZBL) and the closed-form second derivatives of the
basis, the cutoff and the nonlinearities.  Only the derivatives of the SH polynomials in their free variables come from
autograd, as the generator (tools/gen_sh.py) takes them with sympy.  tests/test_host_hvp.py checks every function
against torch.func.jvp / double autograd of the oracle's primal functions; the GPU tests check the kernels against these.
"""
import math

import torch

import fc_spec
from oracle import o3_ref


# ---- spherical harmonics ----------------------------------------------------------------------------------------------
def _poly(lmax, u):
    """The SH polynomials in the free variables u (no normalisation)."""
    return o3_ref.spherical_harmonics(lmax, u, normalize=False, method="explicit" if lmax <= 3 else "recursive")


def _unit(vec, vdot):
    rho = vec.norm(dim=-1, keepdim=True)
    u = vec / rho
    uv = (u * vdot).sum(-1, keepdim=True)
    return rho, u, uv, (vdot - uv * u) / rho


def sh_jvp(vec, vdot, lmax):
    """Yd = J_P(u) u_dot, u_dot = (v - (u.v) u) / |r|."""
    rho, u, uv, ud = _unit(vec, vdot)
    if vec.shape[0] == 0:
        return torch.zeros(0, (lmax + 1) ** 2, dtype=vec.dtype)
    return torch.func.jvp(lambda w: _poly(lmax, w), (u,), (ud,))[1]


def sh_hvp(vec, vdot, gY, lmax, gvec_dot):
    """gvec_dot += (q_dot - s_dot u - s u_dot) / rho - (q - s u) (u.v) / rho^2 with q = grad G(u), G = sum_k g_k P_k,
    s = u.q, q_dot = Hess G(u) u_dot, s_dot = u_dot.q + u.q_dot."""
    if vec.shape[0] == 0:
        return
    rho, u, uv, ud = _unit(vec, vdot)

    def grad_G(w):
        return torch.func.vjp(lambda t: _poly(lmax, t), w)[1](gY)[0]

    q, qd = torch.func.jvp(grad_G, (u,), (ud,))
    s = (u * q).sum(-1, keepdim=True)
    sd = (ud * q).sum(-1, keepdim=True) + (u * qd).sum(-1, keepdim=True)
    gvec_dot += (qd - sd * u - s * ud) / rho - (q - s * u) * uv / rho**2


# ---- the MLP nonlinearities' second derivatives ------------------------------------------------------------------------
def d2phi(code, x):
    from allegro_b200 import _lib

    x = x.double()
    if code == _lib.NL_SILU:
        s = torch.sigmoid(x)
        return s * (1 - s) * (2 + x * (1 - 2 * s))
    if code == _lib.NL_MISH:
        sg = torch.sigmoid(x)
        t = torch.tanh(torch.nn.functional.softplus(x))
        return (1 - t * t) * sg * (2 + x * (1 - sg - 2 * t * sg))
    if code == _lib.NL_GELU:
        return torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi) * (2 - x * x)
    raise KeyError(code)


def dphi(code, x):
    from allegro_b200.nn._mlp import NONLINEARITIES

    return next(nl for nl in NONLINEARITIES.values() if nl.code == code).dphi(x.double())


def act_bwd_jvp(ga_dot, ga, pre, pre_dot, nonlin):
    out = ga.double() * d2phi(nonlin, pre) * pre_dot.double()
    if ga_dot is not None:
        out = out + ga_dot.double() * dphi(nonlin, pre)
    return out.to(ga.dtype)


# ---- radial basis and cutoff --------------------------------------------------------------------------------------------
def bessel_derivs(x, bw, p):
    """B_n'(x), B_n''(x) [E,nb] of B_n = sin(pi w_n x)/(pi x) f_p(x), zero for x >= 1."""
    x = x.unsqueeze(-1)
    a, b, c = (p + 1) * (p + 2) / 2, p * (p + 2), p * (p + 1) / 2
    f = 1 - a * x**p + b * x ** (p + 1) - c * x ** (p + 2)
    df = -a * p * x ** (p - 1) + b * (p + 1) * x**p - c * (p + 2) * x ** (p + 1)
    d2f = -a * p * (p - 1) * x ** (p - 2) + b * (p + 1) * p * x ** (p - 1) - c * (p + 2) * (p + 1) * x**p
    w = bw.reshape(1, -1)
    s = torch.sin(math.pi * w * x) / (math.pi * x)
    ds = (w * torch.cos(math.pi * w * x) - s) / x
    d2s = -((math.pi * w) ** 2) * s - 2 * ds / x
    inside = x < 1
    return (ds * f + s * df) * inside, (d2s * f + 2 * ds * df + s * d2f) * inside


def _radial_m(types, ctr, nbr, rmax_table, PQ=None, Wb=None, cemb=None, nemb=None, nb=8):
    """M[z][n][c] of the edge's type pair for either route, and x = |r| / r_max's r_max per edge."""
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    if PQ is not None:
        T = rmax_table.shape[0]
        M = PQ.reshape(T * T, nb, -1)[tc * T + tn]
    else:
        M = torch.cat([cemb[tc], nemb[tn]], dim=-1).unsqueeze(1) * Wb.unsqueeze(0)
    return M, rmax_table[tc, tn]


def _radial_jvp(p_cut, vec, vdot, M, rmax, bessel_w):
    r = vec.norm(dim=-1)
    d1, _ = bessel_derivs(r / rmax, bessel_w, float(p_cut))
    xd = (vec * vdot).sum(-1) / (r * rmax)
    return torch.einsum("zn,znc->zc", d1, M) * xd.unsqueeze(-1)


def _radial_hvp(p_cut, vec, vdot, M, rmax, bessel_w, g):
    """F'' (u.v) u / r_max^2 + F' / (r_max |r|) (v - (u.v) u), F = sum_c g_c out_c(x)."""
    r = vec.norm(dim=-1)
    d1, d2 = bessel_derivs(r / rmax, bessel_w, float(p_cut))
    G = torch.einsum("zc,znc->zn", g, M)
    F1, F2 = (d1 * G).sum(-1), (d2 * G).sum(-1)
    u = vec / r.unsqueeze(-1)
    uv = (u * vdot).sum(-1, keepdim=True)
    return (F2 / rmax**2).unsqueeze(-1) * uv * u + (F1 / (rmax * r)).unsqueeze(-1) * (vdot - uv * u)


def radial_pq_jvp(dtype, S, p_cut, vec, vdot, ctr, nbr, types, rmax_table, bessel_w, PQ):
    M, rmax = _radial_m(types, ctr, nbr, rmax_table, PQ=PQ, nb=bessel_w.numel())
    return _radial_jvp(p_cut, vec, vdot, M, rmax, bessel_w).to(dtype)


def radial_jvp(dtype, S_rc, p_cut, vec, vdot, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb):
    M, rmax = _radial_m(types, ctr, nbr, rmax_table, Wb=Wb, cemb=cemb, nemb=nemb)
    return _radial_jvp(p_cut, vec, vdot, M, rmax, bessel_w).to(dtype)


def radial_pq_hvp(dtype, S, p_cut, vec, vdot, ctr, nbr, types, rmax_table, bessel_w, PQ, g_out, aux, gvec_dot, nonlin=1):
    M, rmax = _radial_m(types, ctr, nbr, rmax_table, PQ=PQ, nb=bessel_w.numel())
    g = g_out.to(vec.dtype)
    if aux is not None:
        g = g * dphi(nonlin, aux).to(vec.dtype)
    gvec_dot += _radial_hvp(p_cut, vec, vdot, M, rmax, bessel_w, g)


def radial_hvp(dtype, S_rc, p_cut, vec, vdot, ctr, nbr, types, rmax_table, bessel_w, Wb, cemb, nemb, g_e0, gvec_dot):
    M, rmax = _radial_m(types, ctr, nbr, rmax_table, Wb=Wb, cemb=cemb, nemb=nemb)
    gvec_dot += _radial_hvp(p_cut, vec, vdot, M, rmax, bessel_w, g_e0.to(vec.dtype))


# ---- ZBL ----------------------------------------------------------------------------------------------------------------
_ZBL_B = (0.20162, 0.40290, 0.94229, 3.19980)
_ZBL_C = (0.02817, 0.28022, 0.50986, 0.18175)


def zbl_hvp(p_cut, qq, vec, vdot, ctr, nbr, types, Z, rmax_table, gvec_dot):
    """e(r) = K A(r) / r, A = phi(s r) u(r / r_max):  e'' (u.v) u + e'/r (v - (u.v) u), zero beyond r_max."""
    p = float(p_cut)
    tc, tn = types.long()[ctr.long()], types.long()[nbr.long()]
    r = vec.norm(dim=-1)
    zi, zj = Z[tc], Z[tn]
    rmax = rmax_table[tc, tn]
    x = r / rmax
    a, b, c = (p + 1) * (p + 2) / 2, p * (p + 2), p * (p + 1) / 2
    uc = 1 - a * x**p + b * x ** (p + 1) - c * x ** (p + 2)
    du = (-a * p * x ** (p - 1) + b * (p + 1) * x**p - c * (p + 2) * x ** (p + 1)) / rmax
    d2u = (-a * p * (p - 1) * x ** (p - 2) + b * (p + 1) * p * x ** (p - 1) - c * (p + 2) * (p + 1) * x**p) / rmax**2
    s = (zi**0.23 + zj**0.23) / 0.46850
    ek = [ck * torch.exp(-bk * s * r) for bk, ck in zip(_ZBL_B, _ZBL_C)]
    phi = sum(ek)
    dphi_ = s * sum(-bk * e for bk, e in zip(_ZBL_B, ek))
    d2phi_ = s * s * sum(bk * bk * e for bk, e in zip(_ZBL_B, ek))
    A, dA, d2A = phi * uc, dphi_ * uc + phi * du, d2phi_ * uc + 2 * dphi_ * du + phi * d2u
    K = qq * zi * zj
    de = K * (dA / r - A / r**2)
    d2e = K * (d2A / r - 2 * dA / r**2 + 2 * A / r**3)
    inside = (x < 1).to(vec.dtype)
    u = vec / r.unsqueeze(-1)
    uv = (u * vdot).sum(-1, keepdim=True)
    gvec_dot += inside.unsqueeze(-1) * ((d2e.unsqueeze(-1) * uv) * u + (de / r).unsqueeze(-1) * (vdot - uv * u))


# ---- force-constant gather / fold, tangent mode ----------------------------------------------------------------------
def fc_gather_tangent(pos, shift, acc_dtype, atoms, cptr, cen, coff, ea, row_ptr, nbr, u0, u1):
    """Units [u0, u1) one job each: ``fc_spec.gather``'s layout with one job per unit, the undisplaced edge vectors and
    vdot = e_alpha ([nbr = j] - [ctr = j]) -> (row_ptr_b, cen_b, ctr_b, nbr_b, vec_b, vdot_b)."""
    rps, cbs, czs, nzs, vbs, vds = [], [], [], [], [], []
    C0 = E0 = 0
    Cb_total = sum(int(cptr[u // 3 + 1] - cptr[u // 3]) for u in range(u0, u1))
    for u in range(u0, u1):
        a, alpha = divmod(u, 3)
        j = int(atoms[a])
        for c in range(int(cptr[a]), int(cptr[a + 1])):
            k = int(cen[c])
            z0, z1 = int(row_ptr[k]), int(row_ptr[k + 1])
            rps.append(E0)
            cbs.append(k)
            for z in range(z0, z1):
                jn = int(nbr[z])
                czs.append(C0)
                nzs.append(Cb_total + jn)
                vbs.append((pos[jn] - pos[k] + shift[z]).to(acc_dtype))
                d = torch.zeros(3, dtype=acc_dtype)
                d[alpha] = float((jn == j) - (k == j))
                vds.append(d)
                E0 += 1
            C0 += 1
    rps.append(E0)
    stack = (lambda xs: torch.stack(xs) if xs else torch.zeros(0, 3, dtype=acc_dtype))
    return (torch.tensor(rps), torch.tensor(cbs, dtype=torch.int64), torch.tensor(czs, dtype=torch.int64), torch.tensor(nzs, dtype=torch.int64),
            stack(vbs), stack(vds))


def fc_fold_tangent(gvec_dot, atoms, cptr, cen, coff, ea, row_ptr, ctr, nbr, fptr, col, u0, u1):
    """{(p, alpha): -F_dot_i [3] fp64} of units [u0, u1) from one job per unit (the fold of fc_spec without the
    difference and 1/(2h))."""
    out = {}
    e = 0
    for u in range(u0, u1):
        a, alpha = divmod(u, 3)
        cs = cen[int(cptr[a]) : int(cptr[a + 1])].tolist()
        off = {k: e + int(coff[int(cptr[a]) + i]) for i, k in enumerate(cs)}
        for p in range(int(fptr[a]), int(fptr[a + 1])):
            i = int(col[p])
            F = torch.zeros(3, dtype=torch.float64)
            if i in off:
                F += gvec_dot[off[i] : off[i] + int(row_ptr[i + 1] - row_ptr[i])].double().sum(0)
            for z in range(row_ptr[-1]):
                k = int(ctr[z])
                if int(nbr[z]) == i and k in off:
                    F -= gvec_dot[off[k] + z - int(row_ptr[k])].double()
            out[(p, alpha)] = -F
        e += int(ea[a])
    return out


unit_prefix = fc_spec.unit_prefix
