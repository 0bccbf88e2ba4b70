"""Two-body SPLINE scalar embedding (the reference's alternative to the Bessel embedding;
/root/reference/allegro/nn/spline.py:8-89, scalarembed.py:84-175) on the device.

This is the upstream scalar track (SURVEY.md section 8 row f1/f4), outside the named hot path: it is
evaluated with plain torch ops in fp64 (the reference evaluates it in nequip's global dtype), but with a
hand-written adjoint like the rest of the force path -- no autograd graph, no host synchronisation, so
the whole evaluation stays CUDA-graph capturable.  The functions are device-agnostic; the CPU tests
run exactly this code against the oracle.

    basis_k(x) = 1/4 (1 - cos(c (clamp(x, lo_k, up_k) - lo_k)))^2,  c = 2 pi / (up_k - lo_k)
    e0[z, ch]  = sum_k W[class_z, ch, k] basis_k(x_z),   class = t_centre * T + t_neighbour
"""
from __future__ import annotations

from typing import Tuple

import torch


def spline_basis(x: torch.Tensor, lower: torch.Tensor, upper: torch.Tensor, const: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """x [E] -> (basis [E,K], d basis / dx [E,K])."""
    xc = x.unsqueeze(-1)
    t = const * (torch.clamp(xc, min=lower, max=upper) - lower)
    one_m_cos = 1.0 - torch.cos(t)
    inside = (xc > lower) & (xc < upper)
    return 0.25 * one_m_cos.square(), 0.5 * const * one_m_cos * torch.sin(t) * inside


def spline_forward(vec: torch.Tensor, tc: torch.Tensor, tn: torch.Tensor, rmax_table: torch.Tensor, lower: torch.Tensor,
                   upper: torch.Tensor, const: float, w_flat: torch.Tensor, num_types: int, out_dtype: torch.dtype):
    """vec [E,3], centre / neighbour types [E] (int64), rmax_table [T,T] fp64, w_flat [(T*T)*K, C] fp64
    (row (class, k), column channel) -> (e0 [E,C] in out_dtype, saved tensors for spline_backward)."""
    E, K = vec.shape[0], lower.shape[0]
    v = vec.to(torch.float64)
    r = v.norm(dim=-1)
    rmax = rmax_table[tc, tn]
    basis, dbasis = spline_basis(r / rmax, lower, upper, const)
    cls = tc * num_types + tn
    ar = torch.arange(E, device=vec.device)
    onehot = torch.zeros(E, num_types * num_types, K, dtype=torch.float64, device=vec.device)
    onehot[ar, cls] = basis  # scatter of the basis row into its class block: one GEMM serves all classes, no host sync
    e0 = onehot.view(E, -1) @ w_flat
    return e0.to(out_dtype), (v, r, rmax, dbasis, cls, ar)


def spline_backward(saved, g_e0: torch.Tensor, w_flat: torch.Tensor, num_types: int) -> torch.Tensor:
    """g_e0 [E,C] = dE/de0 -> dE/dvec [E,3] (fp64) through x = |vec| / r_max."""
    v, r, rmax, dbasis, cls, ar = saved
    E, K = dbasis.shape
    t = (g_e0.to(torch.float64) @ w_flat.T).view(E, num_types * num_types, K)[ar, cls]  # [E,K]: sum_ch g W[class,ch,k]
    gx = (t * dbasis).sum(-1)
    return (gx / (rmax * r)).unsqueeze(-1) * v


# ---- tangents along edge-vector directions vdot (nn._hessian) --------------------------------------------------------
def _spline_d2basis(x: torch.Tensor, lower: torch.Tensor, upper: torch.Tensor, const: float) -> torch.Tensor:
    """d2 basis / dx2 [E,K] = c^2 / 2 (sin^2 t + (1 - cos t) cos t) inside (lo_k, up_k), else 0."""
    xc = x.unsqueeze(-1)
    t = const * (torch.clamp(xc, min=lower, max=upper) - lower)
    inside = (xc > lower) & (xc < upper)
    return 0.5 * const * const * (torch.sin(t).square() + (1.0 - torch.cos(t)) * torch.cos(t)) * inside


def spline_jvp(vec, vdot, tc, tn, rmax_table, lower, upper, const: float, w_flat, num_types: int, out_dtype):
    """d e0 / d vec . vdot [E,C] in out_dtype, e0 of ``spline_forward``."""
    E, K = vec.shape[0], lower.shape[0]
    v, w = vec.to(torch.float64), vdot.to(torch.float64)
    r = v.norm(dim=-1)
    rmax = rmax_table[tc, tn]
    _, dbasis = spline_basis(r / rmax, lower, upper, const)
    xd = (v * w).sum(-1) / (r * rmax)
    cls = tc * num_types + tn
    onehot = torch.zeros(E, num_types * num_types, K, dtype=torch.float64, device=vec.device)
    onehot[torch.arange(E, device=vec.device), cls] = dbasis * xd.unsqueeze(-1)
    return (onehot.view(E, -1) @ w_flat).to(out_dtype)


def spline_hvp(vec, vdot, tc, tn, rmax_table, lower, upper, const: float, w_flat, num_types: int, g_e0) -> torch.Tensor:
    """(d2 sum_ch g_e0 e0 / dvec2) . vdot [E,3] fp64: with F(x) = sum_k t_k basis_k(x), t = g_e0 W[class],
    F'' (r_hat.v) r_hat / r_max^2 + F' / (r_max |r|) (v - (r_hat.v) r_hat)."""
    E, K = vec.shape[0], lower.shape[0]
    v, w = vec.to(torch.float64), vdot.to(torch.float64)
    r = v.norm(dim=-1)
    rmax = rmax_table[tc, tn]
    x = r / rmax
    _, d1 = spline_basis(x, lower, upper, const)
    d2 = _spline_d2basis(x, lower, upper, const)
    cls = tc * num_types + tn
    t = (g_e0.to(torch.float64) @ w_flat.T).view(E, num_types * num_types, K)[torch.arange(E, device=vec.device), cls]
    F1, F2 = (t * d1).sum(-1), (t * d2).sum(-1)
    u = v / r.unsqueeze(-1)
    uv = (u * w).sum(-1, keepdim=True)
    return (F2 / (rmax * rmax)).unsqueeze(-1) * uv * u + (F1 / (rmax * r)).unsqueeze(-1) * (w - uv * u)
