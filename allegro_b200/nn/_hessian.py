"""Forward-mode tangent of the per-edge force path: with the edge vectors moving along ``vdot``, the tangent of
gvec = dE/dvec,  gvec_dot = (d gvec / d vec) . vdot,  so that  H v = -force_scatter(gvec_dot)  (DESIGN.md section 4.11).

Three steps, all on kernels of liballegro_b200.so:

  (a) primal: the forward on the stored-V path (every V_l kept), then a backward that keeps the adjoints the tangent
      backward reads -- the hidden-layer gradients g_a of every MLP, gX, gV_l, g_gamma_l, g_omega_l, gw0, gY.  It runs the
      MLPs as plain GEMM chains (``_mlp_bwd``): the fused MLP kernels of ``AllegroCore.backward`` keep g_a on chip.
  (b) tangent forward: every multilinear step (GEMM, env sum, tensor product) is the primal kernel called once per input
      replaced by its tangent; the nonlinear steps take ab2_sh_jvp and ab2_radial_*_jvp, and the MLP nonlinearity is
      phi'(pre) in the next GEMM's prologue (ACT_MUL_DSILU, aux = pre).
  (c) tangent backward: the readout's output gradient is constant (its tangent is zero); every adjoint kernel is called
      once per replaced input, keeping only the outputs that are tangent terms (the others go to scratch buffers, since
      gY accumulates in place); the curvature terms are ab2_act_bwd_jvp (phi''), ab2_sh_hvp, ab2_radial_*_hvp and
      ab2_zbl_hvp.

The spline embedding runs its primal in torch ops (nn/_spline.py) and so does its tangent.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .. import _lib
from ..data import EdgeCSR


def _lin(mlp, k: int, a_segs: Sequence[torch.Tensor], outs: Sequence[torch.Tensor], aux=None, accum=None, transpose: bool = False):
    """outs (+)= act(cat(a_segs)) @ W_k (W_k^T if ``transpose``), act = phi'(aux) * (.) where ``aux`` is given."""
    kw = dict(act=_lib.ACT_MUL_DSILU, a_aux=list(aux), **mlp.nl_kw) if aux is not None else {}
    W, Wp = (mlp.WT[k], mlp.WTp[k]) if transpose else (mlp.W[k], mlp.Wp[k])
    _lib.linear(list(a_segs), W, list(outs), o_accum=accum, W_packed=Wp, **kw)


def _mlp_tangent(mlp, pre: List[torch.Tensor], k0: int, xd_segs: Sequence[torch.Tensor], out_segs) -> Dict[int, torch.Tensor]:
    """Tangent forward of layers k0.. of ``mlp`` -> {k: pre_dot_k} of its hidden layers.  ``xd_segs``: the tangent of the
    input of layer k0 (for k0 > 0 the tangent of pre_{k0-1}, whose phi is that input).  ``out_segs`` None: the output
    layer is skipped (the readout's energy tangent is not needed)."""
    M = xd_segs[0].shape[0]
    nl = mlp.nl is not None
    pdot: Dict[int, torch.Tensor] = {}
    cur = list(xd_segs)
    aux = None
    if k0 > 0:
        pdot[k0 - 1] = xd_segs[0]
        aux = [pre[k0 - 1]] if nl else None
    for k in range(k0, mlp.n_layers):
        last = k == mlp.n_layers - 1
        if last and out_segs is None:
            break
        o = list(out_segs) if last else [torch.empty(M, mlp.dims[k + 1], dtype=mlp.dtype, device=xd_segs[0].device)]
        _lin(mlp, k, cur, o, aux=aux)
        if not last:
            pdot[k] = o[0]
            cur, aux = [o[0]], ([pre[k]] if nl else None)
    return pdot


def _mlp_bwd(mlp, pre: List[torch.Tensor], k0: int, gout_segs: Sequence[torch.Tensor], gin_segs: Sequence[torch.Tensor],
             gin_accum: Sequence[bool]) -> Dict[int, torch.Tensor]:
    """Backward of layers k0.. of ``mlp`` as a plain GEMM chain -> {k: g_a_k}, the gradient w.r.t. phi(pre_k) of its hidden
    layers k >= k0.  ``gin_segs`` (+)= the gradient w.r.t. the input of layer k0."""
    M = gout_segs[0].shape[0]
    nl = mlp.nl is not None
    ga: Dict[int, torch.Tensor] = {}
    cur, aux = list(gout_segs), None
    for k in range(mlp.n_layers - 1, k0 - 1, -1):
        if k == k0:
            _lin(mlp, k, cur, gin_segs, aux=aux, accum=list(gin_accum), transpose=True)
        else:
            g = torch.empty(M, mlp.dims[k], dtype=mlp.dtype, device=gout_segs[0].device)
            _lin(mlp, k, cur, [g], aux=aux, transpose=True)
            ga[k - 1] = g
            cur, aux = [g], ([pre[k - 1]] if nl else None)
    return ga


def _mlp_bwd_tangent(mlp, pre, pdot, ga, k0: int, gdot_out: Optional[Sequence[torch.Tensor]], gin_dot: Sequence[torch.Tensor]):
    """Tangent of ``_mlp_bwd``: gin_dot += d(gin)/d(...) . tangents, with g_pre_dot_k = g_a_dot_k phi'(pre_k) +
    g_a_k phi''(pre_k) pre_dot_k (ab2_act_bwd_jvp) at every hidden layer.  ``gdot_out`` None: the output gradient is
    constant.  ``gin_dot`` must hold a value to add to (zeros at first)."""
    nl = mlp.nl
    cur = list(gdot_out) if gdot_out is not None else None
    for k in range(mlp.n_layers - 1, k0 - 1, -1):
        gad = None
        if cur is not None:
            if k == k0:
                _lin(mlp, k, cur, gin_dot, accum=[True] * len(gin_dot), transpose=True)
            else:
                gad = torch.empty(cur[0].shape[0], mlp.dims[k], dtype=mlp.dtype, device=cur[0].device)
                _lin(mlp, k, cur, [gad], transpose=True)
        if k > k0:
            if nl is not None:
                cur = [_lib.act_bwd_jvp(gad, ga[k - 1], pre[k - 1], pdot[k - 1], nl.code)]
            else:
                cur = [gad] if gad is not None else None


def hvp_edge_bytes(core) -> int:
    """Device bytes ``edge_energy_grad_tangent`` allocates per edge, counted from the model's widths: the primal
    activations and the kept adjoints, their tangents and the scratch outputs of the replaced-input adjoint calls, with
    the per-centre tensors (gamma and its gradients, 8 per layer, counted against 16 edges per centre) and 50 % headroom."""
    es = torch.empty(0, dtype=core.dtype).element_size()
    ac = torch.empty(0, dtype=core.acc).element_size()
    hid = max([core.readout.dims[1]] + [ly["mlp"].dims[1] for ly in core.layers] + [core.S])
    tp = sum(ly["d_out"] * core.U for ly in core.layers)
    act = 4 * core.S * (core.L + 1) + 9 * core.nw * (core.L + 1) + 8 * tp + 4 * hid * (core.L + 2) + 4 * core.S_in
    per_centre = 8 * core.L * core.D * core.U // 16
    return int(1.5 * (es * act + ac * (6 * core.D + 18 + per_centre) + 12))


def _tp_fwd(core, l: int, csr: EdgeCSR, gamma, Vin, Y, w0) -> torch.Tensor:
    ly = core.layers[l]
    E = csr.num_edges
    out = torch.empty(E, ly["d_out"], core.U, dtype=core.dtype, device=Y.device)
    _lib.tp_fwd(core.dtype, core.lmax, csr.num_atoms, E, core.U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr, gamma, Vin, Y,
                w0, out)
    return out


def _tp_bwd(core, l: int, csr: EdgeCSR, gamma, Vin, Y, w0, gVout, gVin, gw0, gY, ggamma):
    ly = core.layers[l]
    _lib.tp_bwd(core.dtype, core.lmax, csr.num_atoms, csr.num_edges, core.U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr,
                gamma, Vin, Y, w0, gVout, gVin, gw0, gY, ggamma)


def edge_energy_grad_tangent(core, up, csr: EdgeCSR, vec: torch.Tensor, vdot: torch.Tensor, types_i32: torch.Tensor,
                             gEi_scale: Optional[torch.Tensor], pair=None):
    """Edge vectors ``vec`` and their tangent ``vdot`` [E,3] (acc dtype, CSR order, E > 0) -> (gvec, gvec_dot) [E,3] acc
    dtype: gvec = d E_total / d vec as ``_pipeline.edge_energy_grad`` gives it (to rounding), gvec_dot its tangent along
    vdot.  Arguments as ``edge_energy_grad``; positions never enter."""
    dt, acc, dev = core.dtype, core.acc, vec.device
    E, N, U, S, L, D, nw = csr.num_edges, csr.num_atoms, core.U, core.S, core.L, core.D, core.nw
    assert vec.dtype == acc and vdot.dtype == acc and vdot.shape == vec.shape and E > 0
    lmax, sf = core.lmax, core.sf
    ctr, nbr, row_ptr = csr.ctr, csr.nbr, csr.row_ptr

    def zeros(*shape, dtype=dt):
        return torch.zeros(*shape, dtype=dtype, device=dev)

    def empty(*shape, dtype=dt):
        return torch.empty(*shape, dtype=dtype, device=dev)

    # ---- (a) primal forward (stored-V path) ---------------------------------------------------------------------
    _lib.set_tag("hvp.fwd")
    box = []
    _, _, _, sv = core.forward(csr, vec, None, fill_embed=lambda w0, x0, om0: box.append(up.forward(vec, csr, types_i32, [w0, x0, om0], keep_h=True)),
                               stored_v=True)
    kind, sp_saved, up_pre = box[0]
    k0_up = 1 if kind == "pq_fold" else 0

    # ---- (a) primal backward, keeping the adjoints ----------------------------------------------------------------
    _lib.set_tag("hvp.bwd")
    gEi = gEi_scale if gEi_scale is not None else torch.ones(N, dtype=acc, device=dev)
    gEz = _lib.edge_sum_bwd(gEi.contiguous(), ctr, core.factor).to(dt).view(E, 1)
    gX = zeros(E, S * (L + 1))
    ga_read = _mlp_bwd(core.readout, sv.pre_read, 0, [gEz], [gX], [True])
    gY = zeros(E, D, dtype=acc)
    gV: List[Optional[torch.Tensor]] = [None] * (L + 1)
    gom: List[Optional[torch.Tensor]] = [None] * (L + 1)
    ggam: List[Optional[torch.Tensor]] = [None] * L
    ga_lat: List[Optional[Dict[int, torch.Tensor]]] = [None] * L
    gw0 = None
    for l in range(L - 1, -1, -1):
        ly = core.layers[l]
        if ly["last"]:
            gV[l + 1] = zeros(E, ly["d_out"], U)
        gs = gV[l + 1].view(E, ly["d_out"] * U)[:, :U]
        gouts = [gX[:, S * (l + 1) : S * (l + 2)]] + ([] if ly["last"] else [gom[l + 1]])
        ga_lat[l] = _mlp_bwd(ly["mlp"], sv.pre_lat[l], 0, gouts, [gX[:, : S * (l + 1)], gs], [True, True])
        ggam[l] = empty(N, D, U, dtype=acc)
        if l == 0:
            gw0 = empty(E, nw)
            _tp_bwd(core, 0, csr, sv.gamma[0], None, sv.Y, sv.w0, gV[1], None, gw0, gY, ggam[0])
        else:
            gV[l] = empty(E, ly["d_in"], U)
            _tp_bwd(core, l, csr, sv.gamma[l], sv.V[l], None, None, gV[l + 1], gV[l], None, None, ggam[l])
        gom[l] = empty(E, nw)
        _lib.env_bwd(dt, lmax, U, ctr, sv.Y, sv.omega[l], ggam[l], sf, gom[l], gY, row_ptr=row_ptr)
    g_emb = [gw0, gX[:, :S], gom[0]]
    gvec = _lib.sh_bwd(vec, gY, lmax)
    g_r = empty(E, up.mlp.dims[k0_up])  # gradient w.r.t. the radial output (pq_fold: w.r.t. phi(h))
    ga_up = _mlp_bwd(up.mlp, up_pre, k0_up, g_emb, [g_r], [False])
    _radial_bwd(up, kind, sp_saved, up_pre, vec, csr, types_i32, g_r, gvec)
    if pair is not None:
        pair[0].edge_energy_and_grad(vec, csr, types_i32, pair[1], gvec)

    # ---- (b) tangent forward --------------------------------------------------------------------------------------
    _lib.set_tag("hvp.tfwd")
    Yd = _lib.sh_jvp(vec, vdot, lmax)
    Xd = empty(E, S * (L + 1))
    w0d, omd = empty(E, nw), [empty(E, nw)]
    emb_outs = [w0d, Xd[:, :S], omd[0]]
    rd = _radial_jvp(up, kind, vec, vdot, csr, types_i32)
    pd_up = _mlp_tangent(up.mlp, up_pre, k0_up, [rd], emb_outs)
    Vd: List[Optional[torch.Tensor]] = [None] * (L + 1)
    gamd: List[torch.Tensor] = []
    pd_lat = []
    for l, ly in enumerate(core.layers):
        gd = _lib.env_sum(dt, lmax, N, U, row_ptr, Yd, sv.omega[l], sf)
        gd += _lib.env_sum(dt, lmax, N, U, row_ptr, sv.Y, omd[l], sf)
        gamd.append(gd)
        if l == 0:
            v1 = _tp_fwd(core, 0, csr, gd, None, sv.Y, sv.w0)
            v1 += _tp_fwd(core, 0, csr, sv.gamma[0], None, Yd, sv.w0)
            v1 += _tp_fwd(core, 0, csr, sv.gamma[0], None, sv.Y, w0d)
        else:
            v1 = _tp_fwd(core, l, csr, gd, sv.V[l], sv.Y, None)
            v1 += _tp_fwd(core, l, csr, sv.gamma[l], Vd[l], sv.Y, None)
        Vd[l + 1] = v1
        sd = v1.view(E, ly["d_out"] * U)[:, :U]
        outs = [Xd[:, S * (l + 1) : S * (l + 2)]]
        if not ly["last"]:
            omd.append(empty(E, nw))
            outs.append(omd[l + 1])
        pd_lat.append(_mlp_tangent(ly["mlp"], sv.pre_lat[l], 0, [Xd[:, : S * (l + 1)], sd], outs))
    pd_read = _mlp_tangent(core.readout, sv.pre_read, 0, [Xd], None)

    # ---- (c) tangent backward -------------------------------------------------------------------------------------
    _lib.set_tag("hvp.tbwd")
    gXd = zeros(E, S * (L + 1))
    _mlp_bwd_tangent(core.readout, sv.pre_read, pd_read, ga_read, 0, None, [gXd])
    gYd = zeros(E, D, dtype=acc)
    gY_scratch = zeros(E, D, dtype=acc)     # gY outputs of the calls whose gY part is not a tangent term
    gg_scratch = empty(N, D, U, dtype=acc)  # likewise for g_gamma
    gom_scratch = empty(E, nw)
    gVd: List[Optional[torch.Tensor]] = [None] * (L + 1)
    gomd: List[Optional[torch.Tensor]] = [None] * (L + 1)
    gw0d = None
    for l in range(L - 1, -1, -1):
        ly = core.layers[l]
        if ly["last"]:
            gVd[l + 1] = zeros(E, ly["d_out"], U)
        gsd = gVd[l + 1].view(E, ly["d_out"] * U)[:, :U]
        gouts_d = [gXd[:, S * (l + 1) : S * (l + 2)]] + ([] if ly["last"] else [gomd[l + 1]])
        _mlp_bwd_tangent(ly["mlp"], sv.pre_lat[l], pd_lat[l], ga_lat[l], 0, gouts_d, [gXd[:, : S * (l + 1)], gsd])
        ggd: List[Optional[torch.Tensor]] = [empty(N, D, U, dtype=acc) for _ in range(3)]
        if l == 0:
            # gw0 = f(gamma, Y, gV), gY += f(gamma, w0, gV), g_gamma = f(Y, w0, gV): one call per replaced input
            gw = [empty(E, nw) for _ in range(3)]
            _tp_bwd(core, 0, csr, gamd[0], None, sv.Y, sv.w0, gV[1], None, gw[0], gYd, gg_scratch)
            _tp_bwd(core, 0, csr, sv.gamma[0], None, Yd, sv.w0, gV[1], None, gw[1], gY_scratch, ggd[0])
            _tp_bwd(core, 0, csr, sv.gamma[0], None, sv.Y, w0d, gV[1], None, gom_scratch, gYd, ggd[1])
            _tp_bwd(core, 0, csr, sv.gamma[0], None, sv.Y, sv.w0, gVd[1], None, gw[2], gYd, ggd[2])
            gw0d = gw[0] + gw[1] + gw[2]
        else:
            # gV_in = f(gamma, gV_out), g_gamma = f(V_in, gV_out)
            gvin = [empty(E, ly["d_in"], U) for _ in range(3)]
            _tp_bwd(core, l, csr, gamd[l], sv.V[l], None, None, gV[l + 1], gvin[0], None, None, gg_scratch)
            _tp_bwd(core, l, csr, sv.gamma[l], Vd[l], None, None, gV[l + 1], gvin[2], None, None, ggd[0])  # gvin[2]: scratch
            _tp_bwd(core, l, csr, sv.gamma[l], sv.V[l], None, None, gVd[l + 1], gvin[1], None, None, ggd[1])
            gVd[l] = gvin[0] + gvin[1]
            ggd[2] = None
        ggd_l = ggd[0] + ggd[1] if ggd[2] is None else ggd[0] + ggd[1] + ggd[2]
        # g_omega = f(Y, g_gamma), gY += f(omega, g_gamma)
        go = [empty(E, nw) for _ in range(2)]
        _lib.env_bwd(dt, lmax, U, ctr, Yd, sv.omega[l], ggam[l], sf, go[0], gY_scratch, row_ptr=row_ptr)
        _lib.env_bwd(dt, lmax, U, ctr, sv.Y, omd[l], ggam[l], sf, gom_scratch, gYd, row_ptr=row_ptr)
        _lib.env_bwd(dt, lmax, U, ctr, sv.Y, sv.omega[l], ggd_l, sf, go[1], gYd, row_ptr=row_ptr)
        gomd[l] = go[0] + go[1]
    g_emb_d = [gw0d, gXd[:, :S], gomd[0]]
    gvec_dot = _lib.sh_bwd(vec, gYd, lmax)
    _lib.sh_hvp(vec, vdot, gY, lmax, gvec_dot)
    g_rd = zeros(E, up.mlp.dims[k0_up])
    _mlp_bwd_tangent(up.mlp, up_pre, pd_up, ga_up, k0_up, g_emb_d, [g_rd])
    _radial_bwd_tangent(up, kind, sp_saved, up_pre, pd_up, vec, vdot, csr, types_i32, g_r, g_rd, gvec_dot)
    if pair is not None:
        zbl = pair[0]
        Z = zbl.atomic_numbers.to(device=dev, dtype=acc)
        _lib.zbl_hvp(zbl.CUTOFF_P, zbl.qq, vec, vdot, ctr, nbr, types_i32, Z, pair[1].to(acc).contiguous(), gvec_dot)
    return gvec, gvec_dot


# ---- the radial embedding's three routes and the spline -------------------------------------------------------------
def _radial_bwd(up, kind, sp_saved, pre, vec, csr, types_i32, g_r, gvec):
    """gvec += the radial adjoint of g_r, as ``UpstreamPack.backward`` applies it."""
    dt = up.dtype
    if kind == "pq_fold":
        _lib.radial_pq_bwd(dt, up.S_pq, up.p, vec, csr.ctr, csr.nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_r, pre[0], gvec, **up.mlp.nl_kw)
    elif kind == "spline":
        from ._spline import spline_backward

        gvec += spline_backward(sp_saved, g_r, up.sp_w, up.num_types).to(gvec.dtype)
    elif up.PQ is not None:
        _lib.radial_pq_bwd(dt, up.S_pq, up.p, vec, csr.ctr, csr.nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_r, None, gvec)
    else:
        _lib.radial_bwd(dt, up.S_rc, up.p, vec, csr.ctr, csr.nbr, types_i32, up.rmax_table, up.bessel_w, up.Wb, up.cemb, up.nemb, g_r, gvec)


def _radial_jvp(up, kind, vec, vdot, csr, types_i32) -> torch.Tensor:
    """Tangent of the radial output (pq_fold: of the pre-activation h)."""
    dt = up.dtype
    if kind == "spline":
        from ._spline import spline_jvp

        t64 = types_i32.long()
        return spline_jvp(vec, vdot, t64[csr.ctr.long()], t64[csr.nbr.long()], up.rmax64, up.sp_lower, up.sp_upper, up.sp_const, up.sp_w,
                          up.num_types, dt)
    if up.PQ is not None:
        return _lib.radial_pq_jvp(dt, up.S_pq, up.p, vec, vdot, csr.ctr, csr.nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ)
    return _lib.radial_jvp(dt, up.S_rc, up.p, vec, vdot, csr.ctr, csr.nbr, types_i32, up.rmax_table, up.bessel_w, up.Wb, up.cemb, up.nemb)


def _radial_bwd_tangent(up, kind, sp_saved, pre, pdot, vec, vdot, csr, types_i32, g_r, g_rd, gvec_dot):
    """gvec_dot += the radial adjoint of g_rd + the basis-curvature term of g_r (and, pq_fold, the phi'' term)."""
    dt = up.dtype
    ctr, nbr = csr.ctr, csr.nbr
    if kind == "pq_fold":
        nl = up.mlp.nl
        g_hd = _lib.act_bwd_jvp(g_rd, g_r, pre[0], pdot[0], nl.code)
        _lib.radial_pq_bwd(dt, up.S_pq, up.p, vec, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_hd, None, gvec_dot)
        _lib.radial_pq_hvp(dt, up.S_pq, up.p, vec, vdot, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_r, pre[0], gvec_dot, nl.code)
    elif kind == "spline":
        from ._spline import spline_backward, spline_hvp

        t64 = types_i32.long()
        gvec_dot += spline_backward(sp_saved, g_rd, up.sp_w, up.num_types).to(gvec_dot.dtype)
        gvec_dot += spline_hvp(vec, vdot, t64[ctr.long()], t64[nbr.long()], up.rmax64, up.sp_lower, up.sp_upper, up.sp_const, up.sp_w,
                               up.num_types, g_r).to(gvec_dot.dtype)
    elif up.PQ is not None:
        _lib.radial_pq_bwd(dt, up.S_pq, up.p, vec, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_rd, None, gvec_dot)
        _lib.radial_pq_hvp(dt, up.S_pq, up.p, vec, vdot, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.PQ, g_r, None, gvec_dot)
    else:
        _lib.radial_bwd(dt, up.S_rc, up.p, vec, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.Wb, up.cemb, up.nemb, g_rd, gvec_dot)
        _lib.radial_hvp(dt, up.S_rc, up.p, vec, vdot, ctr, nbr, types_i32, up.rmax_table, up.bessel_w, up.Wb, up.cemb, up.nemb, g_r, gvec_dot)
