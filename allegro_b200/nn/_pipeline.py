"""The fused per-edge pipeline: SH embedding -> L x (env sum, CG tensor product, latent MLP)
-> readout MLP -> edge->atom energy sum, forward AND hand-written backward (forces), all in
liballegro_b200.so.

Replaces, for centre-sorted CSR edges, the reference call stack
  TwoBodySphericalHarmonicTensorEmbed.forward  (allegro/nn/tensorembed.py:85-96)
  Allegro_Module.forward                       (allegro/nn/_allegro.py:237-301)
  edge_readout ScalarMLP                       (allegro/model/allegro_models.py:231-241)
  EdgewiseReduce.forward                       (allegro/nn/edgewise.py:40-60)
and their autograd backward (SURVEY appendix B).

HBM layout (DESIGN.md section 3): per-edge tensors are edge-major, edges sorted by centre;
tensor features are component-major V[E][d][U] (channel fastest), env weights w[E][n_ir][U];
the densenet scalars x_0..x_L live in ONE buffer X[E][S(L+1)] that every MLP writes a column
block of (so torch.cat of _allegro.py:278,300 never happens).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from .. import _lib
from ..data import EdgeCSR
from ._mlp import PackedMLP


def _env_perm(U: int, n_ir: int, individual: bool = True) -> torch.Tensor:
    """Column gather that brings the reference's env-weight columns into the internal [r][u] order.
    individual weights: internal column r*U+u <- reference column u*n_ir+r (_channels.py:46-51);
    shared weights (weight_individual_irreps=False, _channels.py:56-63): every irrep r reads the
    same reference column u, i.e. the U columns are replicated n_ir times."""
    r = torch.arange(n_ir).view(-1, 1)
    u = torch.arange(U).view(1, -1)
    if not individual:
        return (u + 0 * r).reshape(-1)
    return (u * n_ir + r).reshape(-1)


class _Saved:
    __slots__ = ("csr", "vec", "Y", "w0", "omega", "V", "gamma", "pre_lat", "pre_read", "X", "fold")


class AllegroCore:
    """Packed weights + kernel sequencing.  Built from the parameter-holding modules by
    ``FusedAllegroEnergy`` (model/allegro_models.py)."""

    def __init__(self, tensor_embed, allegro, edge_readout, avg_num_neighbors: float, dtype: torch.dtype, device):
        self.dtype = dtype
        self.acc = _lib.ACC_DTYPE[dtype]
        self.device = torch.device(device)
        self.lmax = tensor_embed.lmax
        self.D = (self.lmax + 1) ** 2
        self.n_ir = self.lmax + 1
        self.U = allegro.num_tensor_features
        self.S = allegro.num_scalar_features
        self.L = allegro.num_layers
        self.S_in = tensor_embed.env_embed_linear.input_dim
        self.sf = 1.0 / math.sqrt(avg_num_neighbors)
        self.factor = 1.0 / math.sqrt(2.0 * avg_num_neighbors)
        U, n_ir, S = self.U, self.n_ir, self.S
        # the two weighters are configured independently (the reference builder only forwards
        # weight_individual_irreps to Allegro_Module, allegro_models.py:185-216)
        perm = _env_perm(U, n_ir, allegro._env_weighter.weight_individual_irreps)         # omega columns
        perm_w0 = _env_perm(U, n_ir, tensor_embed._edge_weighter.weight_individual_irreps)  # w0 columns
        nw = n_ir * U                                          # internal env-weight width
        nw0_ref = tensor_embed._edge_weighter.weight_numel     # reference width of the w0 linear
        # one GEMM for both linears that read the two-body embedding:
        #   [ w0 (tensorembed.py:88-89) | x_0 | omega_0 (_allegro.py:251-258) ]
        proj = allegro.first_layer_env_embed_projection.folded_weights()[0]
        proj_perm = torch.cat([torch.arange(S), S + perm])
        self.embed = PackedMLP(
            tensor_embed.env_embed_linear, dtype, device, out_perm=torch.cat([perm_w0, nw0_ref + proj_perm]),
            extra_first=[proj],
        )
        self.layers = []
        for l, (tp, lat) in enumerate(zip(allegro.tps, allegro.latents)):
            last = l == self.L - 1
            ijk, _, _ = tp.sparse_table()
            out_perm = None if last else torch.cat([torch.arange(S), S + perm])
            self.layers.append(
                dict(
                    d_in=tp.base_dim1,
                    d_out=tp.base_dim_out,
                    tab=ijk.to(device),
                    cgw=tp.cgw(self.acc, device),
                    mlp=PackedMLP(lat, dtype, device, out_perm=out_perm),
                    last=last,
                )
            )
            assert tp.base_dim2 == self.D
        self.readout = PackedMLP(edge_readout, dtype, device)
        self.nw = nw
        # "plain GEMM" backward plan (all latent/readout MLPs are 2-layer SiLU): the gradient of the
        # densenet block x_b is ONE GEMM over all its consumers (readout, latents m >= b), concatenated
        # along K, each consumer's g_h scaled by silu'(pre) in the GEMM prologue -- no accumulation.
        import os as _os

        # the epilogue/accumulate plan is the default, this one is opt-in (ALLEGRO_B200_PLAIN_BWD=1); both are covered
        # by the GPU tests.
        self.plain_ok = (_os.environ.get("ALLEGRO_B200_PLAIN_BWD", "0") == "1" and self.readout.is_two_layer_silu
                         and all(ly["mlp"].is_two_layer_silu for ly in self.layers))
        if self.plain_ok:
            L = self.L
            self.gxW, self.gxWp, self.gsW, self.gsWp = [], [], [], []
            for b in range(L + 1):
                blocks = [self.readout.WT[0][:, S * b : S * (b + 1)]]
                blocks += [self.layers[mm]["mlp"].WT[0][:, S * b : S * (b + 1)] for mm in range(L - 1, b - 1, -1) if mm >= b]
                Wg = torch.cat(blocks, dim=0).contiguous()
                self.gxW.append(Wg)
                self.gxWp.append(_lib.linear_pack(Wg))
            for l in range(L):
                Ws = self.layers[l]["mlp"].WT[0][:, S * (l + 1) : S * (l + 1) + U].contiguous()
                self.gsW.append(Ws)
                self.gsWp.append(_lib.linear_pack(Ws))

    # ------------------------------------------------------------------------------------
    def forward(self, csr: EdgeCSR, vec: torch.Tensor, x_emb: Optional[torch.Tensor], keep: bool = True, fill_embed=None):
        """vec [E,3] (acc dtype), x_emb [E,S_in] (act dtype), both in CSR edge order.
        Returns (Ei [N] acc dtype, X [E,S(L+1)], Ez [E,1], saved-for-backward).
        ``fill_embed(w0, x0, omega0)``: instead of x_emb, a callback that fills the three outputs of the embed GEMM
        (the upstream MLP with the embed linears folded into its last layer, energy_forces)."""
        E, N, U, S, L, D = csr.num_edges, csr.num_atoms, self.U, self.S, self.L, self.D
        dt, dev = self.dtype, self.device
        assert vec.dtype == self.acc and (fill_embed is not None or x_emb.dtype == dt)
        sv = _Saved()
        sv.fold = fill_embed is not None
        sv.csr, sv.vec = csr, vec
        _lib.set_tag("fwd.embed")
        Y = _lib.sh_fwd(vec, self.lmax)
        X = torch.empty(E, S * (L + 1), dtype=dt, device=dev)
        w0 = torch.empty(E, self.nw, dtype=dt, device=dev)
        omega = [torch.empty(E, self.nw, dtype=dt, device=dev)]
        if fill_embed is not None:
            fill_embed(w0, X[:, :S], omega[0])
        else:
            self.embed.forward([x_emb], [w0, X[:, :S], omega[0]])
        V: List[Optional[torch.Tensor]] = [None]
        gammas, pre_lat = [], []
        for l, ly in enumerate(self.layers):
            _lib.set_tag(f"fwd.L{l}")
            gamma = _lib.env_sum(dt, self.lmax, N, U, csr.row_ptr, Y, omega[l], self.sf)
            Vn = torch.empty(E, ly["d_out"], U, dtype=dt, device=dev)
            _lib.tp_fwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr, gamma,
                        V[l], Y, w0 if l == 0 else None, Vn)
            s = Vn.view(E, ly["d_out"] * U)[:, :U]  # scalar (k=0) slab, _allegro.py:272-275
            outs = [X[:, S * (l + 1) : S * (l + 2)]]
            if not ly["last"]:
                omega.append(torch.empty(E, self.nw, dtype=dt, device=dev))
                outs.append(omega[l + 1])
            pre_lat.append(ly["mlp"].forward([X[:, : S * (l + 1)], s], outs))
            V.append(Vn)
            gammas.append(gamma)
        _lib.set_tag("fwd.readout")
        Ez = torch.empty(E, 1, dtype=dt, device=dev)
        pre_read = self.readout.forward([X], [Ez])
        Ei = _lib.edge_sum(Ez.view(E).to(self.acc), csr.row_ptr, self.factor)
        sv.Y, sv.w0, sv.omega, sv.V, sv.gamma, sv.pre_lat, sv.pre_read, sv.X = Y, w0, omega, V, gammas, pre_lat, pre_read, X
        return Ei, X, Ez, sv

    # ------------------------------------------------------------------------------------
    def backward(self, sv: _Saved, gEi: torch.Tensor):
        """gEi [N] (acc dtype) -> (gvec [E,3] acc dtype, gx_emb [E,S_in] act dtype)."""
        if self.plain_ok:
            return self._backward_plain(sv, gEi)
        return self._backward_legacy(sv, gEi)

    def _backward_plain(self, sv: _Saved, gEi: torch.Tensor):
        csr = sv.csr
        E, N, U, S, L, D = csr.num_edges, csr.num_atoms, self.U, self.S, self.L, self.D
        dt, dev = self.dtype, self.device
        _lib.set_tag("bwd.readout")
        gEz = _lib.edge_sum_bwd(gEi.contiguous(), csr.ctr, self.factor).to(dt).view(E, 1)
        g_h = {"r": self.readout.hidden_grad([gEz])}
        pre = {"r": sv.pre_read[0]}
        for l in range(L):
            pre[l] = sv.pre_lat[l][0]
        gY = torch.zeros(E, D, dtype=self.acc, device=dev)
        gV_next: Optional[torch.Tensor] = None
        gomega_next: Optional[torch.Tensor] = None
        gw0 = None

        def block_grad(b: int) -> torch.Tensor:
            cons = ["r"] + [mm for mm in range(L - 1, b - 1, -1) if mm >= b]
            out = torch.empty(E, S, dtype=dt, device=dev)
            _lib.linear([g_h[c] for c in cons], self.gxW[b], [out], act=_lib.ACT_MUL_DSILU, a_aux=[pre[c] for c in cons],
                        W_packed=self.gxWp[b])
            return out

        for l in range(L - 1, -1, -1):
            ly = self.layers[l]
            _lib.set_tag(f"bwd.L{l}")
            gouts = [block_grad(l + 1)]
            if not ly["last"]:
                gouts.append(gomega_next)
            g_h[l] = ly["mlp"].hidden_grad(gouts)
            if ly["last"]:
                gV_next = torch.empty(E, ly["d_out"], U, dtype=dt, device=dev)
                if ly["d_out"] > 1:
                    gV_next.zero_()
                gs_acc = False
            else:
                gs_acc = True
            gs = gV_next.view(E, ly["d_out"] * U)[:, :U]
            _lib.linear([g_h[l]], self.gsW[l], [gs], o_accum=[gs_acc], act=_lib.ACT_MUL_DSILU, a_aux=[pre[l]], W_packed=self.gsWp[l])
            ggamma = torch.empty(N, D, U, dtype=self.acc, device=dev)
            if l == 0:
                gw0 = torch.empty(E, self.nw, dtype=dt, device=dev)
                _lib.tp_bwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr,
                            sv.gamma[l], None, sv.Y, sv.w0, gV_next, None, gw0, gY, ggamma)
                gV_in = None
            else:
                gV_in = torch.empty(E, ly["d_in"], U, dtype=dt, device=dev)
                _lib.tp_bwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr,
                            sv.gamma[l], sv.V[l], None, None, gV_next, gV_in, None, None, ggamma)
            gomega = torch.empty(E, self.nw, dtype=dt, device=dev)
            _lib.env_bwd(dt, self.lmax, U, csr.ctr, sv.Y, sv.omega[l], ggamma, self.sf, gomega, gY, row_ptr=csr.row_ptr)
            gV_next, gomega_next = gV_in, gomega
        _lib.set_tag("bwd.embed")
        g_x0 = block_grad(0)
        gvec = _lib.sh_bwd(sv.vec, gY, self.lmax)
        if sv.fold:  # the caller back-propagates the three embed-output gradients through its folded MLP
            return gvec, [gw0, g_x0, gomega_next]
        gx_emb = torch.empty(E, self.S_in, dtype=dt, device=dev)
        self.embed.backward([gw0, g_x0, gomega_next], [], [gx_emb], [False])
        return gvec, gx_emb

    def _backward_legacy(self, sv: _Saved, gEi: torch.Tensor):
        """General MLP depth / nonlinearity: SiLU' in the GEMM epilogue, gradient accumulation."""
        csr = sv.csr
        E, N, U, S, L, D = csr.num_edges, csr.num_atoms, self.U, self.S, self.L, self.D
        dt, dev = self.dtype, self.device
        _lib.set_tag("bwd.readout")
        gEz = _lib.edge_sum_bwd(gEi.contiguous(), csr.ctr, self.factor).to(dt).view(E, 1)
        gX = torch.empty(E, S * (L + 1), dtype=dt, device=dev)
        self.readout.backward([gEz], sv.pre_read, [gX], [False])
        gY = torch.zeros(E, D, dtype=self.acc, device=dev)
        gV_next: Optional[torch.Tensor] = None   # grad wrt V_{l+1}
        gomega_next: Optional[torch.Tensor] = None  # grad wrt omega_{l+1}
        gw0 = None
        for l in range(L - 1, -1, -1):
            ly = self.layers[l]
            _lib.set_tag(f"bwd.L{l}")
            if ly["last"]:
                gV_next = torch.empty(E, ly["d_out"], U, dtype=dt, device=dev)
                if ly["d_out"] > 1:
                    gV_next.zero_()
                gs_acc = False
            else:
                gs_acc = True
            gs = gV_next.view(E, ly["d_out"] * U)[:, :U]
            gouts = [gX[:, S * (l + 1) : S * (l + 2)]]
            if not ly["last"]:
                gouts.append(gomega_next)
            ly["mlp"].backward(gouts, sv.pre_lat[l], [gX[:, : S * (l + 1)], gs], [True, gs_acc])
            ggamma = torch.empty(N, D, U, dtype=self.acc, device=dev)
            if l == 0:
                gw0 = torch.empty(E, self.nw, dtype=dt, device=dev)
                _lib.tp_bwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr,
                            sv.gamma[l], None, sv.Y, sv.w0, gV_next, None, gw0, gY, ggamma)
                gV_in = None
            else:
                gV_in = torch.empty(E, ly["d_in"], U, dtype=dt, device=dev)
                _lib.tp_bwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr,
                            sv.gamma[l], sv.V[l], None, None, gV_next, gV_in, None, None, ggamma)
            gomega = torch.empty(E, self.nw, dtype=dt, device=dev)
            _lib.env_bwd(dt, self.lmax, U, csr.ctr, sv.Y, sv.omega[l], ggamma, self.sf, gomega, gY, row_ptr=csr.row_ptr)
            gV_next, gomega_next = gV_in, gomega
        _lib.set_tag("bwd.embed")
        gvec = _lib.sh_bwd(sv.vec, gY, self.lmax)
        if sv.fold:
            return gvec, [gw0, gX[:, :S], gomega_next]
        gx_emb = torch.empty(E, self.S_in, dtype=dt, device=dev)
        self.embed.backward([gw0, gX[:, :S], gomega_next], [], [gx_emb], [False])
        return gvec, gx_emb


class UpstreamPack:
    """Device constants of the two-body scalar embedding (edge_norm, radial_chemical_embed,
    scalar_embed_mlp) for ab2_radial_fwd/bwd + the packed scalar-embed MLP."""

    def __init__(self, edge_norm, radial, scalar_embed_mlp, dtype, device, fold_embed_of: Optional["AllegroCore"] = None):
        acc = _lib.ACC_DTYPE[dtype]
        # fold_embed_of: x_emb only feeds two LINEAR maps (tensorembed.py:88-89 env_embed_linear, _allegro.py:251
        # first_layer_env_embed_projection), and the scalar-embed MLP ends in a linear layer, so their product is
        # one matrix: [w0 | x_0 | omega_0] = silu(h) @ (W_last @ W_embed).  One GEMM and the x_emb round trip less
        # in each direction.  Default on; ALLEGRO_B200_FOLD_EMBED=0 switches it off.
        self.fold = fold_embed_of is not None
        self.mlp = PackedMLP(scalar_embed_mlp, dtype, device, post=fold_embed_of.embed.W64[0] if self.fold else None)
        self.dtype = dtype
        self.S_rc = radial.out_dim
        self.kind = "spline" if hasattr(radial, "spline") else "bessel"
        if self.kind == "spline":
            # spline embedding (scalarembed.py:84-175): torch ops in fp64 with a hand-written adjoint (nn/_spline.py)
            sp = radial.spline
            self.num_types = radial.num_types
            self.rmax64 = edge_norm.rmax_table.detach().to(device=device, dtype=torch.float64).contiguous()
            self.sp_lower = sp.lower.detach().to(device=device, dtype=torch.float64)
            self.sp_upper = sp.upper.detach().to(device=device, dtype=torch.float64)
            self.sp_const = float(sp._const)
            self.sp_w = sp.flat_weights().to(device=device, dtype=torch.float64)
            return
        te = radial.type_embed
        self.p = float(radial.bessel_encode.p)
        self.S_rc = radial.out_dim
        self.rmax_table = edge_norm.rmax_table.detach().to(device=device, dtype=acc).contiguous()
        self.bessel_w = radial.bessel_encode.bessel_weights.detach().reshape(-1).to(device=device, dtype=acc).contiguous()
        self.Wb = te.basis_linear.folded_weights()[0].to(device=device, dtype=acc).contiguous()
        self.cemb = te.center_embed.weight.detach().to(device=device, dtype=acc).contiguous()
        self.nemb = te.neighbor_embed.weight.detach().to(device=device, dtype=acc).contiguous()
        # Per-type-pair matrices for ab2_radial_pq_*: PQ0[t_c,t_n][n][c] = typeemb(t_c,t_n)[c] * Wb[n][c] (the product embedding,
        # _edgeembed.py:68-85).  Everything between the radial basis and the first SiLU is linear, so when the scalar-embed MLP
        # has exactly one hidden layer its first weight matrix is folded in as well,  PQ = PQ0 @ W_1 : the radial kernel then
        # emits the pre-activation h directly (no [E][S_rc] embedding tensor, one GEMM less per direction).
        self.PQ, self.S_pq, self.fold_radial = None, 0, False
        nb = int(self.bessel_w.numel())
        import os as _os

        if nb == 8 and _os.environ.get("ALLEGRO_B200_RADIAL_PQ", "1") == "1":
            Wb64 = te.basis_linear.folded_weights()[0].detach().double().cpu()             # [nb, S_rc]
            ce, ne = te.center_embed.weight.detach().double().cpu(), te.neighbor_embed.weight.detach().double().cpu()
            T = ce.shape[0]
            temb = torch.cat([ce.unsqueeze(1).expand(T, T, -1), ne.unsqueeze(0).expand(T, T, -1)], dim=-1)  # [tc, tn, S_rc]
            PQ0 = temb.reshape(T * T, 1, -1) * Wb64.unsqueeze(0)                          # [T*T, nb, S_rc]
            if self.mlp.is_two_layer_silu and self.mlp.dims[1] <= 128 and _os.environ.get("ALLEGRO_B200_FOLD_RADIAL", "1") == "1":
                self.fold_radial = True
                PQ0 = PQ0 @ self.mlp.W64[0]                                                # [T*T, nb, width]
            if PQ0.shape[-1] <= 128:
                self.PQ = PQ0.to(device=device, dtype=acc).contiguous()
                self.S_pq = int(PQ0.shape[-1])
            else:
                self.fold_radial = False

    # ---- forward / adjoint of the whole upstream scalar track -----------------------------------------------
    def forward(self, vec, csr: EdgeCSR, types_i32, outs):
        """vec [E,3] -> the scalar-embed MLP's outputs written into ``outs`` ([x_emb], or with the embed fold
        [w0, x_0, omega_0]).  Returns what ``backward`` needs."""
        dt = self.dtype
        if self.kind == "spline":
            from ._spline import spline_forward

            t64 = types_i32.long()
            e0, sp_saved = spline_forward(vec, t64[csr.ctr.long()], t64[csr.nbr.long()], self.rmax64, self.sp_lower, self.sp_upper, self.sp_const,
                                          self.sp_w, self.num_types, dt)
            return ("spline", sp_saved, self.mlp.forward([e0], outs))
        if self.fold_radial:
            h = _lib.radial_pq_fwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ)
            _lib.linear([h], self.mlp.W[1], outs, act=_lib.ACT_SILU, W_packed=self.mlp.Wp[1])
            return ("pq_fold", None, [h])
        if self.PQ is not None:
            e0 = _lib.radial_pq_fwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ)
        else:
            e0 = _lib.radial_fwd(dt, self.S_rc, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.Wb, self.cemb, self.nemb)
        return ("bessel", None, self.mlp.forward([e0], outs))

    def backward(self, saved, gouts, vec, csr: EdgeCSR, types_i32, gvec):
        """gouts = gradients w.r.t. ``outs``; accumulates d/d vec into gvec."""
        kind, sp_saved, pre = saved
        dt = self.dtype
        E = vec.shape[0]
        if kind == "pq_fold":
            g_h = self.mlp.hidden_grad(gouts)  # gradient w.r.t. silu(h); silu'(h) is applied by the radial adjoint (aux = h)
            _lib.radial_pq_bwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ, g_h, pre[0], gvec)
            return
        g_e0 = torch.empty(E, self.S_rc, dtype=dt, device=vec.device)
        if self.mlp.is_two_layer_silu:
            self.mlp.backward_plain(gouts, pre, [g_e0])
        else:
            self.mlp.backward(gouts, pre, [g_e0], [False])
        if kind == "spline":
            from ._spline import spline_backward

            gvec += spline_backward(sp_saved, g_e0, self.sp_w, self.num_types).to(gvec.dtype)
        elif self.PQ is not None:
            _lib.radial_pq_bwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ, g_e0, None, gvec)
        else:
            _lib.radial_bwd(dt, self.S_rc, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.Wb, self.cemb, self.nemb, g_e0, gvec)


def energy_forces(core: "AllegroCore", up: UpstreamPack, csr: EdgeCSR, pos: torch.Tensor, types_i32: torch.Tensor,
                  shift_vec: Optional[torch.Tensor], gEi_scale: Optional[torch.Tensor], want_virial: bool = False, pair=None):
    """Whole path with no torch autograd: positions -> (Ei [N], forces [n_atoms,3], X, Ez, virial).
    ``gEi_scale`` = d E_total / d Ei (per-type scales), None = ones.  ``virial`` (only if asked for) is
    sum_z r_z (x) dE/dr_z [3,3] = dE/d(strain) before symmetrisation, from the per-edge gradients the
    force scatter consumes anyway.  ``pair`` = (ZBL module, r_max table) adds the pair potential's gradient to the
    per-edge gradients and returns its per-atom energies as a sixth value (added AFTER the per-type scale/shift,
    allegro_models.py:270-288)."""
    dt, acc = core.dtype, core.acc
    E = csr.num_edges
    if E == 0:
        # a frame without a single edge (every atom isolated): zero energies before scale/shift, zero forces, empty
        # per-edge outputs -- what the reference's modules produce on empty edge tensors
        dev = pos.device
        return (torch.zeros(csr.num_atoms, dtype=acc, device=dev), torch.zeros(pos.shape[0], 3, dtype=acc, device=dev),
                torch.empty(0, core.S * (core.L + 1), dtype=dt, device=dev), torch.empty(0, 1, dtype=dt, device=dev),
                torch.zeros(3, 3, dtype=acc, device=dev) if want_virial else None,
                torch.zeros(csr.num_atoms, dtype=acc, device=dev) if pair is not None else None)
    _lib.set_tag("fwd.radial")
    vec = _lib.edge_vec(pos, csr.ctr, csr.nbr, shift_vec, acc)
    if up.fold:
        box = []
        Ei, X, Ez, sv = core.forward(csr, vec, None, fill_embed=lambda w0, x0, om0: box.append(up.forward(vec, csr, types_i32, [w0, x0, om0])))
        up_saved = box[0]
    else:
        x_emb = torch.empty(E, core.S_in, dtype=dt, device=pos.device)
        up_saved = up.forward(vec, csr, types_i32, [x_emb])
        Ei, X, Ez, sv = core.forward(csr, vec, x_emb)
    gEi = gEi_scale if gEi_scale is not None else torch.ones_like(Ei)
    gvec, gx_emb = core.backward(sv, gEi)
    _lib.set_tag("bwd.radial")
    up.backward(up_saved, gx_emb if up.fold else [gx_emb], vec, csr, types_i32, gvec)
    Ei_pair = None
    if pair is not None:
        Ez_pair = pair[0].edge_energy_and_grad(vec, csr, types_i32, pair[1], gvec)
        Ei_pair = _lib.edge_sum(Ez_pair, csr.row_ptr, 1.0)
    virial = (vec.T @ gvec.to(vec.dtype)) if want_virial else None
    F = _lib.force_scatter(gvec, csr, pos.shape[0])
    return Ei, F, X, Ez, virial, Ei_pair


class _CoreFn(torch.autograd.Function):
    """(vec, x_emb) -> per-atom energies; backward gives (d/dvec, d/dx_emb).  Weights are not
    differentiated (inference / MD path, like the reference's Triton back-end)."""

    @staticmethod
    def forward(ctx, vec, x_emb, core: AllegroCore, csr: EdgeCSR, stash: Dict):
        Ei, X, Ez, sv = core.forward(csr, vec.detach(), x_emb.detach())
        ctx.core, ctx.sv = core, sv
        stash["edge_features"], stash["edge_energy"] = X, Ez
        return Ei

    @staticmethod
    def backward(ctx, gEi):
        gvec, gx = ctx.core.backward(ctx.sv, gEi.to(ctx.core.acc))
        ctx.sv = None
        return gvec, gx, None, None, None


def core_apply(core: AllegroCore, csr: EdgeCSR, vec: torch.Tensor, x_emb: torch.Tensor, stash: Dict) -> torch.Tensor:
    return _CoreFn.apply(vec, x_emb, core, csr, stash)
