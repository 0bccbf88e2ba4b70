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
    __slots__ = ("csr", "vec", "Y", "w0", "omega", "V", "gamma", "pre_lat", "pre_read", "X", "fold", "chain")


_BAKED_TABLES = {}


def _baked_table(d_out: int) -> torch.Tensor:
    """(i, j, k) structure of the l_max = 2 coupling tables baked into the composed tensor-product kernels
    (Tab9x9x9 / Tab9x9x1 in csrc/tp_tables_generated.cuh, generated from the same Contracter)."""
    if d_out not in _BAKED_TABLES:
        from ._contract import Contracter

        ir = "1x0e+1x1o+1x2e"
        _BAKED_TABLES[d_out] = Contracter(ir, ir, ir if d_out == 9 else "1x0e", mul=1).sparse_table()[0].cpu()
    return _BAKED_TABLES[d_out]


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
        # the last latent MLP and the readout in one kernel per direction (ab2_mlp2_readout); the readout's first layer
        # is packed once more split by rows into the x_0..x_{L-1} block and the x_L block
        last = self.layers[-1]["mlp"]
        # (the kernel applies one nonlinearity to both MLPs, whose kwargs are independent in the reference: on a mismatch the
        # two MLPs run as two mlp2 calls)
        self.ro_fused = (last.is_two_layer_nonlinear and self.readout.is_two_layer_nonlinear and last.dims[1] == self.readout.dims[1]
                         and last.nonlinearity == self.readout.nonlinearity)
        if self.ro_fused:
            P = S * self.L
            W1r = self.readout.W[0]
            self.ro_fwd_p = [last.Wp[0], last.Wp[1], _lib.linear_pack(W1r[:P].contiguous()), _lib.linear_pack(W1r[P:].contiguous())]
            self.ro_bwd_p = [self.readout.WTp[0], last.WTp[1], last.WTp[0]]
        # the two tensor products composed per centre (ab2_tp_chain_*, DESIGN.md section 4.1): a two-layer l_max = 2
        # model whose tables have the baked structure, and (tp_chain_plan) fp32 with U = 32 or 64.
        # Then the forward keeps the compact scalars s_1, s_2 instead of V_1, and the backward passes the compact
        # gradients g1, g2 instead of gV_1.
        self.chain = None
        l0, l1 = (self.layers + [None, None])[:2]
        if (self.L == 2 and self.D == 9
                and (l0["d_in"], l0["d_out"], l1["d_in"], l1["d_out"]) == (9, 9, 9, 1)
                and torch.equal(l0["tab"].cpu(), _baked_table(9)) and torch.equal(l1["tab"].cpu(), _baked_table(1))):
            self.chain = _lib.tp_chain_plan(dtype, U, l0["cgw"], l1["cgw"])

    # ------------------------------------------------------------------------------------
    def forward(self, csr: EdgeCSR, vec: torch.Tensor, x_emb: Optional[torch.Tensor], keep: bool = True, fill_embed=None,
                stored_v: bool = False):
        """vec [E,3] (acc dtype), x_emb [E,S_in] (act dtype), both in CSR edge order.
        Returns (Ei [N] acc dtype, X [E,S(L+1)], Ez [E,1], saved-for-backward).
        ``fill_embed(w0, x0, omega0)``: instead of x_emb, a callback that fills the three outputs of the embed GEMM
        (the upstream MLP with the embed linears folded into its last layer, energy_forces).
        ``stored_v``: take the stored-V path even where the composed tensor products would run, so every V_l is kept
        (the tangent of nn._hessian reads them)."""
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
        Ez = torch.empty(E, 1, dtype=dt, device=dev)
        pre_read = None
        chain = None if stored_v else self.chain
        for l, ly in enumerate(self.layers):
            _lib.set_tag(f"fwd.L{l}")
            gamma = _lib.env_sum(dt, self.lmax, N, U, csr.row_ptr, Y, omega[l], self.sf)
            Vn = None
            if chain is not None:
                # composed path: s_1 = V_1[:, 0] from gamma_0, then s_2 from gamma_0 and gamma_1; V_1 is not formed
                s = torch.empty(E, U, dtype=dt, device=dev)
                if not _lib.tp_chain_fwd(chain, ly["last"], csr.row_ptr, csr.ctr, gammas[0] if l else gamma, gamma if l else None, Y, w0, s):
                    if l:
                        raise RuntimeError("tp_chain_fwd declined the last layer after taking the first")
                    chain = None  # declined (e.g. no edges): this call takes the stored-V path throughout
            if chain is None:
                Vn = torch.empty(E, ly["d_out"], U, dtype=dt, device=dev)
                _lib.tp_fwd(dt, self.lmax, N, E, U, ly["d_in"], ly["d_out"], ly["tab"], ly["cgw"], csr.row_ptr, csr.ctr, gamma,
                            V[l], Y, w0 if l == 0 else None, Vn)
                s = Vn.view(E, ly["d_out"] * U)[:, :U]  # scalar (k=0) slab, _allegro.py:272-275
            outs = [X[:, S * (l + 1) : S * (l + 2)]]
            if not ly["last"]:
                omega.append(torch.empty(E, self.nw, dtype=dt, device=dev))
                outs.append(omega[l + 1])
            if ly["last"] and self.ro_fused:
                P = S * L
                pre_l = torch.empty(E, ly["mlp"].dims[1], dtype=dt, device=dev)
                pre_r = torch.empty(E, self.readout.dims[1], dtype=dt, device=dev)
                if _lib.mlp2_readout(False, X[:, :P], s, X[:, P:], pre_l, pre_r, Ez, self.readout.W[1], self.ro_fwd_p, S, **self.readout.nl_kw):
                    pre_lat.append([pre_l])
                    pre_read = [pre_r]
            if pre_read is None:
                pre_lat.append(ly["mlp"].forward([X[:, : S * (l + 1)], s], outs))
            V.append(Vn)
            gammas.append(gamma)
        if pre_read is None:
            _lib.set_tag("fwd.readout")
            pre_read = self.readout.forward([X], [Ez])
        Ei = _lib.edge_sum(Ez.view(E).to(self.acc), csr.row_ptr, self.factor)
        sv.Y, sv.w0, sv.omega, sv.V, sv.gamma, sv.pre_lat, sv.pre_read, sv.X = Y, w0, omega, V, gammas, pre_lat, pre_read, X
        sv.chain = chain
        return Ei, X, Ez, sv

    # ------------------------------------------------------------------------------------
    def backward(self, sv: _Saved, gEi: torch.Tensor):
        """gEi [N] (acc dtype) -> (gvec [E,3] acc dtype, gx_emb [E,S_in] act dtype), or, when the forward ran with
        ``fill_embed``, (gvec, [gw0, gx_0, gomega_0]): the gradients of the three embed outputs.  phi' is applied in the
        GEMM epilogues, and the gradients of shared inputs are accumulated."""
        csr = sv.csr
        E, N, U, S, L, D = csr.num_edges, csr.num_atoms, self.U, self.S, self.L, self.D
        dt, dev = self.dtype, self.device
        _lib.set_tag("bwd.readout")
        gEz = _lib.edge_sum_bwd(gEi.contiguous(), csr.ctr, self.factor).to(dt).view(E, 1)
        gX = torch.empty(E, S * (L + 1), dtype=dt, device=dev)
        last = self.layers[-1]
        gV_last = torch.empty(E, last["d_out"], U, dtype=dt, device=dev)
        if last["d_out"] > 1:
            gV_last.zero_()
        # readout and last latent MLP in one kernel: gX[:, :S L] and gs of the last layer (gX[:, S L:] is not formed)
        fused = self.ro_fused and _lib.mlp2_readout(True, gX[:, : S * L], gV_last.view(E, -1)[:, :U], None, sv.pre_lat[-1][0],
                                                     sv.pre_read[0], gEz, self.readout.W[1], self.ro_bwd_p, S, **self.readout.nl_kw)
        if not fused:
            self.readout.backward([gEz], sv.pre_read, [gX], [False])
        gY = torch.zeros(E, D, dtype=self.acc, device=dev)
        gV_next: Optional[torch.Tensor] = None   # grad wrt V_{l+1}
        gomega_next: Optional[torch.Tensor] = None  # grad wrt omega_{l+1}
        gw0 = None
        chain = sv.chain
        g1 = None  # composed path: d/ds_1 [E][U]; d/ds_2 is gV_last
        for l in range(L - 1, -1, -1):
            ly = self.layers[l]
            _lib.set_tag(f"bwd.L{l}")
            if ly["last"]:
                gV_next = gV_last
                gs_acc = False
            else:
                gs_acc = True
            if chain is not None and not ly["last"]:
                g1 = torch.empty(E, U, dtype=dt, device=dev)
                gs, gs_acc = g1, False
            else:
                gs = gV_next.view(E, ly["d_out"] * U)[:, :U]
            gouts = [gX[:, S * (l + 1) : S * (l + 2)]]
            if not ly["last"]:
                gouts.append(gomega_next)
            if not (ly["last"] and fused):
                ly["mlp"].backward(gouts, sv.pre_lat[l], [gX[:, : S * (l + 1)], gs], [True, gs_acc])
            ggamma = torch.empty(N, D, U, dtype=self.acc, device=dev)
            if chain is not None:
                # last layer: gamma_1's gradient from g2; first layer: gw0, gY and gamma_0's gradient from g1 and g2
                if l == 0:
                    gw0 = torch.empty(E, self.nw, dtype=dt, device=dev)
                ok = _lib.tp_chain_bwd(chain, l == 0, csr.row_ptr, csr.ctr, sv.gamma[0], sv.gamma[1] if l == 0 else None, sv.Y, sv.w0, g1,
                                       gV_last.view(E, U), gw0, gY if l == 0 else None, ggamma)
                if not ok:
                    raise RuntimeError("tp_chain_bwd declined a case its forward took")
                gV_in = None
            elif l == 0:
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

    def __init__(self, edge_norm, radial, scalar_embed_mlp, dtype, device, core: "AllegroCore"):
        acc = _lib.ACC_DTYPE[dtype]
        # x_emb only feeds two LINEAR maps of the core (tensorembed.py:88-89 env_embed_linear, _allegro.py:251
        # first_layer_env_embed_projection), and the scalar-embed MLP ends in a linear layer, so their product is
        # one matrix: [w0 | x_0 | omega_0] = silu(h) @ (W_last @ W_embed).  One GEMM and the x_emb round trip less
        # in each direction.
        self.mlp = PackedMLP(scalar_embed_mlp, dtype, device, post=core.embed.W64[0])
        self.dtype = dtype
        # route of the last pq_fold backward: "fused" (ab2_radial_pq_bwd_gemm) or "two_launch" (hidden_grad + radial_pq_bwd)
        self.bwd_path: Optional[str] = None
        # route of the last pq_fold forward: "fused" (ab2_radial_embed_fwd) or "two_launch" (radial_pq_fwd + linear)
        self.fwd_path: Optional[str] = None
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
        if nb == 8:
            Wb64 = te.basis_linear.folded_weights()[0].detach().double().cpu()             # [nb, S_rc]
            ce, ne = te.center_embed.weight.detach().double().cpu(), te.neighbor_embed.weight.detach().double().cpu()
            T = ce.shape[0]
            temb = torch.cat([ce.unsqueeze(1).expand(T, T, -1), ne.unsqueeze(0).expand(T, T, -1)], dim=-1)  # [tc, tn, S_rc]
            PQ0 = temb.reshape(T * T, 1, -1) * Wb64.unsqueeze(0)                          # [T*T, nb, S_rc]
            if self.mlp.is_two_layer_nonlinear and self.mlp.dims[1] <= 128:
                self.fold_radial = True
                PQ0 = PQ0 @ self.mlp.W64[0]                                                # [T*T, nb, width]
            if PQ0.shape[-1] <= 128:
                self.PQ = PQ0.to(device=device, dtype=acc).contiguous()
                self.S_pq = int(PQ0.shape[-1])
            else:
                self.fold_radial = False

    # ---- forward / adjoint of the whole upstream scalar track -----------------------------------------------
    def forward(self, vec, csr: EdgeCSR, types_i32, outs, keep_h: bool = False):
        """vec [E,3] -> the scalar-embed MLP's outputs, with the embed linears folded in, written into ``outs``
        ([w0, x_0, omega_0]).  Returns what ``backward`` needs.  With the first layer folded into PQ, the hidden
        pre-activation h is stored only if ``keep_h``: the fused forward does not form it, and saves a meta tensor of its
        shape in its place (``backward`` recomputes h where it needs it)."""
        dt = self.dtype
        if self.kind == "spline":
            from ._spline import spline_forward

            t64 = types_i32.long()
            e0, sp_saved = spline_forward(vec, t64[csr.ctr.long()], t64[csr.nbr.long()], self.rmax64, self.sp_lower, self.sp_upper, self.sp_const,
                                          self.sp_w, self.num_types, dt)
            return ("spline", sp_saved, self.mlp.forward([e0], outs))
        if self.fold_radial:
            # One kernel where it takes the case: the radial basis and h formed in the GEMM's producers, all output columns
            # from one on-chip tile; bitwise the two launches below, which run where the entry declines.
            if not keep_h and self.mlp.Wp[1] is not None and _lib.radial_embed_fwd(
                    dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ, self.mlp.Wp[1], outs,
                    **self.mlp.nl_kw):
                self.fwd_path = "fused"
                return ("pq_fold", None, [torch.empty(vec.shape[0], self.S_pq, dtype=dt, device="meta")])
            self.fwd_path = "two_launch"
            h = _lib.radial_pq_fwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ)
            _lib.linear([h], self.mlp.W[1], outs, act=_lib.ACT_SILU, W_packed=self.mlp.Wp[1], **self.mlp.nl_kw)
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
            # One kernel where it takes the case: the hidden-gradient GEMM with the radial adjoint as its epilogue, so g_h
            # and h never reach memory.  fp32 storage, hidden width 32 or 64, a packed W2^T image; the entry itself declines
            # the rest (segment layout, PQ beyond the shared-memory budget), and then the two launches below run.
            if dt == torch.float32 and self.S_pq in (32, 64) and self.mlp.WTp[1] is not None and _lib.radial_pq_bwd(
                    dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ, None, pre[0], gvec,
                    gemm=(gouts, self.mlp.WTp[1]), **self.mlp.nl_kw):
                self.bwd_path = "fused"
                return
            self.bwd_path = "two_launch"
            h = pre[0]
            if h.is_meta:  # the fused forward did not store h
                h = _lib.radial_pq_fwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ)
            g_h = self.mlp.hidden_grad(gouts)  # gradient w.r.t. phi(h); phi'(h) is applied by the radial adjoint (aux = h)
            _lib.radial_pq_bwd(dt, self.S_pq, self.p, vec, csr.ctr, csr.nbr, types_i32, self.rmax_table, self.bessel_w, self.PQ, g_h, h, gvec,
                               **self.mlp.nl_kw)
            return
        g_e0 = torch.empty(E, self.S_rc, dtype=dt, device=vec.device)
        if self.mlp.is_two_layer_nonlinear:
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


def edge_energy_grad(core: "AllegroCore", up: UpstreamPack, csr: EdgeCSR, vec: torch.Tensor, types_i32: torch.Tensor,
                     gEi_scale: Optional[torch.Tensor], pair=None):
    """The per-edge part of ``energy_forces``: edge vectors ``vec`` [E,3] (acc dtype, CSR order, E > 0) -> (Ei [n_centres],
    X, Ez, gvec [E,3] = d E_total / d vec (acc dtype), Ei_pair or None).  ``types_i32`` is indexed by both ``csr.ctr`` and
    ``csr.nbr``; ``gEi_scale`` and ``pair`` as in ``energy_forces``.  Positions never enter: the caller may hand in edge
    vectors of any geometry (phonons.force_constants passes displaced copies of the rows of a cluster)."""
    box = []
    Ei, X, Ez, sv = core.forward(csr, vec, None, fill_embed=lambda w0, x0, om0: box.append(up.forward(vec, csr, types_i32, [w0, x0, om0])))
    gEi = gEi_scale if gEi_scale is not None else torch.ones_like(Ei)
    gvec, g_emb = core.backward(sv, gEi)
    _lib.set_tag("bwd.radial")
    up.backward(box[0], g_emb, vec, csr, types_i32, gvec)
    Ei_pair = None
    if pair is not None:
        Ez_pair = pair[0].edge_energy_and_grad(vec, csr, types_i32, pair[1], gvec)
        Ei_pair = _lib.edge_sum(Ez_pair, csr.row_ptr, 1.0)
    return Ei, X, Ez, gvec, Ei_pair


def energy_forces(core: "AllegroCore", up: UpstreamPack, csr: EdgeCSR, pos: torch.Tensor, types_i32: torch.Tensor,
                  shift_vec: Optional[torch.Tensor], gEi_scale: Optional[torch.Tensor], want_virial: bool = False, pair=None,
                  frame_ptr: Optional[torch.Tensor] = None, want_atomic_virial: bool = False):
    """Whole path with no torch autograd: positions -> (Ei [N], forces [n_atoms,3], X, Ez, virial, Ei_pair, W).
    ``gEi_scale`` = d E_total / d Ei (per-type scales), None = ones.  ``virial`` (only if asked for) is
    sum_z r_z (x) dE/dr_z [3,3] = dE/d(strain) before symmetrisation, from the per-edge gradients the
    force scatter consumes anyway.  ``pair`` = (ZBL module, r_max table) adds the pair potential's gradient to the
    per-edge gradients and returns its per-atom energies as a sixth value (added AFTER the per-type scale/shift,
    allegro_models.py:270-288).  ``frame_ptr`` [B+1] int32 (a batch of frames concatenated into one graph): the virial is
    then per frame, [B,3,3] (ab2_frame_virial).  ``want_atomic_virial``: W (the seventh value, else None) is the centroid
    per-atom virial [n_atoms,3,3], W[a] = -sum_{z: nbr[z] = a} r_z (x) dE/dr_z, formed by the force scatter itself
    (ab2_force_virial_scatter)."""
    dt, acc = core.dtype, core.acc
    vshape = (3, 3) if frame_ptr is None else (frame_ptr.shape[0] - 1, 3, 3)
    E = csr.num_edges
    if E == 0:
        # a frame without a single edge (every atom isolated): zero energies before scale/shift, zero forces, empty
        # per-edge outputs -- what the reference's modules produce on empty edge tensors
        dev = pos.device
        return (torch.zeros(csr.num_atoms, dtype=acc, device=dev), torch.zeros(pos.shape[0], 3, dtype=acc, device=dev),
                torch.empty(0, core.S * (core.L + 1), dtype=dt, device=dev), torch.empty(0, 1, dtype=dt, device=dev),
                torch.zeros(vshape, dtype=acc, device=dev) if want_virial else None,
                torch.zeros(csr.num_atoms, dtype=acc, device=dev) if pair is not None else None,
                torch.zeros(pos.shape[0], 3, 3, dtype=acc, device=dev) if want_atomic_virial else None)
    _lib.set_tag("fwd.radial")
    vec = _lib.edge_vec(pos, csr.ctr, csr.nbr, shift_vec, acc)
    Ei, X, Ez, gvec, Ei_pair = edge_energy_grad(core, up, csr, vec, types_i32, gEi_scale, pair)
    virial = None
    if want_virial:
        virial = (vec.T @ gvec.to(vec.dtype)) if frame_ptr is None else _lib.frame_virial(vec, gvec.to(vec.dtype), frame_ptr, csr.row_ptr)
    W = None
    if want_atomic_virial:
        F, W = _lib.force_virial_scatter(vec, gvec, csr, pos.shape[0])
    else:
        F = _lib.force_scatter(gvec, csr, pos.shape[0])
    return Ei, F, X, Ez, virial, Ei_pair, W


class _CoreFn(torch.autograd.Function):
    """(vec, x_emb) -> per-atom energies; backward gives (d/dvec, d/dx_emb).  Weights are not
    differentiated (inference / MD path, like the reference's Triton back-end)."""

    @staticmethod
    def forward(ctx, vec, x_emb, core: AllegroCore, csr: EdgeCSR, stash: Dict):
        if csr.num_edges == 0:
            # no edge at all: zero energies and empty per-edge outputs, as energy_forces gives (the kernels take no
            # empty inputs)
            ctx.core, ctx.sv, ctx.empty = core, None, (vec.shape, vec.dtype, x_emb.shape, x_emb.dtype, vec.device)
            stash["edge_features"] = torch.empty(0, core.S * (core.L + 1), dtype=core.dtype, device=vec.device)
            stash["edge_energy"] = torch.empty(0, 1, dtype=core.dtype, device=vec.device)
            return torch.zeros(csr.num_atoms, dtype=core.acc, device=vec.device)
        Ei, X, Ez, sv = core.forward(csr, vec.detach(), x_emb.detach())
        ctx.core, ctx.sv = core, sv
        stash["edge_features"], stash["edge_energy"] = X, Ez
        return Ei

    @staticmethod
    def backward(ctx, gEi):
        if ctx.sv is None:  # no edge: zero gradients of the empty vec and x_emb
            vs, vd, xs, xd, dev = ctx.empty
            return torch.zeros(vs, dtype=vd, device=dev), torch.zeros(xs, dtype=xd, device=dev), None, None, None
        gvec, gx = ctx.core.backward(ctx.sv, gEi.to(ctx.core.acc))
        ctx.sv = None
        return gvec, gx, None, None, None


def core_apply(core: AllegroCore, csr: EdgeCSR, vec: torch.Tensor, x_emb: torch.Tensor, stash: Dict) -> torch.Tensor:
    return _CoreFn.apply(vec, x_emb, core, csr, stash)
