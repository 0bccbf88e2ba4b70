"""Contracter: the reference's kernel plug-in point, backed by the sm_90a operator kernels.

Mirrors allegro/nn/_strided/_contract.py:11-313 -- same constructor kwargs, same
``state_dict`` (``weights`` of shape (mul,P)/(mul,)/(P,)/(), dense ``w3j`` buffer), same
``forward(x1, x2, idxs, scatter_dim_size)`` on the strided [z][u][i] layout -- but the
arithmetic runs in ``liballegro_b200.so`` (ab2_op_scatter_env / ab2_op_contract /
ab2_op_gather_rows / ab2_op_contract_wgrad).  Every derivative of the underlying trilinear form is one of four
hand-written products (_Tri), so the operator has gradients w.r.t. x1, x2 AND the weights and is differentiable to
any order (forces in the loss) -- the reference gets that from autograd through its einsum path; its Triton back-end
is inference-only (_flashallegro.py:583-666,727).
There is no CPU path: tensors must be CUDA tensors.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch

from .. import _lib
from ..o3 import CouplingTable, Irreps, build_coupling_table


class _Meta:
    """Non-differentiable context of one contraction: shapes, table, scatter indices."""

    __slots__ = ("U", "d1", "d2", "dout", "tab", "idxs", "n_atoms", "csr", "lmax")

    def __init__(self, U, d1, d2, dout, tab, idxs, n_atoms, csr=None, lmax=-1):
        self.U, self.d1, self.d2, self.dout, self.tab, self.idxs, self.n_atoms = U, d1, d2, dout, tab, idxs, n_atoms
        # centre-sorted indices + a full spherical-harmonic second operand: the products can run on the fused pipeline's
        # tensor-product kernels (component-major layout, CSR rows) instead of the generic operator kernels
        self.csr, self.lmax = csr, lmax


def _fast_product(which: str, m: _Meta, c, a, b, g):
    """One of the products "g" / "a" / "b" of _Tri on the fused pipeline's kernels (ab2_tp_fwd / ab2_tp_bwd): the operands
    are transposed to the component-major layout, the kernels see the CSR of the sorted indices.  The backward kernel
    produces both input gradients at once; the one that is not asked for is computed against a zero operand and dropped."""
    csr, dt = m.csr, (a if a is not None else g).dtype
    E, N, U = csr.num_edges, m.n_atoms, m.U
    dev = (a if a is not None else g).device
    c = c.contiguous()
    if which == "g":
        Vi, gi = _lib.transpose_ui(a, True), _lib.transpose_ui(b, True)
        out = torch.empty(E, m.dout, U, dtype=dt, device=dev)
        _lib.tp_fwd(dt, m.lmax, N, E, U, m.d1, m.dout, m.tab, c, csr.row_ptr, csr.ctr, gi, Vi, None, None, out)
        return _lib.transpose_ui(out, False)
    go = _lib.transpose_ui(g, True)
    Vi = _lib.transpose_ui(a, True) if a is not None else torch.zeros(E, m.d1, U, dtype=dt, device=dev)
    gi = _lib.transpose_ui(b, True) if b is not None else torch.zeros(N, m.d2, U, dtype=dt, device=dev)
    gVin = torch.empty(E, m.d1, U, dtype=dt, device=dev)
    ggam = torch.empty(N, m.d2, U, dtype=dt, device=dev)
    _lib.tp_bwd(dt, m.lmax, N, E, U, m.d1, m.dout, m.tab, c, csr.row_ptr, csr.ctr, gi, Vi, None, None, go, gVin, None, None, ggam)
    return _lib.transpose_ui(gVin if which == "a" else ggam, False)


_SLOTS = ("c", "a", "b", "g")


class _Tri(torch.autograd.Function):
    """One partial derivative of the trilinear form behind Contracter._contract (_contract.py:213-251)

        T(c, a, b, g) = sum_{z,u,n} c[n,u] a[z,u,i_n] b[idxs[z],u,j_n] g[z,u,k_n]

    with c = value * weights (the reference's ww3j), a = x1, b = the per-atom environment, g = a cotangent of the
    output.  ``which`` names the slot that is differentiated away: "g" is the forward contraction, "a" / "b" the two
    backward products of the Triton back-end (_flashallegro.py:347-360), "c" the weight gradient.  T is linear in every
    slot, so the gradient of any of these products w.r.t. one of its inputs is again one of the four products with the
    incoming cotangent put into the differentiated slot -- backward() therefore calls _Tri.apply itself, which makes the
    operator differentiable to any order (weight gradients, and double backward for forces in the loss) on four kernels."""

    @staticmethod
    def forward(ctx, which: str, meta: _Meta, c, a, b, g):
        ctx.which, ctx.meta = which, meta
        ctx.save_for_backward(*[t for t in (c, a, b, g) if t is not None])
        m = meta
        if m.csr is not None and which != "c":
            return _fast_product(which, m, c, a, b, g)
        if which == "g":
            out = torch.empty(a.shape[0], m.U, m.dout, dtype=a.dtype, device=a.device)
            return _lib.op_contract(0, m.U, m.d1, m.d2, m.dout, m.tab, c.contiguous(), a, b, m.idxs, out)
        if which == "a":
            out = torch.empty(g.shape[0], m.U, m.d1, dtype=g.dtype, device=g.device)
            return _lib.op_contract(1, m.U, m.d1, m.d2, m.dout, m.tab, c.contiguous(), g, b, m.idxs, out)
        if which == "b":
            out = torch.zeros(m.n_atoms, m.U, m.d2, dtype=a.dtype, device=a.device)
            return _lib.op_contract(2, m.U, m.d1, m.d2, m.dout, m.tab, c.contiguous(), a, g, m.idxs, out)
        return _lib.op_contract_wgrad(m.U, m.d1, m.d2, m.dout, m.tab, a, b, g, m.idxs)

    @staticmethod
    def backward(ctx, h):
        saved = list(ctx.saved_tensors)
        slots = {}
        for name in _SLOTS:
            slots[name] = h.contiguous() if name == ctx.which else saved.pop(0)
        grads = []
        for pos, name in enumerate(_SLOTS):
            if name == ctx.which or not ctx.needs_input_grad[2 + pos]:
                grads.append(None)
                continue
            args = dict(slots)
            args[name] = None
            grads.append(_Tri.apply(name, ctx.meta, args["c"], args["a"], args["b"], args["g"]))
        return (None, None, *grads)


class _ScatterRows(torch.autograd.Function):
    """gamma[n] = sf * sum_{z: idxs[z] = n} x[z]  (_contract.py:199-204); its adjoint is _GatherRows and vice versa."""

    @staticmethod
    def forward(ctx, x, idxs, n_atoms: int, sf: float):
        ctx.idxs, ctx.n_atoms, ctx.sf = idxs, n_atoms, sf
        return _lib.op_scatter_env(x.contiguous(), idxs, n_atoms, sf)

    @staticmethod
    def backward(ctx, h):
        return _GatherRows.apply(h, ctx.idxs, ctx.n_atoms, ctx.sf), None, None, None


class _GatherRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, idxs, n_atoms: int, sf: float):
        ctx.idxs, ctx.n_atoms, ctx.sf = idxs, n_atoms, sf
        return _lib.op_gather_rows(src.contiguous(), idxs, sf)

    @staticmethod
    def backward(ctx, h):
        return _ScatterRows.apply(h, ctx.idxs, ctx.n_atoms, ctx.sf), None, None, None


class Contracter(torch.nn.Module):
    def __init__(
        self,
        irreps_in1,
        irreps_in2,
        irreps_out,
        mul: int,
        instructions: Optional[List[Tuple[int, int, int]]] = None,
        path_channel_coupling: bool = True,
        scatter_factor: Optional[float] = None,
        irrep_normalization: Optional[str] = "component",
    ):
        super().__init__()
        assert mul > 0
        self.scatter_factor = scatter_factor
        self.instructions = instructions
        self.irreps_in1, self.irreps_in2, self.irreps_out = Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out)
        self.table: CouplingTable = build_coupling_table(
            self.irreps_in1, self.irreps_in2, self.irreps_out, instructions, irrep_normalization
        )
        self.irrep_normalization = irrep_normalization
        self.mul = mul
        self.base_dim1, self.base_dim2, self.base_dim_out = self.table.dim1, self.table.dim2, self.table.dim_out
        self.num_paths = self.table.num_paths
        self.w3j_is_ij_diagonal = self.table.is_ij_diagonal
        self.path_channel_coupling = path_channel_coupling
        # dense w3j buffer exactly as the reference registers it (_contract.py:135-168)
        if self.w3j_is_ij_diagonal:
            w3j = torch.zeros(self.num_paths, self.base_dim1, self.base_dim_out)
            for i, j, k, p, v in self.table.entries:
                w3j[p, i, k] = v
        else:
            w3j = torch.zeros(self.num_paths, self.base_dim1, self.base_dim2, self.base_dim_out)
            for i, j, k, p, v in self.table.entries:
                w3j[p, i, j, k] = v
        if self.num_paths == 1:
            w3j = w3j.squeeze(0)
        self.register_buffer("w3j", w3j)
        shape = (mul,) if path_channel_coupling else tuple()
        if self.num_paths > 1:
            shape = shape + (self.num_paths,)
        self.weights = torch.nn.Parameter(torch.empty(shape).uniform_(-math.sqrt(3), math.sqrt(3)))
        self._tab_cache = {}

    # ---- tables for the kernels --------------------------------------------------------
    def w3j_entries(self):
        """Non-zeros of the REGISTERED ``w3j`` buffer as (i, j, k, path, value) -- the buffer is state
        (_contract.py:168), so after ``load_state_dict`` of a reference / real-e3nn checkpoint the kernels
        contract with the checkpoint's coupling tensor (its block signs and normalisation), not with the
        table this class generated at construction.  The layouts are the reference's: [P,]i,j,k or, when
        every path is i==j diagonal, [P,]i,k (_contract.py:135-167)."""
        w = self.w3j.detach().to(device="cpu", dtype=torch.float64)
        if self.num_paths == 1:
            w = w.unsqueeze(0)
        nz = w.nonzero()
        vals = w[tuple(nz.T)]
        if self.w3j_is_ij_diagonal:
            return [(int(i), int(i), int(k), int(p), float(v)) for (p, i, k), v in zip(nz.tolist(), vals.tolist())]
        return [(int(i), int(j), int(k), int(p), float(v)) for (p, i, j, k), v in zip(nz.tolist(), vals.tolist())]

    def sparse_table(self):
        """(ijk int32 [nnz,3], path int64 [nnz], value fp64 [nnz]) on the CPU, from the ``w3j`` buffer."""
        key = (self.w3j._version, self.w3j.data_ptr())
        hit = self._tab_cache.get("sparse")
        if hit is not None and hit[0] == key:
            return hit[1]
        # sorted by output target (i, k), then j: the fast kernels gather each M[i][k] entry from a
        # contiguous table segment (include/allegro_b200.h, ab2_tp_fwd)
        e = sorted(self.w3j_entries(), key=lambda a: (a[0], a[2], a[1], a[3]))
        ijk = torch.tensor([[a[0], a[1], a[2]] for a in e], dtype=torch.int32).reshape(-1, 3)
        path = torch.tensor([a[3] for a in e], dtype=torch.long)
        val = torch.tensor([a[4] for a in e], dtype=torch.float64)
        self._tab_cache["sparse"] = (key, (ijk, path, val))
        return ijk, path, val

    def cgw(self, dtype: torch.dtype, device) -> torch.Tensor:
        """cgw[nnz][u] = value[nnz] * weights[u, path[nnz]] (the reference's ww3j, _contract.py:218-219)."""
        _, path, val = self.sparse_table()
        w = self.weights.detach().to(device="cpu", dtype=torch.float64)
        if self.num_paths > 1:
            wp = w[..., path]  # (mul, nnz) or (nnz,)
        else:
            wp = w.unsqueeze(-1).expand(*w.shape, path.shape[0])
        if self.path_channel_coupling:
            out = (wp * val).T  # (nnz, mul)
        else:
            out = (wp * val).unsqueeze(-1).expand(path.shape[0], self.mul)
        return out.contiguous().to(device=device, dtype=dtype)

    def cgw_live(self, dtype, device) -> torch.Tensor:
        """cgw as a differentiable function of ``self.weights`` (training): same values as ``cgw``."""
        _, path, val = self.sparse_table()
        path, val = path.to(device), val.to(device=device, dtype=dtype)
        w = self.weights.to(device=device, dtype=dtype)
        if self.num_paths > 1:
            wp = w[..., path]
        else:
            wp = w.unsqueeze(-1).expand(*w.shape, path.shape[0])
        if self.path_channel_coupling:
            return (wp * val).transpose(0, 1).contiguous()
        return (wp * val).unsqueeze(-1).expand(path.shape[0], self.mul).contiguous()

    def device_tables(self, dtype, device):
        key = (dtype, str(device), self.weights._version, self.weights.data_ptr(), self.w3j._version, self.w3j.data_ptr())
        hit = self._tab_cache.get("k")
        if hit is None or hit[0] != key:
            ijk, _, _ = self.sparse_table()
            hit = (key, ijk.to(device), self.cgw(dtype, device))
            self._tab_cache["k"] = hit
        return hit[1], hit[2]

    # ---- the operator -------------------------------------------------------------------
    def forward(self, x1: torch.Tensor, x2: torch.Tensor, idxs: torch.Tensor, scatter_dim_size) -> torch.Tensor:
        if not x1.is_cuda:
            raise RuntimeError("allegro_b200.nn.Contracter has no CPU path (B200 kernels only)")
        if x1.dtype not in (torch.float32, torch.float64):
            raise RuntimeError("operator-level Contracter supports float32/float64")
        n = int(scatter_dim_size.reshape(-1)[0]) if isinstance(scatter_dim_size, torch.Tensor) else int(scatter_dim_size)
        return self._forward_impl(x1, x2, idxs, n)

    def _forward_impl(self, x1: torch.Tensor, x2: torch.Tensor, idxs: torch.Tensor, n: int) -> torch.Tensor:
        U, d1, d2, dout = self.mul, self.base_dim1, self.base_dim2, self.base_dim_out
        idxs, checked = self._checked_indices(x1, x2, idxs, n)
        tab, cgw = self.device_tables(x1.dtype, x1.device)
        if torch.is_grad_enabled() and self.weights.requires_grad:
            cgw = self.cgw_live(x1.dtype, x1.device)
        sf = 1.0 if self.scatter_factor is None else float(self.scatter_factor)
        gamma = _ScatterRows.apply(x2.to(x1.dtype).reshape(-1, U, d2), idxs, n, sf)
        csr, lmax = self._fast_route(checked, n, d2)
        return _Tri.apply("g", _Meta(U, d1, d2, dout, tab, idxs, n, csr, lmax), cgw, x1.reshape(-1, U, d1).contiguous(), gamma, None)

    def _checked_indices(self, x1: torch.Tensor, x2: torch.Tensor, idxs: torch.Tensor, n: int):
        """(idxs as a contiguous int64 tensor, the cached check of this index tensor or None).

        x1 and x2 must hold one row of mul * dim values per entry of the 1-D ``idxs``; other integer index types are
        converted to int64, as torch's index ops accept them.  Every index must lie in [0, n): the kernels scatter into
        and gather from n rows of the environment sum without a bounds test.  That check and the sortedness test of
        ``_fast_route`` are one reduction with one host synchronisation, made once per index tensor (cached on the
        tensor object, its version and n).  While a CUDA graph is being captured no synchronisation is possible: an
        index tensor not checked before the capture is then used unchecked, and takes the generic route."""
        if idxs.dim() != 1:
            raise ValueError(f"Contracter: idxs must be 1-D (got shape {tuple(idxs.shape)})")
        if idxs.dtype == torch.bool or idxs.is_floating_point() or idxs.is_complex():
            raise TypeError(f"Contracter: idxs must be an integer tensor (got {idxs.dtype})")
        E = idxs.shape[0]
        for x, dim, name in ((x1, self.base_dim1, "x1"), (x2, self.base_dim2, "x2")):
            if x.dim() < 1 or x.shape[0] != E or math.prod(x.shape[1:]) != self.mul * dim:
                raise ValueError(f"Contracter: {name} of shape {tuple(x.shape)} does not match {E} edges of {self.mul} x {dim}")
            if x.device != idxs.device:
                raise ValueError(f"Contracter: {name} is on {x.device}, idxs on {idxs.device}")
        hit = self._tab_cache.get("route")
        if hit is not None and hit[0] is idxs and hit[1] == idxs._version and hit[2] == n:
            return hit[4], hit
        prepared = idxs.to(torch.int64).contiguous()
        if idxs.is_cuda and torch.cuda.is_current_stream_capturing():
            return prepared, None
        is_sorted = False
        if E:
            lo, hi, is_sorted = torch.stack([prepared.min(), prepared.max(), (prepared[1:] >= prepared[:-1]).all().long()]).tolist()
            if lo < 0 or hi >= n:
                raise ValueError(f"Contracter: scatter index out of range: indices span [{lo}, {hi}], scatter_dim_size is {n}")
        # (index tensor, version, n, CSR of the fast route: built on first use, prepared int64 indices, sorted by centre)
        hit = (idxs, idxs._version, n, None, prepared, bool(is_sorted))
        self._tab_cache["route"] = hit
        return prepared, hit

    def _fast_route(self, checked, n: int, d2: int):
        """(EdgeCSR, l_max) when the call can use the fused pipeline's tensor-product kernels: scatter indices sorted by
        centre (what a centre-sorted neighbour list gives; ``checked`` by ``_checked_indices``) and a second operand that is
        a full spherical-harmonic basis (d2 = (l+1)^2).  ALLEGRO_B200_OP_FAST=0 keeps the generic operator kernels."""
        import os

        from ..data import build_csr

        lmax = int(round(d2 ** 0.5)) - 1
        if os.environ.get("ALLEGRO_B200_OP_FAST", "1") != "1" or (lmax + 1) ** 2 != d2 or lmax > 4 or checked is None or not checked[5]:
            return None, -1
        if checked[3] is None:
            idxs = checked[4]
            if idxs.is_cuda and torch.cuda.is_current_stream_capturing():
                return None, -1  # building the CSR synchronises
            checked = checked[:3] + (build_csr(torch.stack([idxs, idxs]), n),) + checked[4:]
            self._tab_cache["route"] = checked
        return checked[3], lmax

    def extra_repr(self):
        return f"{self.irreps_in1} x {self.irreps_in2} -> {self.irreps_out} | {self.mul} channels | {self.num_paths} paths"

    # ---- model modifier (the reference's enable_<Name>Contracter pattern, :253-310) ------
    @classmethod
    def enable_B200Contracter(cls, model: torch.nn.Module) -> torch.nn.Module:
        """Replace every module whose class is named ``Contracter`` (reference or ours) by a
        CUDA-backed one with identical constructor kwargs and state_dict."""

        def factory(old):
            dt = old.w3j.dtype
            prev = torch.get_default_dtype()
            torch.set_default_dtype(dt)
            try:
                new = cls(
                    irreps_in1=repr(old.irreps_in1).replace(" ", ""),
                    irreps_in2=repr(old.irreps_in2).replace(" ", ""),
                    irreps_out=repr(old.irreps_out).replace(" ", ""),
                    mul=old.mul,
                    instructions=old.instructions,
                    path_channel_coupling=old.path_channel_coupling,
                    scatter_factor=old.scatter_factor,
                    irrep_normalization=old.irrep_normalization,
                )
            finally:
                torch.set_default_dtype(prev)
            new.load_state_dict(old.state_dict())
            return new.to(old.w3j.device)

        def walk(mod):
            for name, child in list(mod.named_children()):
                if type(child).__name__ == "Contracter" and not isinstance(child, cls):
                    setattr(mod, name, factory(child))
                elif isinstance(child, torch.nn.ModuleList):
                    for i, c in enumerate(child):
                        if type(c).__name__ == "Contracter" and not isinstance(c, cls):
                            child[i] = factory(c)
                        else:
                            walk(c)
                else:
                    walk(child)

        walk(model)
        return model


B200Contracter = Contracter
