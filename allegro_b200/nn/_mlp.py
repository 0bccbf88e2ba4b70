"""ScalarMLPFunction: parameter holder + the fused-linear execution plan.

Mirrors nequip.nn.ScalarMLPFunction as the reference uses it
(/root/reference/allegro/nn/_allegro.py:90-93,192-213; tensorembed.py:76-81;
_edgeembed.py:59-64; allegro_models.py:173-183,231-241): layer k computes x @ (alpha_k W_k),
W_k ~ U(-sqrt3, sqrt3) of shape [h_in, h_out], alpha_k = gain_k / sqrt(fan), SiLU between
layers, no bias (SURVEY appendix A.3).  alpha is folded into the packed device weights, so
the kernels see plain [K, N] matrices.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch

from .. import _lib

# second-moment gain of SiLU: 1/sqrt(E_{z~N(0,1)}[silu(z)^2]) (e3nn normalize2mom), by quadrature
def _silu_gain() -> float:
    n = 200001
    z = torch.linspace(-12.0, 12.0, n, dtype=torch.float64)
    w = torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    s = z * torch.sigmoid(z)
    return float(1.0 / math.sqrt(torch.trapezoid(s * s * w, z)))


SILU_GAIN = _silu_gain()


class ScalarMLPFunction(torch.nn.Module):
    def __init__(
        self,
        input_dim: int,
        output_dim: int,
        hidden_layers_depth: int = 0,
        hidden_layers_width: Optional[int] = None,
        nonlinearity: Optional[str] = "silu",
        bias: bool = False,
        forward_weight_init: bool = True,
    ):
        super().__init__()
        if bias:
            raise NotImplementedError("bias=True is not used by Allegro models (allegro_models.py:204-210)")
        if nonlinearity not in ("silu", None):
            raise NotImplementedError(f"nonlinearity {nonlinearity!r}: only 'silu' / None have CUDA kernels")
        if hidden_layers_depth > 0 and hidden_layers_width is None:
            raise ValueError("hidden_layers_width required")
        self.dims = [input_dim] + hidden_layers_depth * [hidden_layers_width] + [output_dim]
        self.nonlinearity = nonlinearity
        self.is_nonlinear = hidden_layers_depth > 0 and nonlinearity is not None
        self.weights = torch.nn.ParameterList()
        self.alphas: List[float] = []
        gain = 1.0
        for h_in, h_out in zip(self.dims, self.dims[1:]):
            w = torch.empty(h_in, h_out)
            torch.nn.init.uniform_(w, -math.sqrt(3), math.sqrt(3))
            self.weights.append(torch.nn.Parameter(w))
            self.alphas.append(gain / math.sqrt(h_in if forward_weight_init else h_out))
            gain = SILU_GAIN if nonlinearity == "silu" else 1.0

    @property
    def input_dim(self):
        return self.dims[0]

    @property
    def output_dim(self):
        return self.dims[-1]

    def folded_weights(self) -> List[torch.Tensor]:
        """alpha_k * W_k in fp64 (host packing input)."""
        return [a * w.detach().double() for w, a in zip(self.weights, self.alphas)]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """Library (torch) evaluation; only used for the upstream two-body scalar embedding,
        which is outside the named hot path (SURVEY section 8 row f1)."""
        n = len(self.weights)
        for k, (w, a) in enumerate(zip(self.weights, self.alphas)):
            x = x @ (a * w).to(x.dtype)
            if k < n - 1 and self.nonlinearity == "silu":
                x = torch.nn.functional.silu(x)
        return x


class PackedMLP:
    """Device-resident weights of one ScalarMLPFunction + forward/backward through ab2_linear.

    ``out_perm``: optional permutation applied to the output columns of the last layer (used to
    bring env weights from the reference's [u][r] order to the internal [r][u] order).
    ``in_perm``: likewise for the input rows of the first layer.
    """

    def __init__(self, mlp: ScalarMLPFunction, dtype: torch.dtype, device, out_perm=None, in_perm=None, extra_first=None, post=None):
        ws = [w.cpu() for w in mlp.folded_weights()]  # packing is done on the host in fp64
        if extra_first is not None:
            extra_first = [w.detach().double().cpu() for w in extra_first]
        if post is not None:
            post = post.detach().double().cpu()
        if extra_first is not None:  # horizontally fused sibling linears sharing the input
            assert len(ws) == 1
            ws = [torch.cat([ws[0]] + list(extra_first), dim=1)]
        if in_perm is not None:
            ws[0] = ws[0][in_perm, :]
        if out_perm is not None:
            ws[-1] = ws[-1][:, out_perm]
        if post is not None:  # a following LINEAR map folded into the (linear) output layer: x W_last post
            ws[-1] = ws[-1].to(torch.float64) @ post.to(torch.float64)
        self.W64 = [w.detach().to(torch.float64).cpu() for w in ws]
        self.silu = mlp.nonlinearity == "silu"
        self.W = [w.to(device=device, dtype=dtype).contiguous() for w in ws]
        self.WT = [w.T.to(device=device, dtype=dtype).contiguous() for w in ws]
        # wgmma path: packed bf16 hi/lo images (None where the shape is not eligible)
        self.Wp = [_lib.linear_pack(w) for w in self.W]
        self.WTp = [_lib.linear_pack(w) for w in self.WT]
        # a width-<16 output (the readout's single energy column) makes the backward GEMM's K < 16, which the
        # tensor-core path cannot take: zero-pad K to 16 (the padded gradient columns are zero)
        self.out_pad = None
        n_out = ws[-1].shape[1]
        if n_out < 16 and dtype != torch.float64:
            wt = torch.zeros(16, ws[-1].shape[0], dtype=torch.float64)
            wt[:n_out] = ws[-1].T
            self.out_pad = wt.to(device=device, dtype=dtype).contiguous()
            self.out_pad_p = _lib.linear_pack(self.out_pad)
        self.dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
        self.dtype = dtype
        self.device = device

    @property
    def n_layers(self):
        return len(self.W)

    def forward(self, in_segs: Sequence[torch.Tensor], out_segs: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """Returns the list of stored pre-activations (needed by backward)."""
        M = in_segs[0].shape[0]
        pre: List[torch.Tensor] = []
        cur = list(in_segs)
        for k in range(self.n_layers):
            last = k == self.n_layers - 1
            act = _lib.ACT_SILU if (k > 0 and self.silu) else _lib.ACT_NONE
            if last:
                _lib.linear(cur, self.W[k], out_segs, act=act, W_packed=self.Wp[k])
            else:
                h = torch.empty(M, self.dims[k + 1], dtype=self.dtype, device=self.device)
                _lib.linear(cur, self.W[k], [h], act=act, W_packed=self.Wp[k])
                pre.append(h)
                cur = [h]
        return pre

    def backward(self, gout_segs: Sequence[torch.Tensor], pre: List[torch.Tensor], gin_segs: Sequence[torch.Tensor], gin_accum: Sequence[bool]):
        M = gout_segs[0].shape[0]
        cur = list(gout_segs)
        WT, WTp = list(self.WT), list(self.WTp)
        if self.out_pad is not None and self.out_pad_p is not None and len(cur) == 1 and cur[0].is_contiguous():
            pad = torch.zeros(M, 16, dtype=self.dtype, device=self.device)
            pad[:, : cur[0].shape[1]] = cur[0]
            cur = [pad]
            WT[-1], WTp[-1] = self.out_pad, self.out_pad_p
        for k in range(self.n_layers - 1, -1, -1):
            if k == 0:
                _lib.linear(cur, WT[0], gin_segs, o_accum=gin_accum, W_packed=WTp[0])
            else:
                g = torch.empty(M, self.dims[k], dtype=self.dtype, device=self.device)
                if self.silu:
                    _lib.linear(cur, WT[k], [g], epi=_lib.EPI_MUL_DSILU, aux=pre[k - 1], W_packed=WTp[k])
                else:
                    _lib.linear(cur, WT[k], [g], W_packed=WTp[k])
                cur = [g]

    # ---- "plain GEMM" backward for the common 2-layer SiLU MLP -------------------------------
    @property
    def is_two_layer_silu(self) -> bool:
        return self.n_layers == 2 and self.silu

    def hidden_grad(self, gout_segs: Sequence[torch.Tensor]) -> torch.Tensor:
        """g_h = g_out @ W2^T (no epilogue): gradient w.r.t. the hidden layer's *output*.  The SiLU'
        factor is applied by whichever GEMM consumes g_h (act=ACT_MUL_DSILU with aux=pre)."""
        M = gout_segs[0].shape[0]
        g_h = torch.empty(M, self.dims[1], dtype=self.dtype, device=self.device)
        _lib.linear(list(gout_segs), self.WT[1], [g_h], W_packed=self.WTp[1])
        return g_h

    def backward_plain(self, gout_segs: Sequence[torch.Tensor], pre: List[torch.Tensor], gin_segs: Sequence[torch.Tensor]):
        """Whole backward of a 2-layer SiLU MLP with two plain GEMMs (no epilogue-side global reads)."""
        g_h = self.hidden_grad(gout_segs)
        _lib.linear([g_h], self.WT[0], list(gin_segs), act=_lib.ACT_MUL_DSILU, a_aux=[pre[0]], W_packed=self.WTp[0])
