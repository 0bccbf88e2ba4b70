"""Parameter-holding mirrors of the reference graph modules.

Same constructor hyper-parameters, sub-module names and ``state_dict`` keys as
/root/reference/allegro/nn/{tensorembed,_allegro,edgewise,_edgeembed,scalarembed}.py so a
checkpoint of the reference architecture maps one-to-one (see INTEGRATION.md for the key
map).  The hot-path arithmetic of TwoBodySphericalHarmonicTensorEmbed / Allegro_Module /
EdgewiseReduce is NOT implemented here in torch: it runs in the fused CUDA pipeline
(nn/_pipeline.py).  Only the upstream two-body scalar embedding (SURVEY section 8 row f1,
outside the named hot path) is evaluated with torch ops, on the same device.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch

from .. import data as D
from ..o3 import Irrep, Irreps, allegro_layer_irreps
from ._contract import Contracter
from ._mlp import ScalarMLPFunction


class MakeWeightedChannels(torch.nn.Module):
    """allegro/nn/_strided/_channels.py:7-63 (bookkeeping only; the product Y[z,i]*w[z,u,l(i)]
    is formed on the fly inside ab2_env_sum / ab2_tp_fwd and never stored)."""

    def __init__(self, irreps_in, multiplicity_out: int, alpha: float = 1.0, weight_individual_irreps: bool = True):
        super().__init__()
        irreps_in = Irreps(irreps_in)
        assert all(m == 1 for m, _ in irreps_in) and multiplicity_out >= 1
        if alpha != 1.0:
            raise NotImplementedError("alpha != 1")
        self._num_irreps = len(irreps_in)
        self.multiplicity_out = multiplicity_out
        # weight_individual_irreps=False (one weight per channel shared by all irreps, _channels.py:56-63) runs on
        # the same kernels: the pipeline replicates the U weight columns over the irreps when it packs the linears
        self.weight_individual_irreps = bool(weight_individual_irreps)
        self.weight_numel = (len(irreps_in) if weight_individual_irreps else 1) * multiplicity_out
        if not weight_individual_irreps:
            self.register_buffer("_rtoi", torch.Tensor())  # the reference keeps this empty buffer in its state_dict (_channels.py:31)
        self.irreps_in = irreps_in


class EdgeLengthNormalizer(torch.nn.Module):
    """nequip EdgeLengthNormalizer (allegro_models.py:153-157): x = r / r_max[(t_i, t_j)]."""

    def __init__(self, r_max: float, type_names: Sequence[str], per_edge_type_cutoff=None):
        super().__init__()
        self.r_max = float(r_max)
        self.num_types = len(type_names)
        tab = torch.full((self.num_types, self.num_types), float(r_max), dtype=torch.float64)
        self.per_type = per_edge_type_cutoff is not None
        if self.per_type:
            names = list(type_names)
            for a, va in per_edge_type_cutoff.items():
                if isinstance(va, dict):
                    for b, vb in va.items():
                        tab[names.index(a), names.index(b)] = float(vb)
                else:
                    tab[names.index(a), :] = float(va)
            assert float(tab.max()) <= r_max + 1e-12
        self.register_buffer("rmax_table", tab, persistent=self.per_type)

    def forward(self, r: torch.Tensor, type_c: torch.Tensor, type_n: torch.Tensor) -> torch.Tensor:
        if self.per_type:
            return r / self.rmax_table[type_c, type_n].to(r.dtype)
        return r / self.r_max


def polynomial_cutoff(x: torch.Tensor, p: float) -> torch.Tensor:
    out = 1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x**p + p * (p + 2.0) * x ** (p + 1.0) - (p * (p + 1.0) / 2.0) * x ** (p + 2.0)
    return out * (x < 1.0)


class BesselEdgeLengthEncoding(torch.nn.Module):
    def __init__(self, num_bessels: int = 8, polynomial_cutoff_p: float = 6.0, trainable: bool = False):
        super().__init__()
        self.p = float(polynomial_cutoff_p)
        self.num_bessels = num_bessels
        w = torch.linspace(1.0, num_bessels, num_bessels, dtype=torch.float64).unsqueeze(0)
        if trainable:
            self.bessel_weights = torch.nn.Parameter(w)
        else:
            self.register_buffer("bessel_weights", w)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x.unsqueeze(-1)
        bw = self.bessel_weights.to(x.dtype)
        return torch.sinc(x * bw) * bw * polynomial_cutoff(x, self.p)


class ProductTypeEmbedding(torch.nn.Module):
    """allegro/nn/_edgeembed.py:13-85."""

    def __init__(self, num_types: int, in_dim: int, initial_embedding_dim: int, forward_weight_init: bool = True):
        super().__init__()
        assert initial_embedding_dim % 2 == 0, "`initial_embedding_dim` must be an even number"
        self.center_embed = torch.nn.Embedding(num_types, initial_embedding_dim // 2)
        self.neighbor_embed = torch.nn.Embedding(num_types, initial_embedding_dim // 2)
        self.basis_linear = ScalarMLPFunction(in_dim, initial_embedding_dim, forward_weight_init=forward_weight_init)
        assert not self.basis_linear.is_nonlinear

    def forward(self, basis: torch.Tensor, type_c: torch.Tensor, type_n: torch.Tensor) -> torch.Tensor:
        te = torch.cat((self.center_embed(type_c), self.neighbor_embed(type_n)), dim=-1)
        return te.to(basis.dtype) * self.basis_linear(basis)


class TwoBodyBesselScalarEmbed(torch.nn.Module):
    """allegro/nn/scalarembed.py:19-81."""

    def __init__(self, type_names, num_bessels=8, bessel_trainable=False, polynomial_cutoff_p=6, module_output_dim=64,
                 forward_weight_init=True, **_unused):
        super().__init__()
        self.bessel_encode = BesselEdgeLengthEncoding(num_bessels, polynomial_cutoff_p, bessel_trainable)
        self.type_embed = ProductTypeEmbedding(len(type_names), num_bessels, module_output_dim, forward_weight_init)
        self.out_dim = module_output_dim

    def forward(self, x_norm: torch.Tensor, type_c, type_n, model_dtype) -> torch.Tensor:
        return self.type_embed(self.bessel_encode(x_norm).to(model_dtype), type_c, type_n)


class PerClassSpline(torch.nn.Module):
    """allegro/nn/spline.py:8-89 (same buffers / parameter: lower, upper, class_embed.weight in fp64)."""

    def __init__(self, num_classes: int, num_channels: int, num_splines: int, spline_span: int, dtype=torch.float64):
        super().__init__()
        assert 0 <= spline_span <= num_splines and num_splines > 0
        self.num_classes, self.num_channels, self.num_splines, self.spline_span = num_classes, num_channels, num_splines, spline_span
        lower = torch.arange(-spline_span, num_splines - spline_span, dtype=dtype) / num_splines
        diff = (spline_span + 1) / num_splines
        self.register_buffer("lower", lower)
        self.register_buffer("upper", lower + diff)
        self._const = 2 * math.pi / diff
        self.class_embed = torch.nn.Embedding(num_classes, num_channels * num_splines, dtype=dtype)

    def flat_weights(self) -> torch.Tensor:
        """[(class, k), channel] view of class_embed.weight ([class, channel*K + k]) for the one-GEMM evaluation."""
        w = self.class_embed.weight.detach().view(self.num_classes, self.num_channels, self.num_splines)
        return w.permute(0, 2, 1).reshape(self.num_classes * self.num_splines, self.num_channels).contiguous()

    def forward(self, x: torch.Tensor, classes: torch.Tensor) -> torch.Tensor:
        from ._spline import spline_basis

        basis, _ = spline_basis(x.reshape(-1).to(self.lower.dtype), self.lower, self.upper, self._const)
        w = self.class_embed(classes).view(classes.size(0), self.num_channels, self.num_splines)
        return torch.bmm(w, basis.unsqueeze(-1)).squeeze(-1)


class TwoBodySplineScalarEmbed(torch.nn.Module):
    """allegro/nn/scalarembed.py:84-175."""

    def __init__(self, type_names, num_splines: int = 16, spline_span: int = 12, module_output_dim: int = 64,
                 forward_weight_init: bool = True, **_unused):
        super().__init__()
        self.num_types = len(type_names)
        self.spline = PerClassSpline(self.num_types * self.num_types, module_output_dim, num_splines, spline_span, dtype=torch.float64)
        bound = math.sqrt(3 / spline_span) if forward_weight_init else math.sqrt(3 / module_output_dim)
        torch.nn.init.uniform_(self.spline.class_embed.weight, a=-bound, b=bound)
        self.out_dim = module_output_dim

    def forward(self, x_norm: torch.Tensor, type_c: torch.Tensor, type_n: torch.Tensor, model_dtype: torch.dtype) -> torch.Tensor:
        return self.spline(x_norm, type_c * self.num_types + type_n).to(model_dtype)


class TwoBodySphericalHarmonicTensorEmbed(torch.nn.Module):
    """allegro/nn/tensorembed.py:16-96 (holder; arithmetic in ab2_sh_fwd + fused kernels)."""

    def __init__(self, irreps_edge_sh, num_tensor_features: int, scalar_dim: int, forward_weight_init: bool = True,
                 edge_sh_normalization: str = "component", edge_sh_normalize: bool = True, weight_individual_irreps: bool = True):
        super().__init__()
        irreps = Irreps.spherical_harmonics(irreps_edge_sh) if isinstance(irreps_edge_sh, int) else Irreps(irreps_edge_sh)
        lmax = irreps.lmax
        if lmax > 4:  # AB2_MAX_LMAX (include/allegro_b200.h): the kernels are instantiated for l_max 0..4
            raise NotImplementedError(f"l_max = {lmax}: the kernels support l_max <= 4")
        if repr(irreps) != repr(Irreps.spherical_harmonics(lmax)):
            raise NotImplementedError(f"irreps_edge_sh must be the full SH set 0..l_max with parity (-1)^l, got {irreps}")
        if edge_sh_normalization != "component" or not edge_sh_normalize:
            raise NotImplementedError("only normalize=True, normalization='component' (the reference defaults) have kernels")
        self.lmax = lmax
        self.irreps_edge_sh = irreps
        self.num_tensor_features = num_tensor_features
        self._edge_weighter = MakeWeightedChannels(irreps, num_tensor_features, weight_individual_irreps=weight_individual_irreps)
        self.env_embed_linear = ScalarMLPFunction(scalar_dim, self._edge_weighter.weight_numel, forward_weight_init=forward_weight_init)
        assert not self.env_embed_linear.is_nonlinear


class Allegro_Module(torch.nn.Module):
    """allegro/nn/_allegro.py:17-301 (holder: irreps build/pruning :101-160, TP + latent
    construction :163-213; forward :237-301 runs in the fused pipeline)."""

    def __init__(
        self,
        num_layers: int,
        num_scalar_features: int,
        num_tensor_features: int,
        tensor_track_allowed_irreps,
        input_irreps,
        scalar_input_dim: int,
        avg_num_neighbors: Optional[float] = None,
        tp_path_channel_coupling: bool = True,
        weight_individual_irreps: bool = True,
        latent_kwargs: Optional[dict] = None,
    ):
        super().__init__()
        assert num_layers >= 1
        assert avg_num_neighbors is not None, "`avg_num_neighbors` must be set for Allegro models, but `avg_num_neighbors=None` found"
        latent_kwargs = dict(latent_kwargs or {})
        self.num_layers, self.num_scalar_features, self.num_tensor_features = num_layers, num_scalar_features, num_tensor_features
        self.tensor_track_allowed_irreps = Irreps(tensor_track_allowed_irreps)
        assert set(m for m, _ in self.tensor_track_allowed_irreps) == {1}
        input_irreps = Irreps(input_irreps)
        assert all(m == 1 for m, _ in input_irreps)
        self._env_weighter = MakeWeightedChannels(input_irreps, num_tensor_features, weight_individual_irreps=weight_individual_irreps)
        self.first_layer_env_embed_projection = ScalarMLPFunction(
            scalar_input_dim, num_scalar_features + self._env_weighter.weight_numel
        )
        assert not self.first_layer_env_embed_projection.is_nonlinear
        env = Irreps([(1, ir) for _, ir in input_irreps])
        assert env[0][1] == Irrep("0e"), "env_embed_irreps must start with scalars"
        ins, outs = allegro_layer_irreps(input_irreps, self.tensor_track_allowed_irreps, num_layers)
        self.tps_irreps_in, self.tps_irreps_out = ins, outs
        self.latents = torch.nn.ModuleList()
        self.tps = torch.nn.ModuleList()
        self._n_scalar_outs = []
        for layer, (arg, out) in enumerate(zip(ins, outs)):
            tp = Contracter(
                irreps_in1=Irreps([(1, ir) for _, ir in arg]),
                irreps_in2=env,
                irreps_out=Irreps([(1, ir) for _, ir in out]),
                mul=num_tensor_features,
                path_channel_coupling=tp_path_channel_coupling,
                scatter_factor=1.0 / math.sqrt(avg_num_neighbors),
            )
            self.tps.append(tp)
            self._n_scalar_outs.append(1)
            assert tp.irreps_out[0][1] == Irrep("0e")
            self.latents.append(
                ScalarMLPFunction(
                    input_dim=num_scalar_features * (layer + 1) + num_tensor_features,
                    output_dim=num_scalar_features + (self._env_weighter.weight_numel if layer < num_layers - 1 else 0),
                    **latent_kwargs,
                )
            )

    def extra_repr(self) -> str:
        return (f"num layers {self.num_layers} | scalar features {self.num_scalar_features} | tensor features "
                f"{self.num_tensor_features} | scalar output dim {self.num_scalar_features * (self.num_layers + 1)}")


class EdgewiseReduce(torch.nn.Module):
    """allegro/nn/edgewise.py:10-60 (sum only; runs as ab2_edge_sum)."""

    def __init__(self, field: str, out_field: Optional[str] = None, factor: Optional[float] = None, reduce: str = "sum"):
        super().__init__()
        if reduce != "sum":
            raise NotImplementedError("only reduce='sum' is on the Allegro energy path")
        self.reduce, self.field = reduce, field
        self.out_field = f"{reduce}_{field}" if out_field is None else out_field
        self._factor = factor


class PerTypeScaleShift(torch.nn.Module):
    """nequip PerTypeScaleShift (allegro_models.py:251-260)."""

    def __init__(self, type_names, scales=None, shifts=None, scales_trainable=False, shifts_trainable=False):
        super().__init__()
        n = len(type_names)

        def _tab(v, default):
            if v is None:
                return torch.full((n,), default, dtype=torch.float64)
            if isinstance(v, dict):
                return torch.tensor([float(v[t]) for t in type_names], dtype=torch.float64)
            t = torch.as_tensor(v, dtype=torch.float64).reshape(-1)
            return t.expand(n).clone() if t.numel() == 1 else t.clone()

        for name, tab, train in (("scales", _tab(scales, 1.0), scales_trainable), ("shifts", _tab(shifts, 0.0), shifts_trainable)):
            if train:
                self.register_parameter(name, torch.nn.Parameter(tab))
            else:
                self.register_buffer(name, tab)

    def forward(self, e: torch.Tensor, types: torch.Tensor) -> torch.Tensor:
        return e * self.scales[types].to(e.dtype).unsqueeze(-1) + self.shifts[types].to(e.dtype).unsqueeze(-1)
