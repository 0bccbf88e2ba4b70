"""Model builders with the reference's kwargs: AllegroModel / AllegroEnergyModel /
FullAllegroEnergyModel / FullAllegroModel
(/root/reference/allegro/model/allegro_models.py:70-305).

``AllegroModel(**kwargs)(data) -> data`` reads ``pos``, ``edge_index`` [2,E] int64 (row 0 =
centre), ``atom_types`` and optional ``cell``/``edge_cell_shift`` and writes
``atomic_energy`` [N,1], ``total_energy``, ``forces`` [N,3] (+ ``edge_features``,
``edge_energy``), exactly the fields the reference model writes.  Sub-module names are the
reference's SequentialGraphNetwork keys (:222-228,262-268,297) so state_dict prefixes match.

The energy model is ONE fused module: the per-edge hot path runs in liballegro_b200.so;
there is no torch/e3nn fallback for it.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Union

import torch

from .. import _lib
from .. import data as D
from ..nn._modules import (
    Allegro_Module,
    EdgeLengthNormalizer,
    EdgewiseReduce,
    PerTypeScaleShift,
    TwoBodyBesselScalarEmbed,
    TwoBodySplineScalarEmbed,
    TwoBodySphericalHarmonicTensorEmbed,
)
from ..nn._mlp import ScalarMLPFunction
from ..nn._pipeline import AllegroCore, UpstreamPack, core_apply, energy_forces
from ..nn._zbl import instantiate_pair_potential
from ..o3 import Irreps

_DTYPES = {"float32": torch.float32, "float64": torch.float64, "bfloat16": torch.bfloat16}
_EMBED_TARGETS = {
    "allegro.nn.TwoBodyBesselScalarEmbed": TwoBodyBesselScalarEmbed,
    "allegro_b200.nn.TwoBodyBesselScalarEmbed": TwoBodyBesselScalarEmbed,
    "allegro.nn.TwoBodySplineScalarEmbed": TwoBodySplineScalarEmbed,
    "allegro_b200.nn.TwoBodySplineScalarEmbed": TwoBodySplineScalarEmbed,
}


def _instantiate_embed(cfg: Dict, **kw):
    cfg = dict(cfg or {"_target_": "allegro.nn.TwoBodyBesselScalarEmbed"})
    target = cfg.pop("_target_", "allegro.nn.TwoBodyBesselScalarEmbed")
    if target not in _EMBED_TARGETS:
        raise NotImplementedError(f"radial_chemical_embed target {target!r}: only the reference's Bessel and spline embeddings exist")
    return _EMBED_TARGETS[target](**cfg, **kw)


class FusedAllegroEnergy(torch.nn.Module):
    """What FullAllegroEnergyModel returns: the reference's module sequence as one module."""

    def __init__(
        self,
        r_max: float,
        type_names: Sequence[str],
        irreps_edge_sh,
        tensor_track_allowed_irreps,
        radial_chemical_embed: Dict,
        radial_chemical_embed_dim: Optional[int] = None,
        per_edge_type_cutoff=None,
        scalar_embed_mlp_hidden_layers_depth: int = 1,
        scalar_embed_mlp_hidden_layers_width: int = 64,
        scalar_embed_mlp_nonlinearity: Optional[str] = "silu",
        num_layers: int = 2,
        num_scalar_features: int = 64,
        num_tensor_features: int = 16,
        allegro_mlp_hidden_layers_depth: int = 1,
        allegro_mlp_hidden_layers_width: int = 64,
        allegro_mlp_nonlinearity: Optional[str] = "silu",
        tp_path_channel_coupling: bool = True,
        readout_mlp_hidden_layers_depth: int = 1,
        readout_mlp_hidden_layers_width: int = 32,
        readout_mlp_nonlinearity: Optional[str] = "silu",
        avg_num_neighbors: Optional[float] = None,
        weight_individual_irreps: bool = True,
        per_type_energy_scales=None,
        per_type_energy_shifts=None,
        per_type_energy_scales_trainable: bool = False,
        per_type_energy_shifts_trainable: bool = False,
        pair_potential: Optional[Dict] = None,
        forward_normalize: bool = True,
        model_dtype: str = "float32",
    ):
        super().__init__()
        assert avg_num_neighbors is not None, "`avg_num_neighbors` must be set for Allegro models"
        self.model_dtype = _DTYPES[model_dtype]
        self.type_names = list(type_names)
        self.r_max = float(r_max)
        self.avg_num_neighbors = float(avg_num_neighbors)
        S = num_scalar_features
        self.edge_norm = EdgeLengthNormalizer(r_max, type_names, per_edge_type_cutoff)
        self.radial_chemical_embed = _instantiate_embed(
            radial_chemical_embed,
            type_names=type_names,
            module_output_dim=S if radial_chemical_embed_dim is None else radial_chemical_embed_dim,
            forward_weight_init=forward_normalize,
        )
        self.scalar_embed_mlp = ScalarMLPFunction(
            self.radial_chemical_embed.out_dim, S, scalar_embed_mlp_hidden_layers_depth,
            scalar_embed_mlp_hidden_layers_width, scalar_embed_mlp_nonlinearity, forward_weight_init=forward_normalize,
        )
        # like the reference builder (allegro_models.py:185-193), `weight_individual_irreps` is NOT forwarded to the
        # tensor embedding: the initial features always carry per-irrep weights
        self.tensor_embed = TwoBodySphericalHarmonicTensorEmbed(
            irreps_edge_sh, num_tensor_features, S, forward_weight_init=forward_normalize,
        )
        self.allegro = Allegro_Module(
            num_layers=num_layers, num_scalar_features=S, num_tensor_features=num_tensor_features,
            tensor_track_allowed_irreps=tensor_track_allowed_irreps, input_irreps=self.tensor_embed.irreps_edge_sh,
            scalar_input_dim=S, avg_num_neighbors=avg_num_neighbors, tp_path_channel_coupling=tp_path_channel_coupling,
            weight_individual_irreps=weight_individual_irreps,
            latent_kwargs=dict(
                hidden_layers_depth=allegro_mlp_hidden_layers_depth, hidden_layers_width=allegro_mlp_hidden_layers_width,
                nonlinearity=allegro_mlp_nonlinearity, bias=False, forward_weight_init=forward_normalize,
            ),
        )
        self.edge_readout = ScalarMLPFunction(
            S * (num_layers + 1), 1, readout_mlp_hidden_layers_depth, readout_mlp_hidden_layers_width,
            readout_mlp_nonlinearity, forward_weight_init=forward_normalize,
        )
        self.edge_eng_sum = EdgewiseReduce(D.EDGE_ENERGY_KEY, D.PER_ATOM_ENERGY_KEY, factor=1.0 / math.sqrt(2 * avg_num_neighbors))
        self.per_type_energy_scale_shift = PerTypeScaleShift(
            type_names, per_type_energy_scales, per_type_energy_shifts, per_type_energy_scales_trainable,
            per_type_energy_shifts_trainable,
        )
        # pair potential after the scale/shift (allegro_models.py:270-288)
        self.pair_potential = instantiate_pair_potential(pair_potential, type_names)
        self._core: Optional[AllegroCore] = None
        self._core_key = None
        self._caches: Dict[str, tuple] = {}

    # ------------------------------------------------------------------------------------
    def _param_key(self):
        # buffers too: the dense w3j tensors are state the kernels' tables are built from
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def core(self) -> AllegroCore:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("allegro_b200: the model must live on a CUDA device (no CPU path for the hot path)")
        return self._core_for(dev)

    def _core_for(self, dev) -> AllegroCore:
        """Packed device constants, rebuilt whenever a parameter or buffer changed (load_state_dict, .to())."""
        key = (self._param_key(), str(dev))
        if self._core is None or self._core_key != key:
            self._core = AllegroCore(self.tensor_embed, self.allegro, self.edge_readout, self.avg_num_neighbors,
                                     self.model_dtype, dev)
            import os

            fold = self._core if os.environ.get("ALLEGRO_B200_FOLD_EMBED", "1") == "1" else None  # default on: one GEMM less per direction
            self._upstream = UpstreamPack(self.edge_norm, self.radial_chemical_embed, self.scalar_embed_mlp, self.model_dtype, dev,
                                          fold_embed_of=fold)
            self._core_key = key
        return self._core

    def energy_and_forces(self, data: D.Type, stress: bool = False) -> D.Type:
        """Energies AND forces in one pass of hand-written kernels (no torch autograd anywhere):
        what ForceStressOutput(AllegroEnergyModel) computes (allegro_models.py:101-103).  With
        ``stress=True`` and a cell in ``data`` also nequip's ``stress`` = sym(sum_z r_z (x) dE/dr_z)/V and
        ``virial`` = -sym(...) ([1,3,3] each), from the same per-edge gradients."""
        pos = data[D.POSITIONS_KEY]
        if not pos.is_cuda:
            raise RuntimeError("allegro_b200: inputs must be CUDA tensors (no CPU fallback on the hot path)")
        return self._energy_and_forces(data, stress)

    def _cached(self, slot: str, srcs, extra, build):
        """Derived per-neighbour-list data (CSR, int32 types, shift vectors) keyed on the IDENTITY of the
        source tensors, their in-place version counters and ``extra``.  The cache keeps references to the
        sources, so their storage cannot be recycled for another frame's tensors while the entry lives (a
        key made of data_ptr alone would match a new frame that the caching allocator placed at the same
        address)."""
        hit = self._caches.get(slot)
        vers = tuple(t._version for t in srcs)
        if hit is not None and len(hit[0]) == len(srcs) and all(a is b for a, b in zip(hit[0], srcs)) and hit[1] == vers and hit[2] == extra:
            return hit[3]
        val = build()
        self._caches[slot] = (tuple(srcs), vers, extra, val)
        return val

    @staticmethod
    def _single_frame(data: D.Type):
        """The fused path evaluates ONE frame (like the reference's compiled/deployed model, _compile.py:10-74):
        a batched dict (``batch`` with more than one frame, or several cells) is rejected instead of being
        summed into one total energy."""
        b = data.get(D.BATCH_KEY)
        if b is not None and b.numel() > 0 and int(b.max()) > 0:
            raise NotImplementedError("allegro_b200: batched frames are not supported on the fused path; evaluate frames one at a time")
        c = data.get(D.CELL_KEY)
        if c is not None and c.numel() != 9:
            raise NotImplementedError("allegro_b200: more than one cell in `data` (batched frames) is not supported")

    def _energy_and_forces(self, data: D.Type, stress: bool) -> D.Type:
        self._single_frame(data)
        pos = data[D.POSITIONS_KEY]
        core = self.core()
        n = pos.shape[0]
        prepared = D.CSR_KEY in data  # prebuilt CSR (+ shift vectors in CSR order): data.neighbor_csr
        csr = data[D.CSR_KEY] if prepared else self._csr(data[D.EDGE_INDEX_KEY], n)
        shift_vec = None
        if prepared:
            shift_vec = data.get(D.EDGE_SHIFT_VEC_KEY)
            if shift_vec is not None:
                shift_vec = shift_vec.to(pos.dtype).contiguous()
        elif D.EDGE_CELL_SHIFT_KEY in data and D.CELL_KEY in data:
            sh, cell = data[D.EDGE_CELL_SHIFT_KEY], data[D.CELL_KEY]

            def _shift():
                s = sh if csr.perm is None else sh[csr.perm]
                return (s.to(pos.dtype) @ cell.view(3, 3).to(pos.dtype)).contiguous()

            shift_vec = self._cached("shift", (sh, cell), (id(csr), pos.dtype), _shift)
        types_in = data[D.ATOM_TYPE_KEY]
        types = types_in.reshape(-1)
        if types.shape[0] != n:
            raise ValueError(f"atom_types has {types.shape[0]} entries for {n} atoms")
        types_i32 = self._cached("types", (types_in,), (n,), lambda: types.to(torch.int32).contiguous())
        ss = self.per_type_energy_scale_shift
        # a prepared CSR may hold rows for the first n_c atoms only (the owned centres of a slab, halo.py; neighbours index
        # all n atoms): energies exist for those centres, forces for every atom
        types_c = types[: csr.num_atoms]
        gscale = ss.scales[types_c].to(core.acc)
        want_virial = bool(stress) and D.CELL_KEY in data
        pair = None
        if self.pair_potential is not None:
            pair = (self.pair_potential, self.edge_norm.rmax_table.to(device=pos.device, dtype=core.acc))
        Ei, F, X, Ez, virial, Ei_pair = energy_forces(core, self._upstream, csr, pos.detach().contiguous(), types_i32, shift_vec,
                                                      gscale, want_virial, pair=pair)
        e_atom = ss(Ei.unsqueeze(-1), types_c)
        if Ei_pair is not None:
            e_atom = e_atom + Ei_pair.unsqueeze(-1).to(e_atom.dtype)
        out = dict(data)
        if csr.perm is not None:
            inv = torch.empty_like(csr.perm)
            inv[csr.perm] = torch.arange(csr.perm.shape[0], device=csr.perm.device)
            X, Ez = X[inv], Ez[inv]
        out[D.EDGE_FEATURES_KEY], out[D.EDGE_ENERGY_KEY] = X, Ez
        out[D.PER_ATOM_ENERGY_KEY] = e_atom
        out[D.TOTAL_ENERGY_KEY] = e_atom.sum(dim=0, keepdim=True)
        out[D.FORCE_KEY] = F.to(pos.dtype)
        if want_virial:
            cell = data[D.CELL_KEY].view(3, 3).to(virial.dtype)
            volume = torch.dot(cell[0], torch.linalg.cross(cell[1], cell[2])).abs()
            sym = 0.5 * (virial + virial.T)
            out[D.STRESS_KEY] = (sym / volume).to(pos.dtype).unsqueeze(0)
            out[D.VIRIAL_KEY] = (-sym).to(pos.dtype).unsqueeze(0)
        return out

    def _csr(self, edge_index: torch.Tensor, n: int):
        return self._cached("csr", (edge_index,), (tuple(edge_index.shape), n), lambda: D.build_csr(edge_index, n))

    def forward(self, data: D.Type) -> D.Type:
        pos = data[D.POSITIONS_KEY]
        if not pos.is_cuda:
            raise RuntimeError("allegro_b200: inputs must be CUDA tensors (no CPU fallback on the hot path)")
        self._single_frame(data)
        core = self.core()
        ei = data[D.EDGE_INDEX_KEY]
        n = pos.shape[0]
        csr = self._csr(ei, n)
        ctr, nbr = csr.ctr.long(), csr.nbr.long()
        # a1: edge vectors (nequip with_edge_vectors_, tensorembed.py:86), in the positions' dtype
        vec = pos[nbr] - pos[ctr]
        if D.EDGE_CELL_SHIFT_KEY in data and D.CELL_KEY in data:
            sh = data[D.EDGE_CELL_SHIFT_KEY]
            if csr.perm is not None:
                sh = sh[csr.perm]
            vec = vec + sh.to(pos.dtype) @ data[D.CELL_KEY].view(3, 3).to(pos.dtype)
        types = data[D.ATOM_TYPE_KEY].reshape(-1)
        tc, tn = types[ctr], types[nbr]
        # upstream two-body scalar embedding (row f1; torch ops on the device)
        r = vec.norm(dim=-1)
        x_norm = self.edge_norm(r, tc, tn)
        mdt = torch.float32 if self.model_dtype == torch.bfloat16 else self.model_dtype
        x_emb = self.scalar_embed_mlp(self.radial_chemical_embed(x_norm, tc, tn, mdt))
        stash: Dict[str, torch.Tensor] = {}
        Ei = core_apply(core, csr, vec.to(core.acc), x_emb.to(self.model_dtype), stash)
        e_atom = self.per_type_energy_scale_shift(Ei.unsqueeze(-1), types)
        if self.pair_potential is not None:
            ez_pair = self.pair_potential.edge_energy(r, x_norm, tc, tn)
            e_atom = e_atom + torch.zeros(n, dtype=ez_pair.dtype, device=ez_pair.device).index_add_(0, ctr, ez_pair).unsqueeze(-1).to(e_atom.dtype)
        out = dict(data)
        inv = None
        if csr.perm is not None:
            inv = torch.empty_like(csr.perm)
            inv[csr.perm] = torch.arange(csr.perm.shape[0], device=csr.perm.device)
        for k_src, k_dst in (("edge_features", D.EDGE_FEATURES_KEY), ("edge_energy", D.EDGE_ENERGY_KEY)):
            v = stash[k_src]
            out[k_dst] = v if inv is None else v[inv]
        out[D.PER_ATOM_ENERGY_KEY] = e_atom
        out[D.TOTAL_ENERGY_KEY] = e_atom.sum(dim=0, keepdim=True)
        return out


class ForceStressOutput(torch.nn.Module):
    """nequip ForceStressOutput (wrapped at allegro_models.py:101-103): forces = -dE/dpos."""

    def __init__(self, model: torch.nn.Module):
        super().__init__()
        self.model = model

    def forward(self, data: D.Type) -> D.Type:
        if hasattr(self.model, "energy_and_forces") and not getattr(self, "use_autograd", False):
            # like nequip's ForceStressOutput, stress/virial come with the forces whenever a cell is given
            return self.model.energy_and_forces(data, stress=getattr(self, "compute_stress", True))
        data = dict(data)
        pos = data[D.POSITIONS_KEY].detach().clone().requires_grad_(True)
        data[D.POSITIONS_KEY] = pos
        with torch.enable_grad():
            out = self.model(data)
            (g,) = torch.autograd.grad(out[D.TOTAL_ENERGY_KEY].sum(), pos)
        out[D.FORCE_KEY] = -g
        out[D.POSITIONS_KEY] = pos.detach()
        return {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in out.items()}


def _builder_common(kwargs: Dict):
    """What nequip's @model_builder consumes: seed, model_dtype, compile_mode."""
    kwargs = dict(kwargs)
    seed = kwargs.pop("seed", None)
    kwargs.pop("compile_mode", None)  # CUDA graphs, not a tracing compiler, on this path
    model_dtype = kwargs.get("model_dtype", "float32")
    if seed is not None:
        torch.manual_seed(seed)
    return kwargs, model_dtype


def FullAllegroEnergyModel(**kwargs) -> FusedAllegroEnergy:
    kwargs, model_dtype = _builder_common(kwargs)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float32 if model_dtype == "bfloat16" else _DTYPES[model_dtype])
    try:
        return FusedAllegroEnergy(**kwargs)
    finally:
        torch.set_default_dtype(prev)


def AllegroEnergyModel(l_max: int, parity: bool = True, **kwargs) -> FusedAllegroEnergy:
    """allegro_models.py:70-92."""
    irreps_edge_sh = Irreps.spherical_harmonics(l_max, p=-1)
    if parity:
        allowed = Irreps([(1, (l, p)) for l in range(l_max + 1) for p in (1, -1)])
    else:
        allowed = irreps_edge_sh
    return FullAllegroEnergyModel(irreps_edge_sh=irreps_edge_sh, tensor_track_allowed_irreps=allowed, **kwargs)


def AllegroModel(**kwargs) -> ForceStressOutput:
    """allegro_models.py:101-103."""
    return ForceStressOutput(AllegroEnergyModel(**kwargs))


def FullAllegroModel(**kwargs) -> ForceStressOutput:
    return ForceStressOutput(FullAllegroEnergyModel(**kwargs))
