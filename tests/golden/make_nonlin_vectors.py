"""Generate golden vectors for models with mish / gelu MLP nonlinearities by EXECUTING THE REFERENCE'S OWN CODE.

    python tests/golden/make_nonlin_vectors.py          # needs /root/reference

The reference's `allegro/nn` and `allegro/model` modules run unmodified, exactly as in make_reference_vectors.py (whose
loader this script reuses), with one difference: the nequip `ScalarMLPFunction` stand-in is the oracle's restatement for
every nonlinearity the reference builder documents (tests/nonlin_oracle.py: silu, mish, gelu or None), installed before
the stand-ins and the reference modules are imported.  The cases are reference cases of ref_models.*.pt with the three
nonlinearity kwargs changed.

Output (committed): tests/golden/ref_models_nonlin.<i>.pt only -- the shards of make_reference_vectors.py are not
touched (the stem `ref_models_nonlin` is not matched by `ref_models.*.pt`).

What these vectors pin (see also tests/golden/_stubs/README.md for the stand-ins in general): the reference's wiring of
the three kwargs -- that `scalar_embed_mlp_nonlinearity` reaches the two-body scalar-embed MLP,
`allegro_mlp_nonlinearity` every latent MLP and `readout_mlp_nonlinearity` the edge readout (allegro_models.py:173-241),
and which layers of which MLP carry an activation.  What they do NOT pin: nequip's own definition of the nonlinearities
and of the gain after each activation -- the stand-in supplies them (second-moment gains by quadrature, the exact erf
form of gelu), as it supplies SiLU's for ref_models.*.pt.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import nonlin_oracle  # noqa: E402
from oracle import nn_ref  # noqa: E402

# before the stand-ins (nequip.nn binds ScalarMLPFunction at import) and the reference modules are imported
nn_ref.ScalarMLPFunction = nonlin_oracle.ScalarMLPFunction

sys.path.insert(0, HERE)
import make_reference_vectors as MRV  # noqa: E402  (registers the reference package, imports allegro.model)
from golden_util import save_sharded  # noqa: E402


def _nl(embed, latent, readout):
    return dict(scalar_embed_mlp_nonlinearity=embed, allegro_mlp_nonlinearity=latent, readout_mlp_nonlinearity=readout)


# (new name, reference case it is built on, overrides)
CASES = [
    ("mish_c2arch_f64", "c2_arch_S64_U32", _nl("mish", "mish", "mish")),
    ("gelu_c2arch_f64", "c2_arch_S64_U32", _nl("gelu", "gelu", "gelu")),
    ("mish_c2arch_f32", "c2_arch_S64_U32", dict(_nl("mish", "mish", "mish"), model_dtype="float32")),
    ("gelu_c2arch_f32", "c2_arch_S64_U32", dict(_nl("gelu", "gelu", "gelu"), model_dtype="float32")),
    ("mixed_c2arch_f64", "c2_arch_S64_U32", _nl("gelu", "mish", "silu")),
    ("mixed_c2arch_f32", "c2_arch_S64_U32", dict(_nl("gelu", "mish", "silu"), model_dtype="float32")),
    ("mish_latent_depth2", "c2_lmax2_L2", dict(_nl("mish", "mish", "mish"), allegro_mlp_hidden_layers_depth=2)),
    ("mish_L1", "c1_lmax1_L1", _nl("mish", "mish", "mish")),
    ("mish_lmax3_L3", "c5_lmax3_L3_5species", _nl("mish", "mish", "mish")),
    ("gelu_spline", "spline_embed_reftest_cfg", _nl("gelu", "gelu", "gelu")),
    ("gelu_mish_no_edges", "no_edges_at_all", _nl("gelu", "mish", "gelu")),
]


def run():
    base = {name: (kw, data) for name, kw, data in MRV.model_cases()}
    out = []
    for name, src, over in CASES:
        kw, data = base[src]
        kw = dict(kw, **over)
        model = MRV.allegro.model.AllegroModel(**kw)  # reference builder
        res = model(dict(data))
        rec = {"name": name, "base": src, "kwargs": kw, "data": data, "state_dict": MRV.pack_state_dict(model.state_dict()),
               "total_energy": res["total_energy"], "atomic_energy": res["atomic_energy"], "forces": res["forces"],
               "edge_energy": res["edge_energy"],
               # which nonlinearity each MLP of the built model carries, as the reference wired it
               "mlp_nonlinearities": {n: m.nonlinearity for n, m in model.named_modules() if isinstance(m, nn_ref.ScalarMLPFunction)}}
        if res["edge_features"].numel() <= 10_000:
            rec["edge_features"] = res["edge_features"]
        out.append(rec)
        print(f"{name:22s} atoms {data['pos'].shape[0]:3d} edges {data['edge_index'].shape[1]:5d} E {float(res['total_energy']):+.6f}")
    n = save_sharded(out, "ref_models_nonlin")
    print(f"{len(out)} cases in {n} shard(s)")


if __name__ == "__main__":
    run()
