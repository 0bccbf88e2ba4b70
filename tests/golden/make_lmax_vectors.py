"""Generate golden vectors for models at the two ends of the supported l_max range (0 and 4) by EXECUTING THE REFERENCE'S
OWN CODE.

    python tests/golden/make_lmax_vectors.py          # needs /root/reference

The reference's `allegro/nn` and `allegro/model` modules run unmodified through the stand-ins, exactly as in
make_reference_vectors.py (whose loader this script reuses).  The cases are the small-width 32-atom FCC case of
ref_models.*.pt (c2_lmax2_L2) with l_max, the number of layers and the parity switch changed.

Output (committed): tests/golden/ref_models_lmax.<i>.pt only -- the shards of make_reference_vectors.py are not touched
(the stem `ref_models_lmax` is not matched by `ref_models.*.pt`).

What these vectors pin: the reference's irreps bookkeeping at l_max 4 (the 25 -> 25, 25 -> 49, 49 -> 25 and 25 -> 1
tensor-product tables with and without parity, their path weights and their w3j values) and at l_max 0 (a scalar-only
tensor track), and the energies and forces the reference computes from them.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_reference_vectors as MRV  # noqa: E402  (registers the reference package, imports allegro.model)
from golden_util import save_sharded  # noqa: E402

# (new name, reference case it is built on, overrides)
CASES = [
    ("lmax4_L2", "c2_lmax2_L2", dict(l_max=4, num_layers=2)),
    ("lmax4_L2_noparity", "c2_lmax2_L2", dict(l_max=4, num_layers=2, parity=False)),
    ("lmax4_L3", "c2_lmax2_L2", dict(l_max=4, num_layers=3)),
    ("lmax4_L3_noparity", "c2_lmax2_L2", dict(l_max=4, num_layers=3, parity=False)),
    ("lmax0_L1", "c2_lmax2_L2", dict(l_max=0, num_layers=1)),
    ("lmax0_L2", "c2_lmax2_L2", dict(l_max=0, num_layers=2)),
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
               "tp_irreps": [(repr(tp.irreps_in1), repr(tp.irreps_in2), repr(tp.irreps_out), tp.num_paths) for tp in model.model.allegro.tps]}
        out.append(rec)
        print(f"{name:20s} atoms {data['pos'].shape[0]:3d} edges {data['edge_index'].shape[1]:5d} E {float(res['total_energy']):+.6f} "
              f"max|F| {float(res['forces'].abs().max()):.4f}")
    n = save_sharded(out, "ref_models_lmax")
    print(f"{len(out)} cases in {n} shard(s)")


if __name__ == "__main__":
    run()
