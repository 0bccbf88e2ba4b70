"""Models at l_max 0 and 4, the two ends of the range the kernels are instantiated for, against vectors produced by the
REFERENCE'S OWN CODE (tests/golden/ref_models_lmax.*.pt, written by tests/golden/make_lmax_vectors.py).

* The oracle reproduces every case to 1e-10 and builds the reference's tensor-product irreps.
* The product's host pipeline, with every kernel replaced by its torch restatement (tests/kernel_spec.py), reproduces
  every case to 1e-10, with and without the plain-GEMM backward, stress included.
* l_max above 4 is refused when the model is built, not at the first kernel launch.
The CUDA kernels on the same vectors: tests/test_gpu_lmax_grid.py.
"""
import glob
import os

import pytest
import torch

from golden_util import GOLDEN, load_sharded, unpack_state_dict
from test_host_pipeline import _rel, spec_kernels  # noqa: F401  (spec_kernels: pytest fixture)

CASES = {r["name"]: r for r in load_sharded("ref_models_lmax")}
KEYS = ("total_energy", "atomic_energy", "forces", "edge_energy")


def test_fixture_cases():
    assert sorted({r["kwargs"]["l_max"] for r in CASES.values()}) == [0, 4]
    assert {(r["kwargs"]["num_layers"], r["kwargs"].get("parity", True)) for r in CASES.values() if r["kwargs"]["l_max"] == 4} == \
        {(2, True), (2, False), (3, True), (3, False)}
    for f in glob.glob(os.path.join(GOLDEN, "ref_models_lmax.*.pt")):
        assert os.path.getsize(f) < 1_000_000
    # the l_max 4 tables the kernels see: 25 -> 25, 25 -> 49, 49 -> 25 and 25 -> 1
    from oracle.o3_ref import Irreps

    dims = {(Irreps(i1).dim, Irreps(o).dim) for r in CASES.values() if r["kwargs"]["l_max"] == 4 for i1, _, o, _ in r["tp_irreps"]}
    assert dims == {(25, 25), (25, 49), (49, 25), (25, 1)}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reproduces_reference(name):
    from oracle.model_ref import AllegroOracle

    rec = CASES[name]
    oracle = AllegroOracle(**rec["kwargs"])
    res = oracle.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    tps = oracle.model.allegro.tps
    assert [(repr(t.irreps_in1), repr(t.irreps_in2), repr(t.irreps_out), t.num_paths) for t in tps] == [tuple(t) for t in rec["tp_irreps"]]
    out = oracle(dict(rec["data"]))
    for key in KEYS:
        assert _rel(out[key], rec[key]) < 1e-10, (key, _rel(out[key], rec[key]))


@pytest.mark.parametrize("name", list(CASES))
def test_host_pipeline_reproduces_reference(name, spec_kernels):  # noqa: F811
    from allegro_b200.model import AllegroModel
    from oracle.model_ref import AllegroOracle

    rec = CASES[name]
    sd = unpack_state_dict(rec["state_dict"])
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(sd, strict=True)
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    for key in KEYS:
        assert _rel(out[key], rec[key]) < 1e-10, (key, _rel(out[key], rec[key]))
    oracle = AllegroOracle(**rec["kwargs"])
    oracle.load_state_dict(sd, strict=True)
    ref = oracle(dict(rec["data"]))
    assert _rel(out["stress"], ref["stress"]) < 1e-10


@pytest.mark.parametrize("l_max", [5, 6])
def test_lmax_above_4_is_refused_at_build(l_max):
    from allegro_b200 import systems
    from allegro_b200.model import AllegroModel

    kw = systems.model_kwargs("c2", 40.0, "float64")
    kw.update(l_max=l_max)
    with pytest.raises(NotImplementedError, match="l_max <= 4"):
        AllegroModel(**kw)
