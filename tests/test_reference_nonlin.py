"""Models with mish / gelu MLP nonlinearities against vectors produced by the REFERENCE'S OWN CODE.

tests/golden/ref_models_nonlin.*.pt were written by tests/golden/make_nonlin_vectors.py, which runs the unmodified
reference builder with the three nonlinearity kwargs set (its nequip ScalarMLPFunction stand-in is the restatement of
tests/nonlin_oracle.py).  They pin the reference's wiring -- which kwarg reaches which MLP -- to the oracle and to the
product's host pipeline; nequip's definitions of the nonlinearities and gains stay unpinned, as for SiLU.

* The oracle reproduces every case: 1e-10 relative in fp64, 1e-5 for the fp32 cases (the reference ran in fp32).
* Each MLP of the oracle carries the nonlinearity the reference gave the MLP of the same name.
* The product's host pipeline, with every kernel replaced by its fp64 restatement (test_host_nonlinearity.py), against the
  reference outputs: 1e-10 in fp64, 5e-5 in fp32.
"""
import pytest
import torch

import nonlin_oracle as NO
from golden_util import load_sharded, unpack_state_dict
from test_host_nonlinearity import _rel, spec  # noqa: F401  (spec: pytest fixture)

CASES = {r["name"]: r for r in load_sharded("ref_models_nonlin")}
KEYS = ("total_energy", "atomic_energy", "forces", "edge_energy", "edge_features")


def _names(d):
    """Module path -> nonlinearity, without the leading wrapper names (reference: model.<key>, oracle: <key>)."""
    return {k.split("model.", 1)[-1] if k.startswith("model.") else k: v for k, v in d.items()}


def test_fixture_cases():
    """The cases the generator writes: uniform mish / gelu, mixed, deeper, one and three layers, spline, no edges."""
    assert len(CASES) == 11
    nls = {tuple(r["kwargs"][k] for k in ("scalar_embed_mlp_nonlinearity", "allegro_mlp_nonlinearity", "readout_mlp_nonlinearity"))
           for r in CASES.values()}
    assert {("mish",) * 3, ("gelu",) * 3, ("gelu", "mish", "silu")} <= nls


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reproduces_reference(name):
    rec = CASES[name]
    oracle = NO.oracle(**rec["kwargs"])
    res = oracle.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    out = oracle(dict(rec["data"]))
    tol = 1e-10 if rec["kwargs"]["model_dtype"] == "float64" else 1e-5
    for key in KEYS:
        if key in rec:
            assert _rel(out[key], rec[key]) < tol, (key, _rel(out[key], rec[key]))
    # the reference's wiring of the three kwargs, MLP by MLP
    own = {n: m.nonlinearity for n, m in oracle.named_modules() if isinstance(m, NO.ScalarMLPFunction)}
    assert _names(own) == _names(rec["mlp_nonlinearities"])


@pytest.mark.parametrize("name", list(CASES))
def test_host_pipeline_reproduces_reference(name, spec):  # noqa: F811
    from allegro_b200.model import AllegroModel

    rec = CASES[name]
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    tol = 5e-5 if rec["kwargs"]["model_dtype"] == "float32" else 1e-10
    for key in ("atomic_energy", "forces", "total_energy", "edge_energy", "edge_features"):
        if key in rec:
            assert _rel(out[key], rec[key]) < tol, (key, _rel(out[key], rec[key]))
    # the product's MLPs carry the reference's nonlinearities too
    from allegro_b200.nn._mlp import ScalarMLPFunction

    own = {n: m.nonlinearity for n, m in model.named_modules() if isinstance(m, ScalarMLPFunction)}
    assert _names(own) == _names(rec["mlp_nonlinearities"])
