"""The kernel plug-in point applied to a whole model, pinned to what the reference's own model builder produced.

`Contracter.enable_B200Contracter(model)` is the analogue of the reference's `enable_TritonContracter` /
`enable_CuEquivarianceContracter` model modifiers (allegro/nn/_strided/_contract.py:253-310).  tests/golden/ref_modifier.pt
records, for one model built by the reference's own `AllegroModel` (third-party imports resolved to tests/golden/_stubs),
its constructor kwargs, its `state_dict` and the constructor state of every `Contracter` in it.  The same model is
assembled here from the oracle's restatement and loaded with the reference's `state_dict`; every `Contracter` must be
replaced by the B200 operator with the reference's constructor state and `state_dict`, and nothing else may change.
(The forward of the replaced operator needs a GPU: tests/test_zx_gpu_reference_golden.py.)
"""
import os

import pytest
import torch

from golden_util import GOLDEN, unpack_state_dict


def test_enable_b200_contracter_on_reference_model():
    from allegro_b200.nn import B200Contracter
    from oracle import nn_ref as R
    from oracle.model_ref import AllegroOracle

    rec = torch.load(os.path.join(GOLDEN, "ref_modifier.pt"), weights_only=False)
    ref_sd = unpack_state_dict(rec["state_dict"])
    model = AllegroOracle(**rec["kwargs"])
    model.model.load_state_dict(ref_sd, strict=True)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    old = list(model.model.allegro.tps)
    assert len(old) == len(rec["tps"]) and all(type(tp) is R.Contracter for tp in old)
    out = B200Contracter.enable_B200Contracter(model)
    assert out is model
    new = list(model.model.allegro.tps)
    assert len(new) == len(old) and all(isinstance(tp, B200Contracter) for tp in new)
    for i, (ref, b) in enumerate(zip(rec["tps"], new)):
        assert (repr(b.irreps_in1), repr(b.irreps_in2), repr(b.irreps_out)) == tuple(ref["irreps"])
        assert (b.mul, b.num_paths, b.path_channel_coupling, b.scatter_factor, bool(b.w3j_is_ij_diagonal)) == (
            ref["mul"], ref["num_paths"], ref["path_channel_coupling"], ref["scatter_factor"], ref["w3j_is_ij_diagonal"])
        w3j, weights = ref_sd[f"allegro.tps.{i}.w3j"], ref_sd[f"allegro.tps.{i}.weights"]
        assert b.w3j.dtype == w3j.dtype and torch.equal(b.w3j, w3j) and torch.equal(b.weights, weights)
    after = model.state_dict()
    assert list(after.keys()) == list(before.keys())
    assert all(torch.equal(after[k], before[k]) for k in before)
    # every other module of the model is untouched
    assert type(model.model.allegro) is R.Allegro_Module
    # the replaced operator refuses CPU tensors instead of silently falling back
    tp = new[0]
    with pytest.raises(RuntimeError):
        tp(torch.zeros(2, tp.mul, tp.base_dim1, dtype=torch.float64), torch.zeros(2, tp.mul, tp.base_dim2, dtype=torch.float64),
           torch.zeros(2, dtype=torch.long), 2)
