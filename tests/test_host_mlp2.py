"""Host logic of the fused two-layer MLP path on a CPU-only box.

tests/kernel_spec.py restates every other kernel; here ``_lib.mlp2`` is restated as well (what include/allegro_b200.h says
ab2_mlp2 computes, in fp64 torch), so that PackedMLP's fused forward and backward -- segment views, accumulate flags, the
stored pre-activation, the rank-1 readout backward without the zero-padded gradient -- run end to end against the
vectors produced by the reference's own code.  The kernel itself is checked on the GPU (tests/test_gpu_mlp2.py).
"""
import pytest
import torch

import kernel_spec
from golden_util import load_models, model_case_ids, unpack_state_dict

MODELS = {r["name"]: r for r in load_models()}


def _dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def _mlp2_spec(calls):
    def mlp2(a_segs, W1, W2, o_segs, pre, o_accum=None, backward=False, W1_packed=None, W2_packed=None):
        if W1.dtype != torch.float32:
            return False  # the kernel takes fp32 storage only; the caller runs two linear calls
        calls.append((backward, W1.shape[0]))
        A = torch.cat([a.to(torch.float64) for a in a_segs], dim=-1)
        h = A @ W1.to(torch.float64)
        if backward:
            h = h * _dsilu(pre.to(torch.float64))
        else:
            pre.copy_(h.to(pre.dtype))
            h = torch.nn.functional.silu(h)
        out = h @ W2.to(torch.float64)
        c = 0
        for s, o in enumerate(o_segs):
            blk = out[:, c : c + o.shape[1]].to(o.dtype)
            if o_accum is not None and o_accum[s]:
                o += blk
            else:
                o.copy_(blk)
            c += o.shape[1]
        return True

    return mlp2


@pytest.fixture()
def spec_kernels_mlp2(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    calls = []
    monkeypatch.setattr(_lib, "mlp2", _mlp2_spec(calls))
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))
    return calls


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    if b.numel() == 0:
        return 0.0
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


@pytest.mark.parametrize("name", model_case_ids())
def test_host_pipeline_with_fused_mlp(name, spec_kernels_mlp2):
    from allegro_b200.model import AllegroModel

    rec = MODELS[name]
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    fp32 = rec["kwargs"]["model_dtype"] == "float32"
    tol = 5e-5 if fp32 else 1e-10
    for key in ("atomic_energy", "forces", "edge_energy", "edge_features", "total_energy"):
        if key in rec:
            assert _rel(out[key], rec[key]) < tol, (key, _rel(out[key], rec[key]))
    calls = spec_kernels_mlp2
    if fp32:
        assert any(not bwd for bwd, _ in calls), "the forward MLPs did not take the fused path"
        assert any(bwd and k == 1 for bwd, k in calls), "the readout backward did not take the rank-1 fused path"
    else:
        assert not calls
