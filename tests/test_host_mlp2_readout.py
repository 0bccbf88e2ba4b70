"""Host logic of the fused last-latent + readout path on a CPU-only box.

``_lib.mlp2_readout`` is restated in fp64 torch (what include/allegro_b200.h says ab2_mlp2_readout computes), on top of
the ``_lib.mlp2`` restatement of tests/test_host_mlp2.py, so that AllegroCore's fused forward and backward -- the split
of X into the prefix and x_L, the stored pre-activations, gX[:, :S L] and the last layer's gs -- run end to end against
the vectors produced by the reference's own code, and against the two separate MLPs.  The real wrapper's own checks run
against a stand-in library.  The kernel itself is checked on the GPU (tests/test_gpu_mlp2_readout.py).
"""
import pytest
import torch

import kernel_spec
from golden_util import load_models, model_case_ids, unpack_state_dict
from test_host_mlp2 import _dsilu, _mlp2_spec, _rel

MODELS = {r["name"]: r for r in load_models()}


def _mlp2_readout_spec(calls, core_of, decline=(), declined=None):
    """``decline``: the directions ("fwd", "bwd") in which the stand-in declines as the library does for a plan that
    does not fit, before writing anything; those calls go to ``declined``, the taken ones to ``calls``."""

    def mlp2_readout(backward, x, s, xl, pre_l, pre_r, ez, w2_ro, W_packed, S):
        if x.dtype != torch.float32:
            return False  # the kernel takes fp32 storage only
        if ("bwd" if backward else "fwd") in decline:
            declined.append(backward)
            return False
        calls.append(backward)
        core = core_of()
        lat, ro = core.layers[-1]["mlp"], core.readout
        d = lambda t: t.to(torch.float64)
        W1l, W2l, W1r, w2r = d(lat.W[0]), d(lat.W[1]), d(ro.W[0]), d(w2_ro)
        P = x.shape[1]
        if not backward:
            hl = torch.cat([d(x), d(s)], dim=-1) @ W1l
            pre_l.copy_(hl.to(pre_l.dtype))
            x_l = torch.nn.functional.silu(hl) @ W2l
            xl.copy_(x_l.to(xl.dtype))
            hr = d(x) @ W1r[:P] + d(xl) @ W1r[P:]
            pre_r.copy_(hr.to(pre_r.dtype))
            ez.copy_((torch.nn.functional.silu(hr) @ w2r).to(ez.dtype))
        else:
            g_r = d(ez) @ w2r.T * _dsilu(d(pre_r))
            g_h = (g_r @ W1r[P:].T) @ W2l.T * _dsilu(d(pre_l))
            x.copy_((g_h @ W1l[:P].T + g_r @ W1r[:P].T).to(x.dtype))
            s.copy_((g_h @ W1l[P:].T).to(s.dtype))
        return True

    return mlp2_readout


def _install_spec(monkeypatch, decline=(), mlp2_declines=False):
    """The kernels replaced by their restatements on the CPU -> (taken mlp2_readout calls, declined mlp2_readout calls,
    mlp2 calls).  ``mlp2_declines``: ab2_mlp2 declines every call (the callers then run two linear layers)."""
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    mlp2_calls = []
    if mlp2_declines:
        monkeypatch.setattr(_lib, "mlp2", lambda *a, **k: mlp2_calls.append(k.get("backward", False)) and False)
    else:
        monkeypatch.setattr(_lib, "mlp2", _mlp2_spec(mlp2_calls))
    cores = []
    calls, declined = [], []
    monkeypatch.setattr(_lib, "mlp2_readout", _mlp2_readout_spec(calls, lambda: cores[-1], decline, declined))

    def core(self):
        c = self._core_for(torch.device("cpu"))
        cores.append(c)
        return c

    monkeypatch.setattr(FusedAllegroEnergy, "core", core)
    return calls, declined, mlp2_calls


@pytest.fixture()
def spec_kernels_fused(monkeypatch):
    return _install_spec(monkeypatch)[0]


@pytest.mark.parametrize("name", model_case_ids())
def test_host_pipeline_with_fused_readout(name, spec_kernels_fused):
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
    kw = rec["kwargs"]
    two_layer = kw.get("allegro_mlp_hidden_layers_depth", 1) == 1 and kw.get("readout_mlp_hidden_layers_depth", 1) == 1
    same_width = kw["allegro_mlp_hidden_layers_width"] == kw["readout_mlp_hidden_layers_width"]
    if fp32 and two_layer and same_width and rec["data"]["pos"].shape[0] > 0:
        assert False in spec_kernels_fused and True in spec_kernels_fused, spec_kernels_fused
    else:
        assert not spec_kernels_fused


def _fused_offered(rec):
    kw = rec["kwargs"]
    two_layer = kw.get("allegro_mlp_hidden_layers_depth", 1) == 1 and kw.get("readout_mlp_hidden_layers_depth", 1) == 1
    same_width = kw["allegro_mlp_hidden_layers_width"] == kw["readout_mlp_hidden_layers_width"]
    return kw["model_dtype"] == "float32" and two_layer and same_width and rec["data"]["edge_index"].shape[1] > 0


@pytest.mark.parametrize("mlp2", ["mlp2_takes", "mlp2_declines"])
@pytest.mark.parametrize("decline", ["fwd", "bwd", "both"])
@pytest.mark.parametrize("name", model_case_ids())
def test_host_pipeline_readout_declines(name, decline, mlp2, monkeypatch):
    """ab2_mlp2_readout declining the forward only, the backward only, or both (as for a plan that does not fit the
    shared memory), with ab2_mlp2 taking or declining the separate MLPs.  The reference cases as they are must give the
    reference's results.  None of them is an fp32 model with equal latent and readout hidden widths, so each also runs
    as one (its other settings kept, new weights): AllegroCore's mixed paths -- the backward of a fused forward through
    the two separate MLPs, the fused backward of a forward that ran them separately -- must give what the fully fused
    path gives, at the bar of the fused-against-separate comparison below."""
    from allegro_b200.model import AllegroModel

    rec = MODELS[name]
    dirs = ("fwd", "bwd") if decline == "both" else (decline,)
    calls, declined, _ = _install_spec(monkeypatch, dirs, mlp2 == "mlp2_declines")
    model = AllegroModel(**rec["kwargs"])
    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    tol = 5e-5 if rec["kwargs"]["model_dtype"] == "float32" else 1e-10
    for key in ("atomic_energy", "forces", "edge_energy", "edge_features", "total_energy"):
        if key in rec:
            assert _rel(out[key], rec[key]) < tol, (key, _rel(out[key], rec[key]))
    assert _fused_offered(rec) or not (calls or declined)

    kw = dict(rec["kwargs"], model_dtype="float32", readout_mlp_hidden_layers_width=rec["kwargs"]["allegro_mlp_hidden_layers_width"])
    if not _fused_offered({"kwargs": kw, "data": rec["data"]}):
        return  # MLP depths the fused kernels are not built for, or no atoms
    torch.manual_seed(0)
    model = AllegroModel(**kw)
    _install_spec(monkeypatch)
    fused = model.model._energy_and_forces(dict(rec["data"]), True)
    calls, declined, mlp2_calls = _install_spec(monkeypatch, dirs, mlp2 == "mlp2_declines")
    mixed = model.model._energy_and_forces(dict(rec["data"]), True)
    # each direction asked once: the declined ones declined, the others taken; the separate MLPs then asked ab2_mlp2
    assert sorted(declined) == sorted(d == "bwd" for d in dirs), declined
    assert sorted(calls) == sorted(d == "bwd" for d in ("fwd", "bwd") if d not in dirs), calls
    assert mlp2_calls
    for key in ("atomic_energy", "forces", "edge_energy", "edge_features", "total_energy"):
        assert _rel(mixed[key], fused[key]) < 5e-5, (key, _rel(mixed[key], fused[key]))


def test_host_pipeline_unequal_hidden_widths(spec_kernels_fused):
    """Latent and readout hidden widths that differ: the fused path is not offered, the two MLPs run separately."""
    from allegro_b200.model import AllegroModel

    rec = MODELS["c2_lmax2_L2_f32"]
    kw = dict(rec["kwargs"], num_scalar_features=64, num_tensor_features=16, allegro_mlp_hidden_layers_width=64,
              readout_mlp_hidden_layers_width=32)
    model = AllegroModel(**kw)
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    assert bool(torch.isfinite(out["forces"]).all())
    assert not spec_kernels_fused


def test_host_pipeline_fused_matches_separate(spec_kernels_fused, monkeypatch):
    """An fp32 model whose latent and readout hidden widths agree takes the fused path in both directions, with the
    results of the two separate MLPs."""
    from allegro_b200 import _lib
    from allegro_b200.model import AllegroModel

    rec = MODELS["c2_lmax2_L2_f32"]
    kw = dict(rec["kwargs"], readout_mlp_hidden_layers_width=rec["kwargs"]["allegro_mlp_hidden_layers_width"])
    torch.manual_seed(0)
    model = AllegroModel(**kw)
    fused = model.model._energy_and_forces(dict(rec["data"]), True)
    assert False in spec_kernels_fused and True in spec_kernels_fused
    monkeypatch.setattr(_lib, "mlp2_readout", lambda *a, **k: False)
    separate = model.model._energy_and_forces(dict(rec["data"]), True)
    # the separate path stores gX in fp32 between its two calls, the restated fused one does not: fp32 tolerance
    for key in ("atomic_energy", "forces", "edge_energy", "edge_features", "total_energy"):
        if key in separate:
            assert _rel(fused[key], separate[key]) < 5e-5, (key, _rel(fused[key], separate[key]))


class _FakeLib:
    """Records the arguments of ab2_mlp2_readout and declines."""

    def __init__(self):
        self.args = None

    def ab2_mlp2_readout(self, *args):
        self.args = args
        from allegro_b200 import _lib

        return _lib.NOT_ELIGIBLE


@pytest.fixture()
def fake_lib(monkeypatch):
    import ctypes

    from allegro_b200 import _lib

    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(_lib, "_ptr", lambda t: None if t is None else ctypes.c_void_p(t.data_ptr()))
    monkeypatch.setattr(_lib, "_stream", lambda: ctypes.c_void_p(0))
    return fake


def _packed(k, n):
    return torch.zeros((n + 31) // 32 * 32 * k * 4, dtype=torch.uint8)


def test_wrapper_declines_unequal_hidden_widths(fake_lib):
    from allegro_b200 import _lib

    M, P, S, U, H, Hr = 10, 128, 64, 32, 64, 32
    z = lambda *sh: torch.zeros(*sh)
    W = [_packed(Hr, P + S), _packed(S, H), _packed(H, P + U)]
    assert not _lib.mlp2_readout(True, z(M, P), z(M, U), None, z(M, H), z(M, Hr), z(M, 1), z(Hr, 1), W, S)
    assert fake_lib.args is None  # declined before the library is called


def test_wrapper_passes_the_width_of_x_l(fake_lib):
    """The backward tells the library the true S (here 32), which it then declines, and not the hidden width."""
    from allegro_b200 import _lib

    M, P, S, U, H = 10, 64, 32, 32, 64
    z = lambda *sh: torch.zeros(*sh)
    W = [_packed(H, P + S), _packed(S, H), _packed(H, P + U)]
    assert not _lib.mlp2_readout(True, z(M, P), z(M, U), None, z(M, H), z(M, H), z(M, 1), z(H, 1), W, S)
    assert fake_lib.args[2:7] == (M, P, S, U, H)
    with pytest.raises(ValueError):  # images of other shapes than those stated are refused
        _lib.mlp2_readout(True, z(M, P), z(M, U), None, z(M, H), z(M, H), z(M, 1), z(H, 1), W, 64)
