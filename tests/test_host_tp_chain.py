"""Host logic of the composed two-layer tensor product (ab2_tp_chain_fwd / ab2_tp_chain_bwd) on a CPU-only box.

The two entries are restated here in fp64 torch from the formulas in include/allegro_b200.h (per-centre A, B, G, H; no
V_1), and AllegroCore runs end to end through them against the vectors produced by the reference's own code.  The
restatement takes every storage type and width, so all two-layer l_max = 2 cases go through the composed path here;
which models take it on the GPU (fp32, U = 32 or 64, default backward) is checked separately.  The kernels themselves
are checked on the GPU (tests/test_gpu_tp_chain.py).
"""
import pytest
import torch

import kernel_spec
from golden_util import load_models, model_case_ids, unpack_state_dict

MODELS = {r["name"]: r for r in load_models()}
L_OF = torch.tensor([0, 1, 1, 1, 2, 2, 2, 2, 2])


def _tables():
    from allegro_b200.nn._pipeline import _baked_table

    return _baked_table(9).tolist(), _baked_table(1).tolist()


def _couplings(plan, gamma0, gamma1):
    """Per centre M0 [N][i][k][U] and M1 [N][k][U] (None without gamma1)."""
    t0, t1 = _tables()
    c0, c1 = plan["cgw0"].double(), plan["cgw1"].double()
    g0 = gamma0.double()
    N, _, U = g0.shape
    M0 = torch.zeros(N, 9, 9, U, dtype=torch.float64)
    for n, (i, j, k) in enumerate(t0):
        M0[:, i, k] += c0[n] * g0[:, j]
    M1 = None
    if gamma1 is not None:
        g1 = gamma1.double()
        M1 = torch.zeros(N, 9, U, dtype=torch.float64)
        for n, (k, j, _) in enumerate(t1):
            M1[:, k] += c1[n] * g1[:, j]
    return M0, M1


def _v0(Y, w0, U):
    return Y.double().unsqueeze(-1) * w0.double().reshape(Y.shape[0], 3, U)[:, L_OF]


def chain_fwd_spec(calls):
    def tp_chain_fwd(plan, last, row_ptr, ctr, gamma0, gamma1, Y, w0, s):
        calls.append(("fwd", bool(last)))
        M0, M1 = _couplings(plan, gamma0, gamma1 if last else None)
        Q = (M0 * M1.unsqueeze(1)).sum(2) if last else M0[:, :, 0]  # B_c or A_c [N][9][U]
        s.copy_((Q[ctr.long()] * _v0(Y, w0, s.shape[1])).sum(1).to(s.dtype))
        return True

    return tp_chain_fwd


def chain_bwd_spec(calls):
    def tp_chain_bwd(plan, first, row_ptr, ctr, gamma0, gamma1, Y, w0, g1, g2, gw0, gY, ggamma):
        calls.append(("bwd", bool(first)))
        t0, t1 = _tables()
        c0, c1 = plan["cgw0"].double(), plan["cgw1"].double()
        E, U = g2.shape
        N = gamma0.shape[0]
        c = ctr.long()
        M0, M1 = _couplings(plan, gamma0, gamma1 if first else None)
        v0 = _v0(Y, w0, U)
        b = g2.double().unsqueeze(1)
        G = torch.zeros(N, 9, U, dtype=torch.float64).index_add_(0, c, b * v0)
        gg = torch.zeros(N, 9, U, dtype=torch.float64)
        if not first:
            gM1 = (M0 * G.unsqueeze(2)).sum(1)  # sum_i M0[i][k] G[i]
            for n, (k, j, _) in enumerate(t1):
                gg[:, j] += c1[n] * gM1[:, k]
        else:
            a = g1.double().unsqueeze(1)
            A, B = M0[:, :, 0], (M0 * M1.unsqueeze(1)).sum(2)
            gv0 = A[c] * a + B[c] * b
            gw = torch.zeros(E, 3, U, dtype=torch.float64).index_add_(1, L_OF, Y.double().unsqueeze(-1) * gv0)
            gw0.copy_(gw.reshape(E, 3 * U).to(gw0.dtype))
            gY += (w0.double().reshape(E, 3, U)[:, L_OF] * gv0).sum(-1).to(gY.dtype)
            H = torch.zeros(N, 9, U, dtype=torch.float64).index_add_(0, c, a * v0)
            for n, (i, j, k) in enumerate(t0):
                gg[:, j] += c0[n] * ((H[:, i] if k == 0 else 0.0) + M1[:, k] * G[:, i])
        ggamma.copy_(gg.to(ggamma.dtype))
        return True

    return tp_chain_bwd


def _patch_spec(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    monkeypatch.setattr(FusedAllegroEnergy, "core", lambda self: self._core_for(torch.device("cpu")))


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    if b.numel() == 0:
        return 0.0
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _model(rec, **over):
    from allegro_b200.model import AllegroModel

    kw = dict(rec["kwargs"], **over)
    model = AllegroModel(**kw)
    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    return model


L2_CASES = [n for n in model_case_ids() if MODELS[n]["kwargs"].get("num_layers") == 2]


@pytest.mark.parametrize("name", L2_CASES)
def test_host_pipeline_with_tp_chain(name, monkeypatch):
    from allegro_b200 import _lib

    _patch_spec(monkeypatch)
    calls = []
    monkeypatch.setattr(_lib, "tp_chain_plan", lambda dtype, U, cgw0, cgw1: {"cgw0": cgw0, "cgw1": cgw1, "U": U})
    monkeypatch.setattr(_lib, "tp_chain_fwd", chain_fwd_spec(calls))
    monkeypatch.setattr(_lib, "tp_chain_bwd", chain_bwd_spec(calls))
    rec = MODELS[name]
    model = _model(rec)
    core = model.model.core()
    out = model.model._energy_and_forces(dict(rec["data"]), True)
    tol = 5e-5 if rec["kwargs"]["model_dtype"] == "float32" else 1e-10
    for key in ("atomic_energy", "forces", "edge_energy", "edge_features", "total_energy"):
        if key in rec:
            assert _rel(out[key], rec[key]) < tol, (key, _rel(out[key], rec[key]))
    if name.startswith("c2_"):  # l_max = 2 with parity: both tables have the baked structure
        assert core.chain is not None
    if core.chain is None:
        assert not calls
    elif rec["data"]["edge_index"].shape[1] > 0:
        assert calls == [("fwd", False), ("fwd", True), ("bwd", False), ("bwd", True)], calls


@pytest.mark.parametrize("dtype,taken", [("float32", True), ("float64", False), ("bfloat16", False)], ids=["fp32", "fp64", "bf16"])
def test_which_models_take_tp_chain(dtype, taken, monkeypatch):
    """The GPU rule of tp_chain_plan (fp32, U = 32 or 64) with the device check left out, on the U = 32 case."""
    from allegro_b200 import _lib

    _patch_spec(monkeypatch)
    takes = _lib.tp_chain_takes
    monkeypatch.setattr(_lib, "tp_chain_plan",
                        lambda dt, U, cgw0, cgw1: {"cgw0": cgw0, "cgw1": cgw1, "U": U} if takes(dt, U) else None)
    rec = MODELS["c2_arch_S64_U32"]
    assert rec["kwargs"]["num_tensor_features"] == 32
    core = _model(rec, model_dtype=dtype).model.core()
    assert (core.chain is not None) == taken
    # U outside {32, 64}: never
    assert _model(MODELS["c2_lmax2_L2_f32"]).model.core().chain is None
