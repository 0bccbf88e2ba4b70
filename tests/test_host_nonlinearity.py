"""Models built with mish or gelu MLP nonlinearities, on a CPU-only box.

* The nonlinearities themselves: the gains of the table in include/allegro_b200.h / DESIGN section 7, phi' against
  autograd of the torch phi, and fp64 gradcheck of the oracle MLP (tests/nonlin_oracle.py) for each of them.
* The product's host pipeline on models with mish / gelu in any of the three MLP families, with every kernel replaced
  by its fp64 restatement (tests/kernel_spec.py, and here the *_nl entries: ``nonlin`` selects phi), against the fp64
  oracle: 1e-10 in fp64, 5e-5 in fp32, the bars of test_host_pipeline.py.
* Dispatch: which fused entries a model asks for.  ab2_mlp2_readout only when the last latent MLP and the readout share
  one nonlinearity, the plain-GEMM backward only when every latent MLP shares the readout's, and a SiLU model passes no
  ``nonlin`` at all, so that it calls the entries without the _nl suffix argument for argument.
The kernels are checked on the GPU (tests/test_gpu_nonlinearity.py).
"""
import math

import pytest
import torch

import kernel_spec
import nonlin_oracle as NO
from golden_util import load_models

MODELS = {r["name"]: r for r in load_models()}
NAMES = ("silu", "mish", "gelu")
TABLE = {"silu": 1.676532, "mish": 1.486848, "gelu": 1.533530}


def _code_name():
    from allegro_b200 import _lib

    return {_lib.NL_SILU: "silu", _lib.NL_MISH: "mish", _lib.NL_GELU: "gelu"}


# ---- the nonlinearities --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_gains_match_the_table(name):
    from allegro_b200.nn._mlp import NONLINEARITIES

    assert abs(NONLINEARITIES[name].gain - TABLE[name]) < 1e-6
    assert abs(NO.GAINS[name] - TABLE[name]) < 1e-6
    assert abs(NONLINEARITIES[name].gain - NO.GAINS[name]) < 1e-8


def _extremes():
    base = torch.tensor([0.0, 1e-30, 3.0, 20.0, 88.0, 1e4], dtype=torch.float64)
    return torch.cat([base, -base, torch.linspace(-30, 30, 6001, dtype=torch.float64)])


@pytest.mark.parametrize("name", NAMES)
def test_dphi_is_the_derivative_of_phi(name):
    from allegro_b200.nn._mlp import NONLINEARITIES

    x = _extremes().requires_grad_(True)
    nl = NONLINEARITIES[name]
    (g,) = torch.autograd.grad(nl.phi(x).sum(), x)
    for d in (nl.dphi(x.detach()), NO.dphi(name, x.detach())):
        assert bool(torch.isfinite(d).all())
        assert float((d - g).abs().max()) < 1e-12
    assert torch.equal(nl.phi(x.detach()), NO.PHI[name](x.detach()))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_mlp_gradcheck(name):
    torch.manual_seed(0)
    mlp = NO.ScalarMLPFunction(5, 3, 2, 7, name).double()
    x = torch.randn(4, 5, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(mlp, (x,))


@pytest.mark.parametrize("name", NAMES + (None,))
def test_product_mlp_is_the_oracle_mlp(name):
    from allegro_b200.nn._mlp import ScalarMLPFunction

    torch.manual_seed(1)
    ref = NO.ScalarMLPFunction(6, 4, 1, 8, name, forward_weight_init=False).double()
    torch.manual_seed(1)
    mlp = ScalarMLPFunction(6, 4, 1, 8, name, forward_weight_init=False).double()
    # (the product's SiLU gain comes from a 200 001-point quadrature, the oracle's from 240 001 points: ~1e-15 apart)
    assert all(abs(a - b) < 1e-12 * b for a, b in zip(mlp.alphas, ref.alphas))
    x = torch.randn(10, 6, dtype=torch.float64)
    assert torch.allclose(mlp(x), ref(x), rtol=1e-12, atol=0)


def test_silu_oracle_is_the_oracle():
    """The oracle extension changes nothing for SiLU: same weights, gains and outputs as oracle.nn_ref's own class."""
    from oracle import nn_ref as R

    torch.manual_seed(2)
    a = R.ScalarMLPFunction(6, 4, 1, 8, "silu").double()
    torch.manual_seed(2)
    b = NO.ScalarMLPFunction(6, 4, 1, 8, "silu").double()
    x = torch.randn(5, 6, dtype=torch.float64)
    assert a.alphas == b.alphas and torch.equal(a(x), b(x))


def test_other_settings_still_raise():
    from allegro_b200.nn._mlp import ScalarMLPFunction

    with pytest.raises(NotImplementedError):
        ScalarMLPFunction(4, 4, 1, 8, "tanh")
    with pytest.raises(NotImplementedError):
        ScalarMLPFunction(4, 4, 1, 8, "mish", bias=True)


# ---- restated *_nl entries -------------------------------------------------------------------------------------------
def _phi(nonlin):
    return NO.PHI[_code_name()[nonlin]]


def _dphi(nonlin, x):
    return NO.dphi(_code_name()[nonlin], x)


def _store(out, o_segs, o_accum):
    c = 0
    for s, o in enumerate(o_segs):
        blk = out[:, c : c + o.shape[1]].to(o.dtype)
        if o_accum is not None and o_accum[s]:
            o += blk
        else:
            o.copy_(blk)
        c += o.shape[1]


def _spec(record):
    """fp64 restatements of linear / mlp2 / mlp2_readout / radial_pq_bwd with ``nonlin``; ``record`` collects
    (entry, nonlin passed or None, taken)."""
    from allegro_b200 import _lib

    def linear(a_segs, W, o_segs, o_accum=None, act=_lib.ACT_NONE, epi=_lib.EPI_NONE, aux=None, W_packed=None, a_aux=None, **kw):
        nl = kw.get("nonlin", _lib.NL_SILU)
        record.append(("linear", kw.get("nonlin"), True))
        cols = []
        for s, a in enumerate(a_segs):
            a = a.to(torch.float64)
            if act == _lib.ACT_SILU:
                a = _phi(nl)(a)
            elif act == _lib.ACT_MUL_DSILU and a_aux is not None and a_aux[s] is not None:
                a = a * _dphi(nl, a_aux[s].to(torch.float64))
            cols.append(a)
        out = torch.cat(cols, dim=-1) @ W.to(torch.float64)
        if epi == _lib.EPI_MUL_DSILU:
            out = out * _dphi(nl, aux.to(torch.float64))
        _store(out, o_segs, o_accum)

    def mlp2(a_segs, W1, W2, o_segs, pre, o_accum=None, backward=False, W1_packed=None, W2_packed=None, **kw):
        nl = kw.get("nonlin", _lib.NL_SILU)
        if W1.dtype != torch.float32:
            record.append(("mlp2", kw.get("nonlin"), False))
            return False
        record.append(("mlp2", kw.get("nonlin"), True))
        h = torch.cat([a.to(torch.float64) for a in a_segs], dim=-1) @ W1.to(torch.float64)
        if backward:
            h = h * _dphi(nl, pre.to(torch.float64))
        else:
            pre.copy_(h.to(pre.dtype))
            h = _phi(nl)(h)
        _store(h @ W2.to(torch.float64), o_segs, o_accum)
        return True

    def mlp2_readout(backward, x, s, xl, pre_l, pre_r, ez, w2_ro, W_packed, S, **kw):
        nl = kw.get("nonlin", _lib.NL_SILU)
        if x.dtype != torch.float32:
            record.append(("ro", kw.get("nonlin"), False))
            return False
        record.append(("ro", kw.get("nonlin"), True))
        core = cores[-1]
        lat, ro = core.layers[-1]["mlp"], core.readout
        d = lambda t: t.to(torch.float64)
        W1l, W2l, W1r, w2r = d(lat.W[0]), d(lat.W[1]), d(ro.W[0]), d(w2_ro)
        P = x.shape[1]
        if not backward:
            hl = torch.cat([d(x), d(s)], dim=-1) @ W1l
            pre_l.copy_(hl.to(pre_l.dtype))
            xl.copy_((_phi(nl)(hl) @ W2l).to(xl.dtype))
            hr = d(x) @ W1r[:P] + d(xl) @ W1r[P:]
            pre_r.copy_(hr.to(pre_r.dtype))
            ez.copy_((_phi(nl)(hr) @ w2r).to(ez.dtype))
        else:
            g_r = d(ez) @ w2r.T * _dphi(nl, d(pre_r))
            g_h = (g_r @ W1r[P:].T) @ W2l.T * _dphi(nl, d(pre_l))
            x.copy_((g_h @ W1l[:P].T + g_r @ W1r[:P].T).to(x.dtype))
            s.copy_((g_h @ W1l[P:].T).to(s.dtype))
        return True

    def radial_pq_bwd(dtype, S, p_cut, vec, ctr, nbr, types, rmax_table, bessel_w, PQ, g_out, aux, gvec, **kw):
        nl = kw.get("nonlin", _lib.NL_SILU)
        record.append(("radial_pq_bwd", kw.get("nonlin"), True))
        g = g_out.to(vec.dtype)
        if aux is not None:
            g = g * _dphi(nl, aux.to(vec.dtype))
        v = vec.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            out = kernel_spec._radial_pq(p_cut, v, ctr, nbr, types, rmax_table, bessel_w, PQ)
            (gv,) = torch.autograd.grad(out, v, g)
        gvec += gv

    cores = []
    return dict(linear=linear, mlp2=mlp2, mlp2_readout=mlp2_readout, radial_pq_bwd=radial_pq_bwd), cores


@pytest.fixture()
def spec(monkeypatch):
    from allegro_b200 import _lib
    from allegro_b200.model.allegro_models import FusedAllegroEnergy

    for name in kernel_spec.ALL:
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))
    record = []
    fns, cores = _spec(record)
    for name, fn in fns.items():
        monkeypatch.setattr(_lib, name, fn)

    def core(self):
        c = self._core_for(torch.device("cpu"))
        cores.append(c)
        return c

    monkeypatch.setattr(FusedAllegroEnergy, "core", core)
    return record


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    assert a.shape == b.shape, (a.shape, b.shape)
    if b.numel() == 0:
        return 0.0
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def _nl(embed, latent, readout):
    return dict(scalar_embed_mlp_nonlinearity=embed, allegro_mlp_nonlinearity=latent, readout_mlp_nonlinearity=readout)


# (golden case whose kwargs and frame are used, overrides); the fp32 cases use equal latent / readout hidden widths so that
# the fused readout is offered
EQ_WIDTH = dict(readout_mlp_hidden_layers_width=64, allegro_mlp_hidden_layers_width=64)
CASES = {
    "mish_c2arch_f64": ("c2_arch_S64_U32", _nl("mish", "mish", "mish")),
    "gelu_c2arch_f64": ("c2_arch_S64_U32", _nl("gelu", "gelu", "gelu")),
    "mish_c2arch_f32": ("c2_arch_S64_U32", dict(_nl("mish", "mish", "mish"), model_dtype="float32", **EQ_WIDTH)),
    "gelu_c2arch_f32": ("c2_arch_S64_U32", dict(_nl("gelu", "gelu", "gelu"), model_dtype="float32", **EQ_WIDTH)),
    "mixed_f64": ("c2_arch_S64_U32", _nl("gelu", "mish", "silu")),
    "mixed_f32": ("c2_arch_S64_U32", dict(_nl("gelu", "mish", "silu"), model_dtype="float32", **EQ_WIDTH)),
    "mish_depth2": ("c2_lmax2_L2", dict(_nl("mish", "mish", "mish"), allegro_mlp_hidden_layers_depth=2)),
    "mish_L1": ("c1_lmax1_L1", _nl("mish", "mish", "mish")),
    "mish_lmax3_L3": ("c5_lmax3_L3_5species", _nl("mish", "mish", "mish")),
    "gelu_spline": ("spline_embed_reftest_cfg", _nl("gelu", "gelu", "gelu")),
    "gelu_spline_f32": ("spline_embed_f32", dict(_nl("gelu", "gelu", "gelu"), **EQ_WIDTH)),
    "gelu_no_edges": ("no_edges_at_all", _nl("gelu", "mish", "gelu")),
}


def _models(case):
    from allegro_b200.model import AllegroModel

    base, over = CASES[case]
    rec = MODELS[base]
    kw = dict(rec["kwargs"], **over)
    torch.manual_seed(0)
    ref = NO.oracle(**dict(kw, model_dtype="float64"))
    model = AllegroModel(**kw)
    model.load_state_dict(ref.state_dict(), strict=True)
    return ref, model, dict(rec["data"]), kw


@pytest.mark.parametrize("case", list(CASES))
def test_host_pipeline_against_oracle(case, spec):
    ref, model, d, kw = _models(case)
    expect = ref(dict(d))
    out = model.model._energy_and_forces(dict(d), True)
    tol = 5e-5 if kw["model_dtype"] == "float32" else 1e-10
    for key in ("atomic_energy", "forces", "total_energy"):
        assert _rel(out[key], expect[key]) < tol, (key, _rel(out[key], expect[key]))
    if d["edge_index"].shape[1] == 0:
        assert spec == []
        return
    names = {v: k for k, v in _code_name().items()}
    core = model.model.core()
    # every call passes the nonlinearity of the MLP it evaluates, and nothing for SiLU
    passed = {n for _, n, _ in spec}
    allowed = {None} | {names[kw[k]] for k in ("scalar_embed_mlp_nonlinearity", "allegro_mlp_nonlinearity", "readout_mlp_nonlinearity")
                        if kw[k] not in ("silu", None)}
    assert passed <= allowed, (passed, allowed)
    assert names.get("silu") not in passed
    # the fused paths follow the nonlinearity, not its name
    fp32, two = kw["model_dtype"] == "float32", kw.get("allegro_mlp_hidden_layers_depth", 1) == 1
    uniform = kw["allegro_mlp_nonlinearity"] == kw["readout_mlp_nonlinearity"]
    same_width = kw["allegro_mlp_hidden_layers_width"] == kw["readout_mlp_hidden_layers_width"]
    assert core.ro_fused == (two and uniform and same_width)
    assert any(e == "ro" for e, _, _ in spec) == core.ro_fused
    assert any(e == "ro" and ok for e, _, ok in spec) == (fp32 and core.ro_fused)
    assert any(e == "mlp2" and ok for e, _, ok in spec) == (fp32 and any(e == "mlp2" for e, _, _ in spec))


def test_mixed_models_decline_the_shared_nonlinearity_paths(spec):
    """A model whose last latent MLP and readout differ in nonlinearity does not ask ab2_mlp2_readout; the uniform model
    of the same shape does."""
    for case, uniform in (("mixed_f32", False), ("mish_c2arch_f32", True)):
        spec.clear()
        _, model, d, _ = _models(case)
        model.model._energy_and_forces(dict(d), True)
        core = model.model.core()
        assert core.ro_fused == uniform
        assert any(e == "ro" for e, _, _ in spec) == uniform


def test_silu_model_calls_without_nonlin(spec):
    """A SiLU model passes no ``nonlin`` keyword anywhere: its calls are those of the entries without the _nl suffix."""
    from allegro_b200.model import AllegroModel

    rec = MODELS["c2_lmax2_L2_f32"]
    model = AllegroModel(**rec["kwargs"])
    from golden_util import unpack_state_dict

    model.load_state_dict(unpack_state_dict(rec["state_dict"]), strict=True)
    model.model._energy_and_forces(dict(rec["data"]), True)
    assert spec and all(n is None for _, n, _ in spec)
