"""The scalar-embed MLP's forward with the radial embedding formed in the GEMM's producers (ab2_radial_embed_fwd, reached
through ``_lib.radial_embed_fwd``) on the H100:

- bitwise against the two launches it replaces (``_lib.radial_pq_fwd`` for h, then ``_lib.linear`` with act = phi into
  [w0 | X[:, :S] | omega_0]) on identical inputs: ragged row counts, one to three species with a per-pair cutoff table,
  edges within an ulp of their pair's cutoff, every nonlinearity, hidden widths 64 and 32, the strided middle output
  segment (as X[:, :S] is) and the widest PQ that fits;
- the cases it declines: nothing computed, outputs untouched, and a model then takes the two launches;
- the backward after a fused forward, which stores no h, on both adjoint routes (h recomputed where the adjoint needs it);
- a c2-architecture model, which takes the fused kernel, against the fp64 oracle; the Hessian path keeps its stored h.
"""
import pytest
import torch

from allegro_b200 import _lib
from allegro_b200 import data as D
from allegro_b200.nn import _pipeline
from allegro_b200.phonons import hessian_vector_product
from test_gpu_force_constants import _cell_frame
from test_gpu_hessian import _oracle_model
from test_gpu_model import _check, _pair, _to_dev
from test_gpu_radial_adjoint import DEV, LD_MID, NLS, P_CUT, SEG, _four_species_pair, _inputs

pytestmark = pytest.mark.gpu


def _outs(M, seg=SEG, dtype=torch.float32, offset=0):
    """[w0 | X[:, :S] | omega_0] as the model lays them out, filled with a marker value."""
    X = torch.full((M, LD_MID + offset), 7.0, dtype=dtype, device=DEV)
    return [torch.full((M, seg[0]), 7.0, dtype=dtype, device=DEV), X[:, offset: offset + seg[1]], torch.full((M, seg[2]), 7.0, dtype=dtype, device=DEV)]


def _weights(a, seg=SEG, seed=0):
    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(a["H"], sum(seg), generator=g, dtype=torch.float64) / a["H"] ** 0.5).float().to(DEV)
    return W, _lib.linear_pack(W)


def _two_launches(a, W, Wp, nl, seg=SEG):
    dt = torch.float32
    outs = _outs(a["vec"].shape[0], seg)
    h = _lib.radial_pq_fwd(dt, a["H"], P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"])
    _lib.linear([h], W, outs, act=_lib.ACT_SILU, W_packed=Wp, nonlin=nl)
    return outs


def _fused(a, Wp, nl, seg=SEG, dtype=torch.float32, offset=0):
    outs = _outs(a["vec"].shape[0], seg, dtype, offset)
    ok = _lib.radial_embed_fwd(dtype, a["H"], P_CUT, a["vec"], a["ctr"], a["nbr"], a["types"], a["rmax"], a["bw"], a["PQ"], Wp, outs, nonlin=nl)
    return ok, outs


def _bitwise(got, ref):
    for i, (x, y) in enumerate(zip(got, ref)):
        assert torch.equal(x, y), f"output {i}: max |diff| {float((x - y).abs().max())}"


CASES = ([(M, 3, "silu", 64) for M in (1, 127, 128, 129, 200003)]
         + [(4097, T, nl, 64) for T in (1, 2, 3) for nl in NLS]
         + [(4097, T, nl, 32) for T in (1, 3) for nl in NLS])


@pytest.mark.parametrize("M,T,nl,H", CASES)
def test_fused_matches_two_launches_bitwise(M, T, nl, H):
    a = _inputs(M, T, H, seed=M + 10 * T + H)
    W, Wp = _weights(a, seed=M)
    ref = _two_launches(a, W, Wp, NLS[nl])
    n0 = _lib.PROF.launches
    ok, got = _fused(a, Wp, NLS[nl])
    assert ok and _lib.PROF.launches == n0 + 1
    _bitwise(got, ref)
    X = got[1].as_strided((M, LD_MID), (LD_MID, 1))
    assert bool((X[:, SEG[1]:] == 7.0).all())  # the rest of X's rows is not written


@pytest.mark.parametrize("H", [64, 32])
def test_widest_pq_that_fits(H):
    """Species are added until the entry declines: the widest PQ it takes still gives the two launches' bits."""
    M = 3000
    T = 1
    while _fused(_inputs(M, T + 1, H, seed=T + 1), _weights(_inputs(1, 1, H, seed=0))[1], _lib.NL_SILU)[0]:
        T += 1
        assert T < 16
    assert T >= 4
    a = _inputs(M, T, H, seed=T)
    W, Wp = _weights(a, seed=1)
    ok, got = _fused(a, Wp, _lib.NL_SILU)
    assert ok
    _bitwise(got, _two_launches(a, W, Wp, _lib.NL_SILU))


def test_zero_rows():
    a = _inputs(1, 1, 64, seed=1)
    e = torch.empty(0, dtype=torch.int32, device=DEV)
    outs = [t[:0] for t in _outs(1)]
    assert _lib.radial_embed_fwd(torch.float32, 64, P_CUT, a["vec"][:0], e, e, a["types"], a["rmax"], a["bw"], a["PQ"], _weights(a)[1], outs)


DECLINES = {
    "bf16": dict(dtype=torch.bfloat16),
    "fp64": dict(dtype=torch.float64),
    "hidden_128": dict(H=128),
    "n_above_256": dict(seg=(96, 64, 128)),
    "pq_beyond_smem": dict(T=12),
    "segment_not_32_wide": dict(seg=(80, 64, 112)),
    "segment_misaligned": dict(offset=1),        # middle segment X[:, 1:65]: not 16-byte aligned
    "not_8_bessels": dict(nb=5),
    "linear_tma_off": dict(option="linear_tma"),
    "linear_tc_off": dict(option="linear_tc"),
}


@pytest.mark.parametrize("case", list(DECLINES))
def test_declines(case):
    c = dict(dtype=torch.float32, H=64, T=2, seg=SEG, offset=0, nb=8, option=None)
    c.update(DECLINES[case])
    a = _inputs(1000, c["T"], c["H"], seed=5)
    dt = c["dtype"]
    # (an image of an fp32 matrix for every dtype, so that the entry itself, not a missing image, declines)
    _, Wp = _weights(a, c["seg"])
    acc = _lib.ACC_DTYPE[dt]
    bw = a["bw"][: c["nb"]].to(acc)
    outs = _outs(1000, c["seg"], dt, c["offset"])
    before = [t.clone() for t in outs]
    n0 = _lib.PROF.launches
    if c["option"]:
        _lib.set_option(c["option"], 0)
    try:
        ok = _lib.radial_embed_fwd(dt, c["H"], P_CUT, a["vec"].to(acc), a["ctr"], a["nbr"], a["types"], a["rmax"].to(acc), bw, a["PQ"].to(acc),
                                   Wp, outs)
    finally:
        if c["option"]:
            _lib.set_option(c["option"], 1)
    torch.cuda.synchronize()
    assert ok is False
    _bitwise(outs, before)
    assert _lib.PROF.launches == n0  # a declined call is not counted as a launch


def test_unknown_nonlinearity_is_an_error():
    a = _inputs(100, 1, 64, seed=2)
    with pytest.raises(RuntimeError, match="nonlinearity"):
        _fused(a, _weights(a)[1], 7)


# ---- the backward after a fused forward ------------------------------------------------------------------------------
def _upstream(model):
    return model.model._upstream


def test_backward_after_fused_forward_on_both_adjoint_routes(monkeypatch):
    """A fused forward saves no h.  The fused adjoint does not need it; with that kernel declined, the two-launch adjoint
    recomputes h, and both meet the oracle and each other."""
    oracle, model, d = _pair("c2", 3, "float32")
    _check(oracle, model, d, 1e-4, 1e-4)
    up = _upstream(model)
    assert (up.fwd_path, up.bwd_path) == ("fused", "fused")
    f_fused = model(_to_dev(d))[D.FORCE_KEY].clone()

    real_bwd, real_fwd = _lib.radial_pq_bwd, _lib.radial_pq_fwd
    calls = []

    def no_gemm(*args, gemm=None, **kw):
        if gemm is not None:
            return False
        return real_bwd(*args, **kw)

    def count_fwd(*args, **kw):
        calls.append(1)
        return real_fwd(*args, **kw)

    monkeypatch.setattr(_lib, "radial_pq_bwd", no_gemm)
    monkeypatch.setattr(_lib, "radial_pq_fwd", count_fwd)
    _check(oracle, model, d, 1e-4, 1e-4)
    assert (up.fwd_path, up.bwd_path) == ("fused", "two_launch")
    assert len(calls) == 1  # h recomputed by the backward, once per model call
    f_two = model(_to_dev(d))[D.FORCE_KEY]
    assert len(calls) == 2
    # the two adjoints sum over the hidden columns in different orders (include/allegro_b200.h, ab2_radial_pq_bwd_gemm)
    assert float((f_two - f_fused).abs().max() / f_fused.abs().max()) <= 1e-5


def test_two_launch_adjoint_recomputes_h():
    """UpstreamPack.backward on the two-launch route, driven directly with the fused forward's stand-in for h (a meta
    tensor), against the same call with the stored h: bitwise the same gvec."""
    _, model, d = _pair("c2", 3, "float32")
    model(_to_dev(d))  # (the upstream constants are built on the first call)
    up = _upstream(model)
    E, S = 3000, up.S_pq
    a = _inputs(E, up.rmax_table.shape[0], S, seed=9)
    vec = a["vec"]
    csr = type("Csr", (), dict(ctr=a["ctr"], nbr=a["nbr"]))()
    g = torch.Generator().manual_seed(4)
    gouts = [torch.randn(E, w, generator=g).to(DEV) for w in SEG]
    h = _lib.radial_pq_fwd(torch.float32, S, up.p, vec, a["ctr"], a["nbr"], a["types"], up.rmax_table, up.bessel_w, up.PQ)
    wtp = up.mlp.WTp[1]
    up.mlp.WTp[1] = None  # the fused adjoint declines: the two launches run
    try:
        got, ref = torch.zeros(E, 3, device=DEV), torch.zeros(E, 3, device=DEV)
        up.backward(("pq_fold", None, [torch.empty(E, S, device="meta")]), gouts, vec, csr, a["types"], got)
        assert up.bwd_path == "two_launch"
        up.backward(("pq_fold", None, [h]), gouts, vec, csr, a["types"], ref)
    finally:
        up.mlp.WTp[1] = wtp
    assert bool(ref.abs().max() > 0)
    assert torch.equal(got, ref)


# ---- whole models ------------------------------------------------------------------------------------------------------
def test_c2_model_takes_the_fused_kernel():
    oracle, model, d = _pair("c2", 3, "float32")
    _check(oracle, model, d, 1e-4, 1e-4)
    assert _upstream(model).fwd_path == "fused"


@pytest.mark.parametrize("case", ["fp64", "hidden_128"])
def test_model_declines_take_two_launches(case):
    if case == "fp64":
        oracle, model, d = _pair("c2", 3, "float64")
        tol = 1e-9
    else:
        oracle, model, d = _pair("c2", 3, "float32", scalar_embed_mlp_hidden_layers_width=128)
        tol = 1e-4
    _check(oracle, model, d, tol, tol)
    assert _upstream(model).fold_radial
    assert _upstream(model).fwd_path == "two_launch"


def test_model_four_species_is_bitwise_the_two_launches(monkeypatch):
    """Four species (PQ of 16 pairs, which the fused adjoint declines but the forward takes): the model's outputs are the
    bits of the same model with the fused forward turned away."""
    oracle, model, d = _four_species_pair("float32")
    dd = _to_dev(d)
    out = model(dd)
    assert _upstream(model).fwd_path == "fused"
    monkeypatch.setattr(_lib, "radial_embed_fwd", lambda *a, **k: False)
    ref = model(dd)
    assert _upstream(model).fwd_path == "two_launch"
    for k in (D.FORCE_KEY, D.PER_ATOM_ENERGY_KEY):
        assert torch.equal(out[k], ref[k]), k
    _check(oracle, model, d, 1e-4, 1e-4)


def test_hessian_path_keeps_its_stored_h(monkeypatch):
    """The forward-mode Hessian reads the stored h (phi'' terms): its upstream forward keeps it, on the two-launch route."""
    _, model, kw = _oracle_model("c2_small", "float32")
    pos, cell, types, _ = _cell_frame("hcp", kw, torch.float32)
    saved = []
    real = _pipeline.UpstreamPack.forward

    def spy(self, *args, **k):
        out = real(self, *args, **k)
        saved.append((k.get("keep_h", False), out, self.fwd_path))
        return out

    monkeypatch.setattr(_pipeline.UpstreamPack, "forward", spy)
    v = torch.randn(pos.shape[0], 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    hv = hessian_vector_product(model, pos, cell, types, v)
    assert bool(torch.isfinite(hv).all())
    assert saved and all(keep for keep, _, _ in saved)
    for _, (kind, _, pre), path in saved:
        assert kind == "pq_fold" and path == "two_launch" and pre[0].is_cuda
