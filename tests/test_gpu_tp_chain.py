"""GPU checks of the composed two-layer tensor product (ab2_tp_chain_fwd / ab2_tp_chain_bwd).

Each kernel is compared with the fp64 composition of the stored-V path: layer 0 (9 x 9 -> 9, implicit V_0) writes V_1,
layer 1 (9 x 9 -> 1) reads it, and the backward runs the two adjoints with gV_1 in between, exactly as
tests/kernel_spec.py's tp_fwd / tp_bwd define them.  Small ragged inputs (centres with 0 and 1 edges, long centres,
one centre per CTA) use kernel_spec itself on the CPU; the c2-sized inputs use the same sums written for the device.
"""
import pytest
import torch

import kernel_spec

pytestmark = pytest.mark.gpu

L_OF = [0, 1, 1, 1, 2, 2, 2, 2, 2]


def _tables():
    from allegro_b200.nn._pipeline import _baked_table

    return _baked_table(9), _baked_table(1)


def _case(N, degrees, U, seed):
    g = torch.Generator().manual_seed(seed)
    deg = torch.as_tensor(degrees, dtype=torch.int64)
    row_ptr = torch.zeros(N + 1, dtype=torch.int64)
    row_ptr[1:] = torch.cumsum(deg, 0)
    E = int(row_ptr[-1])
    ctr = torch.repeat_interleave(torch.arange(N), deg)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    return dict(N=N, E=E, U=U, row_ptr=row_ptr.to(torch.int32), ctr=ctr.to(torch.int32), Y=r(E, 9), w0=r(E, 3 * U),
                gamma0=r(N, 9, U), gamma1=r(N, 9, U), cgw0=r(83, U), cgw1=r(9, U), g1=r(E, U), g2=r(E, U))


def _ragged(U):
    deg = [0, 1, 0, 0, 1, 1, 37, 0, 2, 100, 1, 0, 5, 8, 9, 7, 16, 0, 1, 3] * 8 + [0, 0, 1]
    return _case(len(deg), deg, U, seed=11 + U)


def _c2_sized(U):
    g = torch.Generator().manual_seed(5 + U)
    N = 10976
    deg = torch.poisson(torch.full((N,), 42.0), generator=g).to(torch.int64)
    return _case(N, deg, U, seed=7 + U)


# ---- fp64 reference: the stored-V composition ----------------------------------------------------
def _ref_spec(c):
    """kernel_spec.tp_fwd / tp_bwd on the CPU (small inputs)."""
    t0, t1 = _tables()
    N, E, U = c["N"], c["E"], c["U"]
    rp, ct = c["row_ptr"].long(), c["ctr"].long()
    V1 = torch.empty(E, 9, U, dtype=torch.float64)
    kernel_spec.tp_fwd(None, 2, N, E, U, 9, 9, t0, c["cgw0"], rp, ct, c["gamma0"], None, c["Y"], c["w0"], V1)
    s2 = torch.empty(E, 1, U, dtype=torch.float64)
    kernel_spec.tp_fwd(None, 2, N, E, U, 9, 1, t1, c["cgw1"], rp, ct, c["gamma1"], V1, None, None, s2)
    gV1 = torch.empty(E, 9, U, dtype=torch.float64)
    gg1 = torch.empty(N, 9, U, dtype=torch.float64)
    kernel_spec.tp_bwd(None, 2, N, E, U, 9, 1, t1, c["cgw1"], rp, ct, c["gamma1"], V1, None, None, c["g2"].view(E, 1, U), gV1, None, None, gg1)
    gV1[:, 0] += c["g1"]
    gw0 = torch.empty(E, 3 * U, dtype=torch.float64)
    gY = torch.zeros(E, 9, dtype=torch.float64)
    gg0 = torch.empty(N, 9, U, dtype=torch.float64)
    kernel_spec.tp_bwd(None, 2, N, E, U, 9, 9, t0, c["cgw0"], rp, ct, c["gamma0"], None, c["Y"], c["w0"], gV1, None, gw0, gY, gg0)
    return dict(s1=V1[:, 0], s2=s2[:, 0], gg1=gg1, gw0=gw0, gY=gY, gg0=gg0)


def _ref_dev(c, dev):
    """The same sums on the device in fp64 (c2-sized inputs)."""
    t0, t1 = _tables()
    N, E, U = c["N"], c["E"], c["U"]
    d = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in c.items()}
    ct = d["ctr"].long()
    lo = torch.tensor(L_OF, device=dev)
    g0, g1 = d["gamma0"][ct], d["gamma1"][ct]
    V0 = d["Y"].unsqueeze(-1) * d["w0"].view(E, 3, U)[:, lo]
    V1 = torch.zeros(E, 9, U, dtype=torch.float64, device=dev)
    for n, (i, j, k) in enumerate(t0.tolist()):
        V1[:, k] += d["cgw0"][n] * V0[:, i] * g0[:, j]
    s2 = torch.zeros(E, U, dtype=torch.float64, device=dev)
    for n, (i, j, _) in enumerate(t1.tolist()):
        s2 += d["cgw1"][n] * V1[:, i] * g1[:, j]
    gV1 = torch.zeros(E, 9, U, dtype=torch.float64, device=dev)
    gg1e = torch.zeros(E, 9, U, dtype=torch.float64, device=dev)
    for n, (i, j, _) in enumerate(t1.tolist()):
        gV1[:, i] += d["cgw1"][n] * d["g2"] * g1[:, j]
        gg1e[:, j] += d["cgw1"][n] * V1[:, i] * d["g2"]
    gV1[:, 0] += d["g1"]
    gV0 = torch.zeros(E, 9, U, dtype=torch.float64, device=dev)
    gg0e = torch.zeros(E, 9, U, dtype=torch.float64, device=dev)
    for n, (i, j, k) in enumerate(t0.tolist()):
        gV0[:, i] += d["cgw0"][n] * gV1[:, k] * g0[:, j]
        gg0e[:, j] += d["cgw0"][n] * V0[:, i] * gV1[:, k]
    gw0 = torch.zeros(E, 3, U, dtype=torch.float64, device=dev).index_add_(1, lo, d["Y"].unsqueeze(-1) * gV0)
    gY = (d["w0"].view(E, 3, U)[:, lo] * gV0).sum(-1)
    z = lambda t: torch.zeros(N, 9, U, dtype=torch.float64, device=dev).index_add_(0, ct, t)  # noqa: E731
    return dict(s1=V1[:, 0], s2=s2, gg1=z(gg1e), gw0=gw0.view(E, 3 * U), gY=gY, gg0=z(gg0e))


# ---- the kernels -------------------------------------------------------------------------------------
def _run(c, dev, gY0):
    from allegro_b200 import _lib

    f = {k: (v.to(dev, torch.float32) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in c.items()}
    rp, ct = c["row_ptr"].to(dev), c["ctr"].to(dev)
    E, N, U = c["E"], c["N"], c["U"]
    plan = _lib.tp_chain_plan(torch.float32, U, f["cgw0"], f["cgw1"])
    assert plan is not None
    nan = float("nan")
    o = dict(s1=torch.full((E, U), nan, device=dev), s2=torch.full((E, U), nan, device=dev), gg1=torch.full((N, 9, U), nan, device=dev),
             gg0=torch.full((N, 9, U), nan, device=dev), gw0=torch.full((E, 3 * U), nan, device=dev), gY=gY0.to(dev, torch.float32).clone())
    assert _lib.tp_chain_fwd(plan, False, rp, ct, f["gamma0"], None, f["Y"], f["w0"], o["s1"])
    assert _lib.tp_chain_fwd(plan, True, rp, ct, f["gamma0"], f["gamma1"], f["Y"], f["w0"], o["s2"])
    assert _lib.tp_chain_bwd(plan, False, rp, ct, f["gamma0"], None, f["Y"], f["w0"], None, f["g2"], None, None, o["gg1"])
    assert _lib.tp_chain_bwd(plan, True, rp, ct, f["gamma0"], f["gamma1"], f["Y"], f["w0"], f["g1"], f["g2"], o["gw0"], o["gY"], o["gg0"])
    torch.cuda.synchronize()
    return o


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("U", [32, 64])
@pytest.mark.parametrize("size", ["ragged", "c2"])
def test_tp_chain_matches_stored_composition(size, U):
    dev = torch.device("cuda")
    c = _ragged(U) if size == "ragged" else _c2_sized(U)
    ref = _ref_spec(c) if size == "ragged" else _ref_dev(c, dev)
    gY0 = torch.randn(c["E"], 9, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    out = _run(c, dev, gY0)
    for k in ("s1", "s2", "gg1", "gw0", "gg0"):
        assert torch.isfinite(out[k]).all(), k
        assert _rel(out[k], ref[k]) < 1e-5, (k, _rel(out[k], ref[k]))
    assert _rel(out["gY"].double().cpu() - gY0.float().double(), ref["gY"]) < 1e-5
    if size == "ragged":
        empty = (c["row_ptr"][1:] == c["row_ptr"][:-1]).nonzero().view(-1).to(dev)
        assert empty.numel() > 0 and (out["gg0"][empty] == 0).all() and (out["gg1"][empty] == 0).all()
    again = _run(c, dev, gY0)
    for k in out:
        assert torch.equal(out[k], again[k]), f"{k} differs between two launches"


def test_tp_chain_declined_writes_nothing():
    from allegro_b200 import _lib

    dev = torch.device("cuda")
    c = _ragged(32)
    f = {k: (v.to(dev, torch.float32) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in c.items()}
    rp, ct = c["row_ptr"].to(dev), c["ctr"].to(dev)
    E, N, U = c["E"], c["N"], 32
    plan = _lib.tp_chain_plan(torch.float32, U, f["cgw0"], f["cgw1"])
    assert _lib.tp_chain_plan(torch.float64, U, f["cgw0"], f["cgw1"]) is None
    assert _lib.tp_chain_plan(torch.float32, 16, f["cgw0"][:, :16], f["cgw1"][:, :16]) is None
    # w0 4-byte but not 16-byte aligned: the library declines the bulk copies
    w0_odd = torch.empty(E * 3 * U + 1, device=dev)[1:].view(E, 3 * U)
    w0_odd.copy_(f["w0"])
    s = torch.full((E, U), 7.0, device=dev)
    gg = torch.full((N, 9, U), 7.0, device=dev)
    gw0 = torch.full((E, 3 * U), 7.0, device=dev)
    gY = torch.full((E, 9), 7.0, device=dev)
    assert not _lib.tp_chain_fwd(plan, True, rp, ct, f["gamma0"], f["gamma1"], f["Y"], w0_odd, s)
    assert not _lib.tp_chain_bwd(plan, True, rp, ct, f["gamma0"], f["gamma1"], f["Y"], w0_odd, f["g1"], f["g2"], gw0, gY, gg)
    assert not _lib.tp_chain_fwd(None, False, rp, ct, f["gamma0"], None, f["Y"], f["w0"], s)
    torch.cuda.synchronize()
    for t in (s, gg, gw0, gY):
        assert (t == 7.0).all()
