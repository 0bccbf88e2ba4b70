"""ab2_mlp2_readout, the last latent MLP and the readout MLP in one kernel per direction, against the two ab2_mlp2 calls
it replaces (bitwise, except Ez, which is an fp32 dot product instead of a split-bf16 MMA) and against an fp64 reference."""
import pytest
import torch

from allegro_b200 import _lib

pytestmark = pytest.mark.gpu

S, U, H, L = 64, 32, 64, 2  # the c2 model
P = S * L


def _dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def _weights(gen):
    def w(k, n):
        return (torch.rand(k, n, generator=gen, device="cuda") * 2 - 1) * (3.0 / k) ** 0.5

    return w(P + U, H), w(H, S), w(P + S, H), w(H, 1)


def _pack(W):
    return _lib.linear_pack(W.contiguous())


@pytest.mark.parametrize("M", [77, 129, 40000, 461154])
def test_mlp2_readout(M):
    gen = torch.Generator(device="cuda").manual_seed(M)
    W1l, W2l, W1r, w2r = _weights(gen)
    # column views with leading dimensions wider than the view: X inside a wider buffer, s the first U columns of V
    Xbuf = torch.randn(M, P + S + 32, generator=gen, device="cuda")
    X = Xbuf[:, : P + S]
    s = torch.randn(M, 3 * U, generator=gen, device="cuda")[:, :U]
    Xbuf[:, P:] = float("nan")

    # forward: the two mlp2 calls, then the fused kernel
    X2 = X.clone()
    pre_l2, pre_r2 = torch.empty(M, H, device="cuda"), torch.empty(M, H, device="cuda")
    Ez2 = torch.empty(M, 1, device="cuda")
    assert _lib.mlp2([X2[:, :P], s], W1l, W2l, [X2[:, P:]], pre_l2, W1_packed=_pack(W1l), W2_packed=_pack(W2l))
    assert _lib.mlp2([X2], W1r, w2r, [Ez2], pre_r2, W1_packed=_pack(W1r), W2_packed=_pack(w2r))
    pre_l, pre_r = torch.full((M, H), 7.0, device="cuda"), torch.full((M, H), 7.0, device="cuda")
    Ez = torch.full((M, 1), 7.0, device="cuda")
    fwd_p = [_pack(W1l), _pack(W2l), _pack(W1r[:P]), _pack(W1r[P:])]
    assert _lib.mlp2_readout(False, X[:, :P], s, X[:, P:], pre_l, pre_r, Ez, w2r, fwd_p, S)
    torch.cuda.synchronize()
    assert torch.equal(pre_l, pre_l2)
    assert torch.equal(X[:, P:], X2[:, P:])
    assert torch.equal(pre_r, pre_r2)
    # fp64 reference of the forward
    d = lambda t: t.double()
    hl = torch.cat([d(X[:, :P]), d(s)], -1) @ d(W1l)
    xl = torch.nn.functional.silu(hl) @ d(W2l)
    hr = d(X[:, :P]) @ d(W1r[:P]) + xl @ d(W1r[P:])
    ez = torch.nn.functional.silu(hr) @ d(w2r)
    # Ez: the fp32 dot product is at least as close to fp64 as the split-bf16 MMA of the two-launch path (silu(pre_r)
    # taken from the kernel's own pre_r, so that only the last stage is compared).  The two differ by up to ~4e-6 of
    # max |Ez| -- the rounding of the split-bf16 MMA -- so the bound against it is 1e-5, not 1e-6.
    ez_r = torch.nn.functional.silu(d(pre_r)) @ d(w2r)
    assert float((Ez - Ez2).abs().max()) <= 1e-5 * float(Ez2.abs().max())
    assert float((d(Ez) - ez_r).abs().max()) <= max(float((d(Ez2) - ez_r).abs().max()), 1e-7 * float(ez_r.abs().max()))
    for got, ref in ((pre_l, hl), (X[:, P:], xl), (pre_r, hr), (Ez, ez)):
        assert float((d(got) - ref).abs().max()) <= 2e-4 * float(ref.abs().max())

    # backward: rank-1 readout mlp2 then last-latent mlp2, then the fused kernel
    gEz = torch.randn(M, 1, generator=gen, device="cuda")
    gX2 = torch.empty(M, P + S, device="cuda")
    gs2 = torch.empty(M, U, device="cuda")
    W1rT, W2lT, W1lT = W1r.T.contiguous(), W2l.T.contiguous(), W1l.T.contiguous()
    assert _lib.mlp2([gEz], w2r.T.contiguous(), W1rT, [gX2], pre_r, backward=True, W2_packed=_pack(W1rT))
    assert _lib.mlp2([gX2[:, P:]], W2lT, W1lT, [gX2[:, :P], gs2], pre_l, o_accum=[True, False], backward=True, W1_packed=_pack(W2lT),
                     W2_packed=_pack(W1lT))
    gXbuf = torch.full((M, P + S + 32), 7.0, device="cuda")
    gX = gXbuf[:, : P + S]
    gsbuf = torch.full((M, 3 * U), 7.0, device="cuda")
    gs = gsbuf[:, :U]
    assert _lib.mlp2_readout(True, gX[:, :P], gs, None, pre_l, pre_r, gEz, w2r, [_pack(W1rT), _pack(W2lT), _pack(W1lT)], S)
    torch.cuda.synchronize()
    assert torch.equal(gX[:, :P], gX2[:, :P])
    assert torch.equal(gs, gs2)
    assert bool((gXbuf[:, P:] == 7.0).all()) and bool((gsbuf[:, U:] == 7.0).all())  # nothing beyond the outputs is written
    # fp64 reference of the backward (from the stored pre-activations)
    g_r = d(gEz) @ d(w2r).T * _dsilu(d(pre_r))
    g_h = (g_r @ d(W1r[P:]).T) @ d(W2l).T * _dsilu(d(pre_l))
    for got, ref in ((gX[:, :P], g_h @ d(W1l[:P]).T + g_r @ d(W1r[:P]).T), (gs, g_h @ d(W1l[P:]).T)):
        assert float((d(got) - ref).abs().max()) <= 2e-4 * float(ref.abs().max())


@pytest.mark.parametrize("backward", [False, True], ids=["fwd", "bwd"])
def test_mlp2_readout_declines_without_writing(backward):
    """x_L 32 wide (S = 32, H = 64): the library declines before anything is enqueued, in both directions."""
    M, S2, P2 = 1000, 32, 64
    gen = torch.Generator(device="cuda").manual_seed(1)
    r = lambda k, n: torch.randn(k, n, generator=gen, device="cuda") / k**0.5
    W1l, W2l, W1r, w2r = r(P2 + U, H), r(H, S2), r(P2 + S2, H), r(H, 1)
    X = torch.randn(M, P2 + S2, generator=gen, device="cuda")
    s = torch.randn(M, U, generator=gen, device="cuda")
    pre_l, pre_r = torch.randn(M, H, generator=gen, device="cuda"), torch.randn(M, H, generator=gen, device="cuda")
    Ez = torch.randn(M, 1, generator=gen, device="cuda")
    before = [t.clone() for t in (X, s, pre_l, pre_r, Ez)]
    if backward:
        W = [_pack(W1r.T), _pack(W2l.T), _pack(W1l.T)]
        assert not _lib.mlp2_readout(True, X[:, :P2], s, None, pre_l, pre_r, Ez, w2r, W, S2)
    else:
        W = [_pack(W1l), _pack(W2l), _pack(W1r[:P2]), _pack(W1r[P2:])]
        assert not _lib.mlp2_readout(False, X[:, :P2], s, X[:, P2:], pre_l, pre_r, Ez, w2r, W, S2)
    torch.cuda.synchronize()
    for t, t0 in zip((X, s, pre_l, pre_r, Ez), before):
        assert torch.equal(t, t0)
