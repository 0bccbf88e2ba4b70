"""ab2_mlp2_readout, the last latent MLP and the readout MLP in one kernel per direction, against the two ab2_mlp2 calls
it replaces (bitwise, except Ez, which is an fp32 dot product instead of a split-bf16 MMA) and against an fp64 reference."""
import pytest
import torch

from allegro_b200 import _lib

pytestmark = pytest.mark.gpu

S = H = 64  # the width of x_L and the hidden width of both MLPs: the only ones the kernels are built for
C2_M = 461154  # edges of the c2 benchmark frame
# (layers L, U) with P = S L that the shared-memory plans of ab2_mlp2_readout take in both directions at the H100's
# 232 448-byte opt-in limit (bytes: forward, backward).  The forward plan is 1024 + 2 (H (P + U) + 2 S H + H P) 2
# + 4 x 8 KB on-chip tiles + 20 KB epilogue staging + tail + the deepest {raw slots, stages} ring that fits; the backward
# plan holds the three transposed images and twelve 8 KB tiles.  L = 1 runs the readout's layer-1 hook over 2 k-steps
# of the prefix; U = 96 splits gs into 64 + 32 columns.
TAKEN = [
    (1, 32),   # 227 456 (4 raw slots would not fit: 2 slots, 4 stages), 193 664
    (1, 64),   # 202 880 (2 slots, 2 stages), 201 856
    (1, 96),   # 211 072, 210 048
    (1, 128),  # 219 264, 218 240
    (2, 32),   # 227 456, 226 432: the c2 model, about 5 KB below the limit
]
# declined: (2, 64) 235 648 / 234 624 bytes; (3, 32) 260 224 / 259 200; (3, 96) 276 608 / five 64-column chunks of
# [gX[:, :P] | gs] in the backward (the kernel holds four)
DECLINED = [(2, 64), (3, 32), (3, 96)]
M_ROWS = [1, 77, 128, 129, 132 * 128 + 1, 40000]


def _dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def _weights(gen, P, U):
    def w(k, n):
        return (torch.rand(k, n, generator=gen, device="cuda") * 2 - 1) * (3.0 / k) ** 0.5

    return w(P + U, H), w(H, S), w(P + S, H), w(H, 1)


def _pack(W):
    return _lib.linear_pack(W.contiguous())


def _readout_cases():
    cases = [(L, U, M) for L, U in TAKEN for M in M_ROWS] + [(2, 32, C2_M)]
    return [pytest.param(L, U, M, id=f"L{L}-U{U}-M{M}") for L, U, M in cases]


@pytest.mark.parametrize("L,U,M", _readout_cases())
def test_mlp2_readout(L, U, M):
    """Every (L, U) the kernels take, at one row, partial and exact 128-row tiles, one tile more than the 132 SMs hold
    (a persistent CTA runs a second tile) and large M."""
    P = S * L
    gen = torch.Generator(device="cuda").manual_seed(M + 1000 * U + L)
    W1l, W2l, W1r, w2r = _weights(gen, P, U)
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
    # both roundings scale with sum_k |silu(pre_r) w2r| per row (not with |Ez|, which can be small for a single row)
    ez_abs = torch.nn.functional.silu(d(pre_r)).abs() @ d(w2r).abs()
    assert float((Ez - Ez2).abs().max()) <= 1e-5 * float(ez_abs.max())
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
@pytest.mark.parametrize("S2,P2,U", [(32, 64, 32)] + [(S, S * L, U) for L, U in DECLINED],
                         ids=["S32"] + [f"L{L}-U{U}" for L, U in DECLINED])
def test_mlp2_readout_declines_without_writing(S2, P2, U, backward):
    """x_L 32 wide (S = 32, H = 64), and the (L, U) whose plans exceed the shared memory or the chunk table: the library
    declines before anything is enqueued, in both directions."""
    M = 1000
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
