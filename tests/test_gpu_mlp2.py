"""ab2_mlp2, the two-layer SiLU MLP in one kernel, against an fp64 reference and against the two ab2_linear launches it
replaces (bitwise, except the rank-1 backward, whose first stage is an exact fp32 product instead of a split MMA)."""
import pytest
import torch

from allegro_b200 import _lib

pytestmark = pytest.mark.gpu

C2_M = 461154  # edges of the c2 benchmark frame

# (name, backward, A segment widths, hidden width, output segment widths, output accumulate flags): the c2 MLPs
C2_SHAPES = [
    ("fwd.L0", False, [64, 32], 64, [64, 96], [False, False]),
    ("fwd.L1", False, [128, 32], 64, [64], [False]),
    ("fwd.readout", False, [192], 64, [1], [False]),
    ("bwd.readout", True, [1], 64, [192], [False]),
    ("bwd.L1", True, [64], 64, [128, 32], [True, False]),
    ("bwd.L0", True, [64, 96], 64, [64, 32], [True, True]),
]
# the other shapes fp32 models hand to ab2_mlp2 (tests/test_gpu_fp32_grid.py): every stage of the S = H = 32 model
# (U = 32, L = 2; the fused readout declines H = 32, so the last latent MLP and the readout run here), and the first
# inner latent MLP of a U = 64 model (N = 64 + 3 x 64 = 256: four 64-column chunks, the most the kernel holds)
MODEL_SHAPES = C2_SHAPES + [
    ("H32.fwd.L0", False, [32, 32], 32, [32, 96], [False, False]),
    ("H32.fwd.L1", False, [64, 32], 32, [32], [False]),
    ("H32.fwd.readout", False, [96], 32, [1], [False]),
    ("H32.bwd.readout", True, [1], 32, [96], [False]),
    ("H32.bwd.L1", True, [32], 32, [64, 32], [True, False]),
    ("H32.bwd.L0", True, [32, 96], 32, [32, 32], [True, True]),
    ("U64.fwd.L0", False, [64, 64], 64, [64, 192], [False, False]),
    ("U64.bwd.L0", True, [64, 192], 64, [64, 64], [True, True]),
]


def _dsilu(x):
    s = torch.sigmoid(x)
    return s * (1 + x * (1 - s))


def _views(M, widths, gen, pad=32):
    """Column views of one wider buffer (leading dimension > width)."""
    buf = torch.randn(M, sum(widths) + pad, generator=gen, device="cuda")
    out, c = [], 0
    for w in widths:
        out.append(buf[:, c : c + w])
        c += w
    return out


def _case(M, backward, a_w, H, o_w, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    K, N = sum(a_w), sum(o_w)
    a = _views(M, a_w, gen)
    W1 = (torch.randn(K, H, generator=gen, device="cuda") / K**0.5).contiguous()
    W2 = (torch.randn(H, N, generator=gen, device="cuda") / H**0.5).contiguous()
    pre = torch.randn(M, H, generator=gen, device="cuda") if backward else torch.empty(M, H, device="cuda")
    init = _views(M, o_w, gen)
    return a, W1, W2, pre, init


def _fused(a, W1, W2, pre, init, accum, backward):
    outs = [t.clone() for t in init]  # clone() of a view is contiguous: also checks ld == width
    pre = pre.clone()
    ok = _lib.mlp2(a, W1, W2, outs, pre, o_accum=accum, backward=backward, W1_packed=_lib.linear_pack(W1), W2_packed=_lib.linear_pack(W2))
    return ok, outs, pre


def _pair(a, W1, W2, pre, init, accum, backward):
    """The two ab2_linear launches PackedMLP ran before the fused kernel."""
    M, H = a[0].shape[0], W1.shape[1]
    outs = [t.clone() for t in init]
    if not backward:
        h = torch.empty(M, H, device="cuda")
        _lib.linear(a, W1, [h], W_packed=_lib.linear_pack(W1))
        _lib.linear([h], W2, outs, o_accum=accum, act=_lib.ACT_SILU, W_packed=_lib.linear_pack(W2))
        return outs, h
    g = torch.empty(M, H, device="cuda")
    if W1.shape[0] == 1:  # the readout's one-column gradient, zero-padded to K = 16
        gp = torch.zeros(M, 16, device="cuda")
        gp[:, :1] = a[0]
        W1p = torch.zeros(16, H, device="cuda")
        W1p[:1] = W1
        _lib.linear([gp], W1p, [g], epi=_lib.EPI_MUL_DSILU, aux=pre, W_packed=_lib.linear_pack(W1p))
    else:
        _lib.linear(a, W1, [g], epi=_lib.EPI_MUL_DSILU, aux=pre, W_packed=_lib.linear_pack(W1))
    _lib.linear([g], W2, outs, o_accum=accum, W_packed=_lib.linear_pack(W2))
    return outs, pre


def _reference(a, W1, W2, pre, init, accum, backward):
    A = torch.cat([t.double() for t in a], dim=-1)
    h = A @ W1.double()
    if backward:
        h = h * _dsilu(pre.double())
    else:
        pre = h
        h = torch.nn.functional.silu(h)
    out = h @ W2.double()
    res, c = [], 0
    for t, acc in zip(init, accum):
        blk = out[:, c : c + t.shape[1]]
        res.append(blk + t.double() if acc else blk)
        c += t.shape[1]
    return res, pre


def _rel(x, ref):
    return float((x.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _check(M, backward, a_w, H, o_w, accum, seed=0):
    a, W1, W2, pre, init = _case(M, backward, a_w, H, o_w, seed)
    ok, outs, pre_f = _fused(a, W1, W2, pre, init, accum, backward)
    assert ok, "ab2_mlp2 declined an eligible case"
    pair, pre_p = _pair(a, W1, W2, pre, init, accum, backward)
    ref, pre_r = _reference(a, W1, W2, pre, init, accum, backward)
    torch.cuda.synchronize()
    rank1 = backward and sum(a_w) == 1
    for o, p, r in zip(outs, pair, ref):
        assert _rel(o, r) < 1e-4
        if rank1:
            assert _rel(o, p.double()) < 1e-5
        else:
            assert torch.equal(o, p), float((o - p).abs().max())
    if not backward:
        assert torch.equal(pre_f, pre_p)
        assert _rel(pre_f, pre_r) < 1e-4
    else:
        assert torch.equal(pre_f, pre)  # read only


@pytest.mark.parametrize("shape", MODEL_SHAPES, ids=[s[0] for s in MODEL_SHAPES])
def test_mlp2_c2_shapes(shape):
    _, backward, a_w, H, o_w, accum = shape
    _check(C2_M, backward, a_w, H, o_w, accum)


# one row, a partial and an exact 128-row tile, and one tile less / more than the 132 SMs hold (with M = 132 x 128 + 1
# a persistent CTA runs a second, one-row tile)
@pytest.mark.parametrize("M", [1, 77, 128, 129, 132 * 128 - 1, 132 * 128 + 1, 40000])
@pytest.mark.parametrize("shape", MODEL_SHAPES, ids=[s[0] for s in MODEL_SHAPES])
def test_mlp2_partial_tiles(shape, M):
    _, backward, a_w, H, o_w, accum = shape
    _check(M, backward, a_w, H, o_w, accum, seed=M)


@pytest.mark.parametrize("accum", [[False, False], [True, False], [False, True], [True, True]])
@pytest.mark.parametrize("backward", [False, True])
def test_mlp2_accumulate_flags(backward, accum):
    _check(5000, backward, [32, 64], 32, [96, 64], accum, seed=7)


def test_mlp2_not_eligible_falls_back():
    """Hidden width 128 with a first matrix too wide to stay resident: ab2_mlp2 declines, nothing is written, and
    PackedMLP's two-launch path is what runs."""
    M, K, H, N = 1000, 320, 128, 64
    a, W1, W2, pre, init = _case(M, False, [K], H, [N])
    outs = [torch.full_like(init[0], 7.0)]
    ok = _lib.mlp2(a, W1, W2, outs, pre, W1_packed=_lib.linear_pack(W1), W2_packed=_lib.linear_pack(W2))
    torch.cuda.synchronize()
    assert not ok
    assert bool((outs[0] == 7.0).all())
    # bf16 storage is not taken either
    ok = _lib.mlp2([t.bfloat16() for t in a], W1.bfloat16(), W2.bfloat16(), [outs[0].bfloat16()], pre.bfloat16(),
                   W1_packed=_lib.linear_pack(W1.bfloat16()), W2_packed=_lib.linear_pack(W2.bfloat16()))
    assert not ok
