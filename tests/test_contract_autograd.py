"""Host logic of the trainable operator-level Contracter on CPU: the kernels are replaced by the executable specification
(tests/kernel_spec.py), so what is tested is the autograd structure -- every derivative of the trilinear form expressed
through the four products (allegro_b200/nn/_contract.py::_Tri), to second order -- and that the two routes (generic operator
kernels for unsorted indices, the fused pipeline's tensor-product kernels for centre-sorted indices) give the oracle's
numbers.  The CUDA kernels themselves: tests/test_gpu_kernels.py::test_contracter_weight_grad_and_double_backward."""
import pytest
import torch

import kernel_spec
from oracle import nn_ref as R
from oracle import o3_ref


@pytest.fixture()
def spec_kernels(monkeypatch):
    from allegro_b200 import _lib

    for name in kernel_spec.OPERATOR + ("tp_fwd", "tp_bwd"):
        monkeypatch.setattr(_lib, name, getattr(kernel_spec, name))


# l_max 2; l_max 4 with the parity-doubled output of an inner Allegro layer (25 x 25 -> 49: 2052 table entries)
IRREPS = [("0e + 1o + 2e",) * 3, ("0e + 1o + 2e + 3o + 4e", "0e + 1o + 2e + 3o + 4e", "0e + 1e + 1o + 2e + 2o + 3e + 3o + 4e + 4o")]


@pytest.mark.parametrize("irreps", IRREPS, ids=["lmax2", "lmax4"])
@pytest.mark.parametrize("sorted_idx", [False, True], ids=["generic", "sorted"])
@pytest.mark.parametrize("coupling", [True, False])
def test_operator_first_and_second_order_on_cpu(spec_kernels, coupling, sorted_idx, irreps):
    from allegro_b200.nn import B200Contracter

    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        torch.manual_seed(5)
        i1, i2, io = (o3_ref.Irreps(x) for x in irreps)
        mul, E, N = 3, 19, 5
        c_base = R.Contracter(i1, i2, io, mul=mul, path_channel_coupling=coupling, scatter_factor=0.41)
        c_k = B200Contracter(*irreps, mul=mul, instructions=c_base.instructions, path_channel_coupling=coupling, scatter_factor=0.41)
        c_k.load_state_dict(c_base.state_dict())
        idx = torch.randint(0, N, (E,))
        if sorted_idx:
            idx = torch.sort(idx).values
        x1, x2 = torch.randn(E, mul, i1.dim), torch.randn(E, mul, i2.dim)
        go, v1, v2 = torch.randn(E, mul, io.dim), torch.randn(E, mul, i1.dim), torch.randn(E, mul, i2.dim)

        def losses(fwd, weights):
            a, b = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
            out = fwd(a, b)
            first = torch.autograd.grad((out * go).sum(), [weights, a, b], retain_graph=True)
            ga, gb = torch.autograd.grad((out * torch.tanh(out)).sum(), [a, b], create_graph=True)
            second = torch.autograd.grad((ga * v1).sum() + (gb * v2).pow(2).sum(), [weights, a, b])
            return [t.detach() for t in (out, *first, *second)]

        ref = losses(lambda a, b: c_base(a, b, idx, torch.tensor([N])), c_base.weights)
        got = losses(lambda a, b: c_k._forward_impl(a, b, idx, N), c_k.weights)
        route = c_k._tab_cache.get("route")
        assert (route is not None and route[3] is not None) == sorted_idx
        for name, r, g in zip(("out", "dL/dw", "dL/dx1", "dL/dx2", "d2/dw", "d2/dx1", "d2/dx2"), ref, got):
            assert g.shape == r.shape, name
            err = float((g - r).abs().max() / r.abs().max())
            assert err < 1e-10, (name, err)
    finally:
        torch.set_default_dtype(prev)


def _small_operator(sorted_idx=True):
    from allegro_b200.nn import B200Contracter

    torch.manual_seed(7)
    irr = "0e + 1o + 2e"
    c = B200Contracter(irr, irr, irr, mul=3, scatter_factor=0.3).double()
    E, N = 11, 4
    idx = torch.randint(0, N, (E,))
    if sorted_idx:
        idx = torch.sort(idx).values
    return c, torch.randn(E, 3, 9, dtype=torch.float64), torch.randn(E, 3, 9, dtype=torch.float64), idx, N


@pytest.mark.parametrize("sorted_idx", [False, True], ids=["generic", "sorted"])
def test_operator_refuses_bad_indices_before_any_kernel(spec_kernels, sorted_idx):
    """Scatter indices outside [0, scatter_dim_size), negative ones and edge counts that differ between x1, x2 and idxs
    are refused by the Contracter before a kernel sees them; another integer index type gives the int64 result."""
    c, x1, x2, idx, N = _small_operator(sorted_idx)
    ref = c._forward_impl(x1, x2, idx, N)
    with pytest.raises(ValueError, match="out of range"):
        c._forward_impl(x1, x2, torch.where(idx == idx.max(), N, idx), N)
    with pytest.raises(ValueError, match="out of range"):
        c._forward_impl(x1, x2, idx, int(idx.max()))  # scatter_dim_size too small for the same indices
    neg = idx.clone()
    neg[3] = -1
    with pytest.raises(ValueError, match="out of range"):
        c._forward_impl(x1, x2, neg, N)
    for a, b, i in ((x1[:-1], x2, idx), (x1, x2[:-1], idx), (x1, x2, idx[:-1]), (x1[:, :2], x2, idx)):
        with pytest.raises(ValueError, match="does not match"):
            c._forward_impl(a, b, i, N)
    with pytest.raises(TypeError):
        c._forward_impl(x1, x2, idx.double(), N)
    for dt in (torch.int32, torch.int16):
        assert torch.equal(c._forward_impl(x1, x2, idx.to(dt), N), ref)


@pytest.fixture()
def no_library(monkeypatch):
    """Any call into liballegro_b200 fails the test: a refusal must come before the kernel launch."""
    from allegro_b200 import _lib

    def reached(*a, **k):
        raise AssertionError("the library was reached with arguments that must be refused")

    monkeypatch.setattr(_lib, "load", reached)
    return _lib


def test_operator_wrappers_refuse_bad_index_tensors(no_library):
    """The ctypes wrappers of the operator kernels pass idxs to an int64_t* parameter: an index tensor of another type,
    of another length than the operands' rows, or not 1-D is refused before the library is reached."""
    _lib = no_library
    E, N, U, d = 6, 3, 2, 4
    x = torch.zeros(E, U, d)
    tab = torch.zeros(1, 3, dtype=torch.int32)
    cgw = torch.zeros(1, U)
    good = torch.zeros(E, dtype=torch.int64)
    bad = [good.int(), good[:-1], good.view(2, 3), torch.zeros(2 * E, dtype=torch.int64)[::2]]
    for idxs in bad:
        with pytest.raises(RuntimeError, match="idxs"):
            _lib.op_scatter_env(x, idxs, N, 1.0)
        with pytest.raises(RuntimeError, match="idxs"):
            _lib.op_contract(0, U, d, d, d, tab, cgw, x, torch.zeros(N, U, d), idxs, torch.zeros(E, U, d))
        with pytest.raises(RuntimeError, match="idxs"):
            _lib.op_contract_wgrad(U, d, d, d, tab, x, torch.zeros(N, U, d), x, idxs)
    with pytest.raises(RuntimeError, match="idxs"):
        _lib.op_gather_rows(torch.zeros(N, U, d), good.int(), 1.0)
    with pytest.raises(RuntimeError, match="rows"):
        _lib.op_contract(2, U, d, d, d, tab, cgw, x, x[:-1], good, torch.zeros(N, U, d))
    with pytest.raises(RuntimeError, match="rows"):
        _lib.op_contract(1, U, d, d, d, tab, cgw, x, torch.zeros(N, U, d), good, torch.zeros(E - 1, U, d))
    with pytest.raises(RuntimeError, match="rows"):
        _lib.op_contract_wgrad(U, d, d, d, tab, x, torch.zeros(N, U, d), x[:-1], good)
