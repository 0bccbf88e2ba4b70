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
