"""The trainable operator ``allegro_b200.nn.Contracter`` on the GPU against the fp64 oracle, at model widths, on both routes.

``Contracter`` runs centre-sorted scatter indices with a full spherical-harmonic second operand on the fused pipeline's
tensor-product kernels (``_fast_product``: ab2_tp_fwd / ab2_tp_bwd, i.e. the streaming, tp_smem / tp_fast and generic
families) and everything else on the generic operator kernels (op.cu).  Every case here compares, for one table, one
channel width and one neighbour list:

- the forward, d/d(weights, x1, x2) of a scalar loss, and the second-order terms a force loss needs (first-order
  gradients with ``create_graph``, a loss on them, differentiated w.r.t. weights, x1 and x2);
- on centre-sorted indices (fast route), on the same edges permuted (generic route) and on sorted indices with
  ALLEGRO_B200_OP_FAST=0;
- with the oracle ``R.Contracter`` in fp64 on the device, loaded with the same weights and coupling tensor rounded to the
  kernel's type, on the same inputs (generated in fp64, rounded to the kernel's type);
- and which kernels ran (torch.profiler): the fast route launches the tensor-product families ``tp_dispatch._expected_for``
  predicts and no ``op_contract_kernel``, the generic route no tensor-product kernel.

The neighbour lists have centres without edges (also the first and last ones), a centre with more than one CTA's share
of the edges, scatter_dim_size beyond the last centre, and enough edges for the weight gradient to span several 512-edge
chunks of ``op_contract_wgrad_kernel``; one list puts every edge on one atom, one has no edges, and one has the c2
benchmark frame's size.  The tail of the file runs a whole reference model with its Contracters replaced, in fp32 and
fp64, through a force-matching training step.
"""
import os

import pytest
import torch

from allegro_b200 import _lib
from allegro_b200.nn import Contracter as B200Contracter
from oracle import nn_ref as R
from oracle import o3_ref
from tp_dispatch import DEFAULTS, FAMILIES, _check_kernels, _expected_for, _families, _from_degrees, _kernels_launched, _ragged_csr, _template_args

pytestmark = pytest.mark.gpu
DEV = "cuda"

# relative to max |reference|, per compared tensor.  fp32: first-order products at the bar of the tensor-product tests
# (test_gpu_tp_ragged._bars); largest error measured over the grid on an H100 80GB HBM3 (700 W): 1.3e-6.  The weight
# gradients sum over all edges (512-edge chunks joined by atomics on the generic route): measured 2.9e-6, bar 1e-5.  The
# second-order terms d/dx1, d/dx2 of a loss on the first-order gradients: measured 5.5e-5 (the kernels' torch restatement
# in fp32 on the CPU errs 2e-5 on the same cases), bar 2e-4.
BARS = {
    torch.float32: {"out": 2e-5, "dL/dx1": 2e-5, "dL/dx2": 2e-5, "dL/dw": 1e-5, "d2/dw": 1e-5, "d2/dx1": 2e-4, "d2/dx2": 2e-4},
    torch.float64: dict.fromkeys(("out", "dL/dx1", "dL/dx2", "dL/dw", "d2/dw", "d2/dx1", "d2/dx2"), 1e-10),
}
FIRST = ("out", "dL/dw", "dL/dx1", "dL/dx2")
SECOND = ("d2/dw", "d2/dx1", "d2/dx2")


# --------------------------------------------------------------------------------------------------------------------
# tables
# --------------------------------------------------------------------------------------------------------------------
def _layer_tables():
    """{name: (irreps_in1, irreps_in2, irreps_out)} of every tensor product of an Allegro model with l_max 0-4 and 1-3
    layers, with the spherical harmonics as allowed irreps and with both parities (R.allegro_layer_irreps)."""
    out = {}
    for lmax in range(5):
        sh = o3_ref.Irreps.spherical_harmonics(lmax)
        both = o3_ref.Irreps([(1, (l, p)) for l in range(lmax + 1) for p in (1, -1)])
        for allowed in (sh, both):
            for L in (1, 2, 3):
                for a, b in zip(*R.allegro_layer_irreps(sh, allowed, L)):
                    key = (repr(a).replace(" ", ""), repr(sh).replace(" ", ""), repr(b).replace(" ", ""))
                    if key not in out.values():
                        name = f"l{lmax}_{a.dim}to{b.dim}"
                        out[name if name not in out else name + "b"] = key
    return out


LAYERS = _layer_tables()
SH2 = "0e+1o+2e"
L2_99 = LAYERS["l2_9to9"]
OFF_MODEL = {  # tables the fused pipeline never builds: D != d_in on the streaming kernels
    "x9_D4": (SH2, "0e+1o", SH2),
    "x4_D9": ("0e+1o", SH2, "0e+1o"),
    "x9_D1": (SH2, "0e", SH2),
    "x9_D16": (SH2, "0e+1o+2e+3o", SH2),
}
NONSQUARE = ("2o+1e+0e", "0e+0o+1e+1o", "1o+2e")  # d2 = 8: the generic route whatever the indices
SUBSET = [(0, 0, 0), (1, 1, 0), (0, 1, 1), (2, 1, 1), (0, 2, 2), (1, 1, 2), (2, 2, 2)]  # of 0e+1o+2e x 0e+1o+2e -> 0e+1o+2e


def _case(table, irreps, U, dtype, kind="ragged", coupling=True, instructions=None, second=True):
    tag = f"{table}-U{U}-{str(dtype)[6:]}-{kind}" + ("" if coupling else "-uncoupled") + ("-subset" if instructions else "")
    return pytest.param(irreps, U, dtype, kind, coupling, instructions, second, id=tag)


def _cases():
    f32, f64 = torch.float32, torch.float64
    cases = []
    for name, irr in {**LAYERS, **OFF_MODEL}.items():
        for U in (32, 64):
            cases.append(_case(name, irr, U, f32))
    cases.append(_case("nonsquare", NONSQUARE, 32, f32))
    cases.append(_case("l2_9to9", L2_99, 32, f32, coupling=False))
    cases.append(_case("l1_4to7", LAYERS["l1_4to7"], 32, f32, coupling=False))
    cases.append(_case("l2_9to9", L2_99, 32, f32, instructions=SUBSET))
    # 8 and 40: the run-time-U streaming builds; 1, 3, 5, 6: declined by the 16-byte row test (12 is not: 48 bytes);
    # 72 and 128: past the streaming builds
    for U in (1, 3, 5, 6, 8, 12, 40, 72, 128):
        for name, irr in (("l2_9to9", L2_99), ("x9_D4", OFF_MODEL["x9_D4"]), ("l1_4to7", LAYERS["l1_4to7"])):
            cases.append(_case(name, irr, U, f32))
    for kind in ("one_atom", "no_edges"):
        for dtype in (f32, f64):
            cases.append(_case("l2_9to9", L2_99, 32, dtype, kind, second=kind != "no_edges"))
    for name, irr in OFF_MODEL.items():
        cases.append(_case(name, irr, 8, f64))
    cases.append(_case("l2_9to9", L2_99, 32, f64))
    cases.append(_case("l1_4to7", LAYERS["l1_4to7"], 8, f64))
    for U, dtype in ((32, f32), (64, f32), (32, f64)):
        cases.append(_case("l2_9to9", L2_99, U, dtype, "c2", second=False))
    return cases


# --------------------------------------------------------------------------------------------------------------------
# neighbour lists and inputs
# --------------------------------------------------------------------------------------------------------------------
def _centres(kind):
    """(centre-sorted scatter indices [E] int64, scatter_dim_size)."""
    if kind == "ragged":  # ~3000 edges: 6 chunks of the weight gradient; 3 atoms past the last centre
        row_ptr, ctr, _ = _ragged_csr(240, 31, long=True, huge=True)
        return ctr.long(), row_ptr.numel() - 1 + 3
    if kind == "one_atom":
        return torch.full((700,), 4, dtype=torch.long), 9
    if kind == "no_edges":
        return torch.zeros(0, dtype=torch.long), 5
    if kind == "c2":  # the benchmark frame's size: 10 976 centres, ~42 edges each
        g = torch.Generator().manual_seed(5)
        row_ptr, ctr, _ = _from_degrees(torch.poisson(torch.full((10976,), 42.0), generator=g).to(torch.int64), 14)
        return ctr.long(), 10976
    raise ValueError(kind)


def _modules(irreps, U, dtype, coupling, instructions, sf=0.37):
    """(fp64 oracle on the device, B200 operator in ``dtype``) with the same weights and coupling tensor, both rounded to
    ``dtype``."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        torch.manual_seed(U)
        i1, i2, io = (o3_ref.Irreps(x) for x in irreps)
        ref = R.Contracter(i1, i2, io, mul=U, instructions=instructions, path_channel_coupling=coupling, scatter_factor=sf)
        with torch.no_grad():
            ref.weights.copy_(ref.weights.to(dtype).double())
            ref.w3j.copy_(ref.w3j.to(dtype).double())
        op = B200Contracter(*irreps, mul=U, instructions=instructions, path_channel_coupling=coupling, scatter_factor=sf)
    finally:
        torch.set_default_dtype(prev)
    op.load_state_dict(ref.state_dict())
    # the dense einsum intermediate of the oracle: at most ~2e8 elements per chunk
    ref.chunk = max(1, int(2e8 // (U * ref.base_dim1 * ref.base_dim2 * ref.base_dim_out)))
    return ref.to(DEV), op.to(DEV, dtype)


def _inputs(op, E, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)

    def r(d):
        return torch.randn(E, op.mul, d, generator=g, dtype=torch.float64, device=DEV).to(dtype).double()

    d1, d2, do = op.base_dim1, op.base_dim2, op.base_dim_out
    return dict(x1=r(d1), x2=r(d2), go=r(do), v1=r(d1), v2=r(d2))


# --------------------------------------------------------------------------------------------------------------------
# the two sides
# --------------------------------------------------------------------------------------------------------------------
def _first_order(c, x, idx, n, dtype):
    """out and d/d(weights, x1, x2) of sum(out * go), all in fp64."""
    a = x["x1"].to(dtype).requires_grad_(True)
    b = x["x2"].to(dtype).requires_grad_(True)
    out = c(a, b, idx, n)
    grads = torch.autograd.grad((out * x["go"].to(dtype)).sum(), [c.weights, a, b])
    return dict(zip(FIRST, [t.detach().double() for t in (out, *grads)]))


def _second_order(c, x, idx, n, dtype):
    """d/d(weights, x1, x2) of (ga . v1) + |gb * v2|^2 with (ga, gb) = d/d(x1, x2) of sum(out * tanh(out))."""
    a = x["x1"].to(dtype).requires_grad_(True)
    b = x["x2"].to(dtype).requires_grad_(True)
    out = c(a, b, idx, n)
    ga, gb = torch.autograd.grad((out * torch.tanh(out)).sum(), [a, b], create_graph=True)
    loss2 = (ga * x["v1"].to(dtype)).sum() + (gb * x["v2"].to(dtype)).pow(2).sum()
    return dict(zip(SECOND, [t.detach().double() for t in torch.autograd.grad(loss2, [c.weights, a, b])]))


def _oracle_first_order(ref, x, idx, n):
    """The oracle's forward (_contract.py:199-211) with gamma = sf * index_add(x2) formed once and the contraction run in
    edge chunks; per-edge outputs are independent given gamma, so d/dx1 is per chunk and d/dgamma, d/dweights add up."""
    E, U = idx.shape[0], ref.mul
    sf = 1.0 if ref.scatter_factor is None else ref.scatter_factor
    gamma = torch.zeros(n, U, ref.base_dim2, dtype=torch.float64, device=DEV).index_add_(0, idx, sf * x["x2"]).requires_grad_(True)
    res = {"out": torch.empty(E, U, ref.base_dim_out, dtype=torch.float64, device=DEV), "dL/dx1": torch.empty_like(x["x1"])}
    ggam, gw = torch.zeros_like(gamma), torch.zeros_like(ref.weights)
    step = max(ref.chunk, 1)
    for s in range(0, E, step):
        e = min(s + step, E)
        a = x["x1"][s:e].detach().requires_grad_(True)
        out = ref._contract(a, gamma[idx[s:e]])
        ga, gg, gwc = torch.autograd.grad(out, [a, gamma, ref.weights], x["go"][s:e])
        res["out"][s:e], res["dL/dx1"][s:e] = out.detach(), ga
        ggam += gg
        gw += gwc
    res["dL/dw"], res["dL/dx2"] = gw, sf * ggam[idx]
    return res


def _rel_errs(got, ref):
    errs = {}
    for k, r in ref.items():
        g = got[k]
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
        assert bool(torch.isfinite(g).all()), f"{k}: non-finite"
        errs[k] = float((g - r).abs().max()) / max(float(r.abs().max()), 1e-30) if r.numel() else 0.0
    return errs


def _perm(res, p):
    """Results of the permuted edge order: per-edge tensors permuted, weight gradients unchanged."""
    return {k: (v if k.endswith("/dw") else v[p]) for k, v in res.items()}


def _is_fast(op, idx):
    """Contracter._fast_route's choice: non-empty centre-sorted indices and a full spherical-harmonic second operand."""
    d2 = op.base_dim2
    return idx.numel() > 0 and round(d2 ** 0.5) ** 2 == d2 and d2 <= 25 and bool((idx[1:] >= idx[:-1]).all())


def _check_route(op, names, fast, dtype, E):
    if names is None:
        return "torch.profiler recorded no CUDA kernel events: values checked, kernel families not"
    contract = [n for n in names if _template_args(n, "op_contract_kernel") is not None]
    tp = [n for n in names if any(_template_args(n, f) is not None for f in FAMILIES)]
    if fast:
        assert not contract, contract
        nnz = op.sparse_table()[0].shape[0]
        _check_kernels(names, *_expected_for(op.base_dim1, op.base_dim_out, op.base_dim2, False, nnz, dtype, op.mul, DEFAULTS))
    else:
        assert not tp, tp
        assert contract or E == 0, names
    return None


# --------------------------------------------------------------------------------------------------------------------
# GPU: the operator grid
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("irreps,U,dtype,kind,coupling,instructions,second", _cases())
def test_operator_vs_oracle(irreps, U, dtype, kind, coupling, instructions, second, monkeypatch):
    for k, v in DEFAULTS.items():
        _lib.set_option(k, v)
    ref, op = _modules(irreps, U, dtype, coupling, instructions)
    idx, n = _centres(kind)
    idx = idx.to(DEV)
    E = idx.shape[0]
    x = _inputs(op, E, dtype, seed=U + E)
    p = torch.randperm(E, generator=torch.Generator().manual_seed(E)).to(DEV)
    xp = {k: v[p] for k, v in x.items()}
    idx_p = idx[p].contiguous()
    bars = BARS[dtype]

    want = _oracle_first_order(ref, x, idx, n)
    if second:
        want.update(_second_order(ref, x, idx, n, torch.float64))
    fast, fast_p = _is_fast(op, idx), _is_fast(op, idx_p)

    got, names = _kernels_launched(lambda: _first_order(op, x, idx, n, dtype), runs=3)
    got_p, names_p = _kernels_launched(lambda: _first_order(op, xp, idx_p, n, dtype), runs=3)
    route = op._tab_cache.get("route")
    assert route[0] is idx_p and (route[3] is not None) == fast_p  # permuted indices take the generic route (unless E = 0 or one atom)
    if second:
        got.update(_second_order(op, x, idx, n, dtype))
        got_p.update(_second_order(op, xp, idx_p, n, dtype))
    monkeypatch.setenv("ALLEGRO_B200_OP_FAST", "0")
    generic = _first_order(op, x, idx.clone(), n, dtype)
    monkeypatch.delenv("ALLEGRO_B200_OP_FAST")

    errs = _rel_errs(got, want)
    errs_p = _rel_errs(_perm(got_p, torch.argsort(p)), want)
    errs_g = _rel_errs(generic, {k: want[k] for k in FIRST})
    cross = _rel_errs({k: got[k] for k in FIRST}, {k: _perm(got_p, torch.argsort(p))[k] for k in FIRST})
    print(f"\n  {' x '.join(irreps)} U={U} {str(dtype)[6:]} {kind}, E={E} fast={fast} sorted: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    print("  permuted: " + " ".join(f"{k} {v:.1e}" for k, v in errs_p.items()))
    print("  OP_FAST=0: " + " ".join(f"{k} {v:.1e}" for k, v in errs_g.items()) + " | sorted vs permuted: "
          + " ".join(f"{k} {v:.1e}" for k, v in cross.items()))
    if names:
        print("  sorted kernels: " + " ".join(_families(names) or ["(no tensor-product kernel)"]))
    bad = [(route_name, k, v) for route_name, ee in (("sorted", errs), ("permuted", errs_p), ("OP_FAST=0", errs_g), ("cross", cross))
           for k, v in ee.items() if not v < bars[k] * (2 if route_name == "cross" else 1)]
    assert not bad, bad
    if E == 0:
        assert bool((got["dL/dw"] == 0).all()) and bool((got_p["dL/dw"] == 0).all())
    skipped = [_check_route(op, names, fast, dtype, E), _check_route(op, names_p, fast_p, dtype, E)]
    if any(skipped):
        pytest.skip(next(s for s in skipped if s))


# --------------------------------------------------------------------------------------------------------------------
# GPU: CUDA-graph capture of the operator
# --------------------------------------------------------------------------------------------------------------------
def test_operator_graph_capture_routes(monkeypatch):
    """A forward captured after an eager call with the same index tensor uses the cached fast route; one captured with an
    index tensor never seen before takes the generic route without synchronising (no index check while capturing).  Both
    replays give the eager results."""
    ref, op = _modules(L2_99, 32, torch.float32, True, None)
    idx, n = _centres("ragged")
    idx = idx.to(DEV)
    x = _inputs(op, idx.shape[0], torch.float32, seed=4)
    x1, x2 = x["x1"].float(), x["x2"].float()
    calls = []
    for name in ("tp_fwd", "op_contract"):
        real = getattr(_lib, name)
        monkeypatch.setattr(_lib, name, lambda *a, _r=real, _n=name: (calls.append(_n), _r(*a))[1])

    with torch.no_grad():
        eager = op(x1, x2, idx, n)
        assert calls == ["tp_fwd"]
        fresh = idx.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            calls.clear()
            g_cached, g_fresh = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
            with torch.cuda.graph(g_cached):
                out_cached = op(x1, x2, idx, n)
            assert calls == ["tp_fwd"], calls
            calls.clear()
            with torch.cuda.graph(g_fresh):
                out_fresh = op(x1, x2, fresh, n)
            assert calls == ["op_contract"], calls
        torch.cuda.current_stream().wait_stream(s)
        g_cached.replay()
        g_fresh.replay()
        torch.cuda.synchronize()
    want = _oracle_first_order(ref, x, idx, n)["out"]
    for got in (eager, out_cached, out_fresh):  # not bitwise: the environment sum is a scatter with atomics
        assert _rel_errs({"out": got.double()}, {"out": want})["out"] < BARS[torch.float32]["out"]


# --------------------------------------------------------------------------------------------------------------------
# GPU: refusals, with every kernel entry point replaced by a sentinel
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def sentinel(monkeypatch):
    def reached(*a, **k):
        raise AssertionError("a kernel entry point was reached with arguments that must be refused")

    for name in ("op_scatter_env", "op_gather_rows", "op_contract", "op_contract_wgrad", "tp_fwd", "tp_bwd", "transpose_ui"):
        monkeypatch.setattr(_lib, name, reached)
    monkeypatch.setattr(_lib, "load", reached)


@pytest.mark.parametrize("sorted_idx", [True, False], ids=["sorted", "unsorted"])
def test_operator_refuses_bad_indices_on_device(sentinel, sorted_idx):
    """Indices outside [0, scatter_dim_size), negative indices and edge counts that differ between x1, x2 and idxs are
    refused on CUDA tensors before any kernel entry point is reached."""
    _, op = _modules(L2_99, 8, torch.float32, True, None)
    E, N = 50, 6
    idx = torch.randint(0, N, (E,), generator=torch.Generator().manual_seed(1)).to(DEV)
    if sorted_idx:
        idx = torch.sort(idx).values
    x1, x2 = torch.randn(E, 8, 9, device=DEV), torch.randn(E, 8, 9, device=DEV)
    for bad, n in ((torch.where(idx == idx.max(), N, idx), N), (idx, int(idx.max())), (idx - 1, N)):
        with pytest.raises(ValueError, match="out of range"):
            op(x1, x2, bad, n)
    for a, b, i in ((x1[:-1], x2, idx), (x1, x2[:-1], idx), (x1, x2, idx[:-1])):
        with pytest.raises(ValueError, match="does not match"):
            op(a, b, i, N)
    with pytest.raises(ValueError):
        op(x1, x2, idx.cpu(), N)


# --------------------------------------------------------------------------------------------------------------------
# GPU: a reference model with its Contracters replaced
# --------------------------------------------------------------------------------------------------------------------
def _frame(n_atoms, seed):
    """An open-boundary frame of H / C / O atoms at ~15 neighbours per atom within 4 A: (data with centre-sorted edges,
    data with the same edges shuffled)."""
    g = torch.Generator().manual_seed(seed)
    side = (18.0 * n_atoms) ** (1 / 3)
    pos = torch.rand(n_atoms, 3, generator=g, dtype=torch.float64) * side
    types = torch.randint(0, 3, (n_atoms,), generator=g)
    d = torch.cdist(pos, pos)
    ei = ((d < 4.0) & ~torch.eye(n_atoms, dtype=torch.bool)).nonzero().T.contiguous()  # row-major: sorted by centre
    shuffled = ei[:, torch.randperm(ei.shape[1], generator=g)]
    return [{R.POSITIONS_KEY: pos, R.ATOM_TYPE_KEY: types, R.EDGE_INDEX_KEY: e} for e in (ei, shuffled)]


def _model_kwargs(name):
    import golden_util

    kw = dict(torch.load(os.path.join(golden_util.GOLDEN, "ref_modifier.pt"), weights_only=False)["kwargs"])
    if name != "ref_modifier":
        lmax, width = (int(v) for v in name.split("_"))
        kw.update(l_max=lmax, num_tensor_features=width)
    return kw


def _energy_forces_and_step(model, data):
    """Energies and forces of an AllegroOracle-shaped model, and d/d(parameters) of a force-matching loss taken through
    ``model.model`` with the forces' graph kept (double backward through every Contracter)."""
    data = {k: v.to(DEV) for k, v in data.items()}
    pos = data[R.POSITIONS_KEY].requires_grad_(True)
    out = model.model(dict(data, **{R.POSITIONS_KEY: pos}))
    energy = out[R.TOTAL_ENERGY_KEY].sum()
    (g,) = torch.autograd.grad(energy, pos, create_graph=True)
    forces = -g
    target = torch.sin(torch.arange(forces.numel(), device=DEV, dtype=torch.float64)).view_as(forces)
    loss = (forces.double() - target).pow(2).sum()
    params = dict(model.model.named_parameters())
    grads = torch.autograd.grad(loss, list(params.values()), allow_unused=True)
    res = {"atomic_energy": out[R.PER_ATOM_ENERGY_KEY].detach().double(), "forces": forces.detach().double()}
    res.update({k: (gr.double() if gr is not None else torch.zeros_like(p, dtype=torch.float64)) for (k, p), gr in zip(params.items(), grads)})
    return res


# (energies and forces, parameter gradients).  fp32, largest measured on an H100 80GB HBM3 (700 W) over two runs: 8.1e-6
# and 8.6e-5.
MODEL_BARS = {torch.float64: (1e-9, 1e-9), torch.float32: (3e-5, 3e-4)}


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["float64", "float32"])
@pytest.mark.parametrize("name", ["ref_modifier", "1_32", "1_64", "2_32", "2_64", "3_32", "3_64"])
def test_replaced_model_energy_forces_and_training_step(name, dtype):
    """enable_B200Contracter on a model built like the reference's (the ref_modifier.pt kwargs: l_max 2, 3 layers, mul 4;
    and l_max 1 / 2 / 3 at 32 and 64 tensor features), on the GPU, against the unmodified fp64 oracle: energies, forces
    and the gradient of a force-matching loss w.r.t. every parameter, on centre-sorted edges (the tensor-product kernels)
    and on the same edges shuffled (the generic operator kernels)."""
    from oracle.model_ref import AllegroOracle

    kw = _model_kwargs(name)
    oracle = AllegroOracle(**dict(kw, model_dtype="float64")).to(DEV)
    model = AllegroOracle(**dict(kw, model_dtype="float32" if dtype == torch.float32 else "float64"))
    model.load_state_dict(oracle.state_dict())
    model = B200Contracter.enable_B200Contracter(model).to(DEV)
    assert all(isinstance(tp, B200Contracter) for tp in model.model.allegro.tps)
    with torch.no_grad():  # the oracle sees the parameters the kernels see
        theirs = dict(model.named_parameters())
        for k, p in oracle.named_parameters():
            p.copy_(theirs[k].double())
    bar_ef, bar_grad = MODEL_BARS[dtype]
    worst = {}
    for order, data in zip(("sorted", "shuffled"), _frame(48, 3)):
        want = _energy_forces_and_step(oracle, data)
        got = _energy_forces_and_step(model, data)
        routes = [tp._tab_cache.get("route") for tp in model.model.allegro.tps]
        assert all((r is not None and r[3] is not None) == (order == "sorted") for r in routes), order
        gmax = max(float(v.abs().max()) for k, v in want.items() if k not in ("atomic_energy", "forces") and v.numel())
        for k, r in want.items():
            ef = k in ("atomic_energy", "forces")
            err = float((got[k] - r).abs().max()) / max(float(r.abs().max()), 1e-30 if ef else 1e-6 * gmax) if r.numel() else 0.0
            what = (order, "E,F" if ef else "dL/dparams")
            worst[what] = max(worst.get(what, 0.0), err)
            assert err < (bar_ef if ef else bar_grad), (order, k, err)
    print(f"\n  {name} {dtype}: " + " ".join(f"{o}/{q} {v:.1e}" for (o, q), v in worst.items()))
